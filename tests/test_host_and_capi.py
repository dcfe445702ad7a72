"""Host-side logic + C-ABI surface (no GPU compute)."""
import ctypes
import os
import re

import pytest
import torch

from conftest import ROOT, load_golden, max_rel
import diff_pruning_b200 as dp
from oracle import unet_oracle as orc


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200 import _lib as L
    lib = L.load()
    hdr = open(os.path.join(ROOT, "include", "dpb200.h")).read()
    declared = set(re.findall(r"\b(dp_[a-z0-9_]+)\s*\(", hdr))
    declared -= {n for n in declared if n.endswith("_args")}
    assert len(declared) >= 30
    for name in sorted(declared):
        assert hasattr(lib, name), name
        assert name in L.EXPORTS, f"{name} declared in dpb200.h but not bound in _lib.py"
    assert lib.dp_version() == 100
    assert b"NULL" in lib.dp_strerror(-5)
    # argument validation happens before any launch: safe to call without a GPU
    assert lib.dp_conv2d_fprop(None, None) == -5
    a = L.ConvArgs()
    assert lib.dp_conv2d_fprop(ctypes.byref(a), None) == -5
    assert lib.dp_groupnorm_workspace_bytes(16, 1024, 128, 32) > 0


def test_struct_layouts_match_header():
    from diff_pruning_b200 import _lib as L
    assert ctypes.sizeof(L.ConvArgs) == 56 + 18 * 8
    assert ctypes.sizeof(L.GemmArgs) == 16 + 11 * 8 + 8
    assert ctypes.sizeof(L.WgradReduceArgs) == 24 + 7 * 8
    assert ctypes.sizeof(L.TaylorArgs) == 16 + 8 * 8
    assert ctypes.sizeof(L.GnArgs) == 24 + 19 * 8 + 8 + 8 + 8 + 16 + 16 + 8
    assert ctypes.sizeof(L.ConvBf16Args) == 56 + 13 * 8
    assert ctypes.sizeof(L.AdamArgs) == 8 + 6 * 8 + 6 * 8 + 4 + 4 + 8


def test_no_cpu_fallback():
    torch.manual_seed(0)
    m = dp.UNet2DModel(**dp.TINY_TEST_CONFIG)
    with pytest.raises(RuntimeError, match="No CPU fallback"):
        m(torch.randn(1, 3, 16, 16), torch.tensor([1]))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        dp.DDPMScheduler().add_noise(torch.randn(1, 3, 4, 4), torch.randn(1, 3, 4, 4), torch.tensor([1]))


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "diff-pruning_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "oracle" not in src.replace("# oracle", ""), fn


def test_module_tree_matches_reference_and_trace_mode_equals_oracle():
    G = load_golden("cifar_fwd.pt")
    torch.manual_seed(0)
    m = dp.UNet2DModel(**dp.CIFAR10_DDPM_CONFIG).eval()
    assert list(m.state_dict().keys()) == list(G["sd_fp"].keys())
    g1, g2 = torch.Generator().manual_seed(1), torch.Generator().manual_seed(2)
    clean, noise = torch.randn(16, 3, 32, 32, generator=g1)[:2], torch.randn(16, 3, 32, 32, generator=g2)[:2]
    t = (500 * torch.ones(2)).long()
    with torch.no_grad(), dp.trace_mode():
        out = m(dp.DDPMScheduler().add_noise(clean, noise, t), t).sample
    assert max_rel(out, G["eps_b2"][500]) < 1e-5
    # forward hooks fire on real leaf modules in trace mode (what dependency tracing needs, SURVEY.md §3.4)
    seen = []
    hs = [mod.register_forward_hook(lambda mod_, i, o: seen.append(type(mod_).__name__))
          for mod in m.modules() if isinstance(mod, (torch.nn.Conv2d, torch.nn.Linear, torch.nn.GroupNorm))]
    with dp.trace_mode():
        out = m(torch.randn(1, 3, 32, 32), torch.ones(1).long()).sample
    for h in hs:
        h.remove()
    assert len(seen) == 65 + 48 + 51 - 0 and out.grad_fn is not None   # SURVEY.md §8(a) A3 leaf counts


def test_lsun_config_param_count():
    torch.manual_seed(0)
    m = dp.UNet2DModel(**dp.LSUN256_DDPM_CONFIG)
    assert round(sum(p.numel() for p in m.parameters()) / 1e6, 3) == 113.673   # SURVEY.md §8 "C3"


def test_ddim_timesteps_host_logic():
    """The reference's modified timestep spacing (scheduling_ddim.py:257-266) — pure host logic."""
    from diff_pruning_b200.sampling import DDIMScheduler
    G = load_golden("ddim_tiny.pt")
    for name in ("uniform_eta0", "quad_eta05"):
        s = DDIMScheduler(num_train_timesteps=1000, skip_type=G[name]["skip_type"])
        s.set_timesteps(G[name]["steps"])
        assert torch.equal(s.timesteps, G[name]["timesteps"])
    s = DDIMScheduler.from_config(dp.DDPMScheduler(num_train_timesteps=1000).config)
    assert s.config.clip_sample and s.skip_type == "uniform"


def test_wgrad_split_count_respects_wave_boundaries():
    """engine._wgrad_splits: the tensor-core wgrad runs one CTA per SM, so tiles x splits must not spill a few CTAs into an
    extra wave (the 592 -> 594 CTA bug), every split must be non-empty, and the modelled cost must beat the old rule."""
    import diff_pruning_b200  # noqa: F401
    from diff_pruning_b200.engine import _wgrad_splits, _SM_COUNT, _WGRAD_CTA_OVERHEAD
    cases = [(9, 4096), (36, 1024), (144, 256), (54, 1024), (72, 1024), (4, 1024), (1, 4096), (144, 64), (18, 4096), (7, 4096),
             (1, 1), (300, 64), (2, 3)]
    for tiles, chunks in cases:
        sp = _wgrad_splits(tiles, chunks)
        assert 1 <= sp <= chunks
        cps = -(-chunks // sp)
        assert cps * (sp - 1) < chunks, (tiles, chunks, sp)          # last split non-empty
        ctas = tiles * sp
        waves = -(-ctas // _SM_COUNT)
        if tiles <= _SM_COUNT:
            # the last wave is not a near-empty straggler: either one wave, or the grid fills >= 80 % of its waves
            assert waves == 1 or ctas >= 0.8 * waves * _SM_COUNT, (tiles, chunks, sp, ctas)
        old = max(1, min((592 + tiles - 1) // tiles, (chunks * 32 + 511) // 512))
        old = -(-chunks // -(-chunks // old)) if old <= chunks else old
        cost = lambda s: -(-(tiles * s) // _SM_COUNT) * (_WGRAD_CTA_OVERHEAD + -(-chunks // s))
        assert cost(sp) <= cost(min(old, chunks)), (tiles, chunks, sp, old)


def test_tc_weight_row_padding_rule():
    """dp_tc_weight_row (host function of the C-ABI), fp16 elements: 16-byte multiples up to 64 channels, 128-byte multiples beyond."""
    from diff_pruning_b200 import _lib as L
    lib = L.load()
    for c, want in [(1, 8), (3, 8), (8, 8), (27, 32), (64, 64), (65, 128), (90, 128), (96, 128), (128, 128), (179, 192), (358, 384),
                    (512, 512)]:
        assert lib.dp_tc_weight_row(c) == want, (c, lib.dp_tc_weight_row(c), want)
    assert lib.dp_tc_weight_row(0) == 0


def test_planner_fuses_qkv_and_moves_groupnorm_param_grads_off_the_chain():
    """Host-side planning only (no launch): with the tensor path forced on, a CPU-built plan of the tiny UNet shows the launch structure
    the GPU runs — to_q / to_k / to_v as one fprop and one dgrad with three weight gradients (engine.conv_qkv), and every GroupNorm's
    dgamma / dbeta launch flagged for the side stream right behind its dx launch."""
    from collections import Counter
    from diff_pruning_b200 import engine

    class P(engine.Plan):
        def _build(self):
            self.tc = True          # what dp_tc_available() answers on an sm_90a device
            return super()._build()

    torch.manual_seed(0)
    m = dp.UNet2DModel(**dp.TINY_TEST_CONFIG)
    n_attn = sum(1 for mod in m.modules() if type(mod).__name__ == "Attention")
    n_gn = sum(1 for mod in m.modules() if isinstance(mod, torch.nn.GroupNorm))
    assert n_attn > 0

    def counts(fuse):
        P.FUSE_QKV = fuse
        try:
            p = P(m, 2, 16, 16, "cpu", need_grad=True)
        finally:
            P.FUSE_QKV = True
        return p, Counter(f.what for f in p.fwd), Counter(f.what for f in p.bwd_steps), Counter(f.what for f in p.pack)

    p1, f1, b1, k1 = counts(True)
    p0, f0, b0, k0 = counts(False)
    assert f0["conv fprop"] - f1["conv fprop"] == 2 * n_attn and b0["conv dgrad"] - b1["conv dgrad"] == 2 * n_attn
    assert b0["conv wgrad"] == b1["conv wgrad"] and b0["conv wgrad reduce"] == b1["conv wgrad reduce"]
    assert k1["pack qkv"] == 6 * n_attn and k0["pack qkv"] == 0          # three weights + three biases gathered per block
    assert f1["gn fwd"] == n_gn and b1["gn bwd"] == n_gn and b1["gn bwd param"] == n_gn
    steps = p1.bwd_steps
    for i, f in enumerate(steps):
        if f.what == "gn bwd":
            assert steps[i + 1].what == "gn bwd param" and getattr(steps[i + 1], "side", 0) == 2 and not getattr(f, "side", 0)


def test_groupnorm_param_split_argument_checks():
    """dp_groupnorm_bwd_param / the `fin` field: validation happens before any launch (no GPU needed; the pointers are never dereferenced
    on the host).  The one-pixel LayerNorm shapes take dgamma / dbeta from x and dy, so `fin` is refused there."""
    from diff_pruning_b200 import _lib as L
    lib = L.load()
    a = L.GnArgs()
    fake = 0x10000
    a.N, a.HW, a.C, a.G, a.eps, a.silu = 64, 1, 320, 1, 1e-5, 0
    a.x, a.ldx, a.gamma, a.beta, a.mean, a.rstd, a.workspace = fake, 320, fake, fake, fake, fake, fake
    a.dy, a.lddy, a.dx, a.lddx = fake, 320, fake, 320
    assert lib.dp_groupnorm_bwd_param(ctypes.byref(a), None) == -5          # no fin
    a.fin = fake
    assert lib.dp_groupnorm_bwd(ctypes.byref(a), None) == -3                # LayerNorm rows + fin
    assert lib.dp_groupnorm_bwd_param(ctypes.byref(a), None) == -3
    assert lib.dp_groupnorm_bwd_param(None, None) == -5
    assert lib.dp_copy_rows(None, 4, None, 4, 1, 4, None) == -5
    assert lib.dp_copy_rows(fake, 2, fake, 4, 1, 4, None) == -1             # row pitch shorter than the row
