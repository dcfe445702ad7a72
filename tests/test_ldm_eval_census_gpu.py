"""Launch census of the class-conditional LDM evaluation path at the batch sizes its scripts run: guided DDIM sampling of cin256-v2 at
2 x 6 images per forward (prune_ldm's sample-then-score loop, n_samples_per_class = 6) and at 2 x 50 (sample_for_FID, batch_size = 50),
and the VQ-f4 decode of 8 latents of 64 x 64 (sample_for_FID's decode_batch = 8) to 8 x 256 x 256 images.  Each configuration is
captured in one eager run; every distinct launch (launch_census.launch_key) is replayed on fresh seeded buffers at its own geometry and
checked against float64 with the replays of the training and evaluation censuses, the VQ census and the dp_ddim_cfg_step census.

Then the batch positions of the 2 x 50 no-grad forward against the float64 oracle: images {0, 1, 49, 50, 98, 99} of one run_forward of
the batch-100 plan (context [uc x 50; 50 class contexts], t = 500), the first and last image of each half and the boundary where the
conditional half begins, which a per-launch replay on fresh buffers does not see.
"""
import gc

import pytest
import torch

import launch_census as lc
from conftest import max_rel
from test_eval_census_gpu import EVAL_REPLAY, _LOG
from test_launch_census_gpu import S, _capture, _config, _unique, lib  # noqa: F401  (lib: the module-scoped fixture)
from test_ldm_sampling_gpu import _c5_ld, _conds, replay_ddim_cfg_step
from test_vq_decoder_gpu import _replay_decode_images, _replay_vq, _vq_f4

pytestmark = pytest.mark.gpu

REPLAY = dict(EVAL_REPLAY)
REPLAY.update({"dp_vq_quantize": _replay_vq, "dp_decode_images": _replay_decode_images, "dp_ddim_cfg_step": replay_ddim_cfg_step})

_C5_KEYS = []         # launch keys of the C5 b6 training census (the Taylor pass of test_launch_census_gpu), captured once


def _ldm_sample(B, eta, seed):
    """A guided (scale 3) DDIM sample of cin256-v2, S = 2, at batch_size B (2B images per forward): B distinct classes against the
    unconditional class 1000."""
    from diff_pruning_b200.ldm_sampling import DDIMSampler
    ld, _ = _c5_ld()
    labels = torch.randperm(1000, generator=torch.Generator().manual_seed(seed))[:B]
    c, uc = _conds(ld, labels, torch.full((B,), 1000))

    def run():
        sm = DDIMSampler(ld)
        sm.use_graph = False
        sm.sample(S=2, batch_size=B, shape=[3, 64, 64], conditioning=c, eta=eta, unconditional_guidance_scale=3.0,
                  unconditional_conditioning=uc, generator=torch.Generator().manual_seed(seed))
    return run


def _vq_decode(B):
    m = _vq_f4().cuda()
    m.use_graph = False
    m.decode_batch = B
    h = (torch.randn(B, 3, 64, 64, generator=torch.Generator().manual_seed(8)) * 2e-4).cuda()

    def run():
        from diff_pruning_b200 import _lib as L
        y = m.decode_chunk(h).plan.y_out
        u8 = torch.empty(B, y.H, y.W, 3, dtype=torch.uint8, device="cuda")
        f = torch.empty(B, 3, y.H, y.W, device="cuda")
        assert (y.H, y.W) == (256, 256)
        assert L.load().dp_decode_images(y.ptr, y.ld, B, 3, y.H, y.W, u8.data_ptr(), f.data_ptr(), S()) == 0
    return run


LDM_KINDS = {"dp_conv2d_fprop", "dp_groupnorm_fwd", "dp_gemm_nt_tc", "dp_split_h3", "dp_softmax_fwd", "dp_ddim_cfg_step",
             "dp_nchw_to_nhwc"}
VQ_KINDS = {"dp_vq_quantize", "dp_decode_images", "dp_conv2d_fprop", "dp_groupnorm_fwd", "dp_gemm_nt_tc", "dp_split_h3",
            "dp_upsample2x_fwd"}
CONFIGS = {
    "LDM guided DDIM cin256-v2 2x6": (lambda: _ldm_sample(6, 0.0, 61), LDM_KINDS),
    "LDM guided DDIM cin256-v2 2x50": (lambda: _ldm_sample(50, 0.5, 62), LDM_KINDS),
    "VQ-f4 decode b8": (lambda: _vq_decode(8), VQ_KINDS),
}


def _c5_training_keys(lib):
    if not _C5_KEYS:
        run = _config("C5 b6")
        _C5_KEYS.append({lc.launch_key(n, lc.argkinds(n), a) for n, a in _capture(lib, run)})
        del run
        gc.collect()
        torch.cuda.empty_cache()
    return _C5_KEYS[0]


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_ldm_eval_census(lib, tag, monkeypatch):
    make, must = CONFIGS[tag]
    run = make()
    calls = _capture(lib, run)
    del run
    gc.collect()              # the plans and their models form reference cycles
    torch.cuda.empty_cache()
    kinds = {n for n, _ in calls}
    assert must <= kinds, f"{tag}: the plan no longer issues {sorted(must - kinds)}"
    missing = kinds - set(REPLAY)
    assert not missing, f"{tag}: launch kinds without a replay: {sorted(missing)}"
    if tag.endswith("2x50"):      # eta 0.5: the sigma-noise path of the update, at the batch-50 geometry
        assert any(a[3] for n, a in calls if n == "dp_ddim_cfg_step"), "no dp_ddim_cfg_step launch took the noise path"
    uniq = _unique(calls)
    c5 = _c5_training_keys(lib)
    new = sum(1 for n, a in uniq if lc.launch_key(n, lc.argkinds(n), a) not in c5)
    # chain lengths of the product-sum replays: every replay asserts L <= L_MAX for its tensor-core launches; recorded here for the log
    Ls = []
    for fn in ("chain_fprop", "chain_general"):
        orig = getattr(lc, fn)
        monkeypatch.setattr(lc, fn, lambda *a, orig=orig, **kw: Ls.append(orig(*a, **kw)) or Ls[-1])
    _LOG.clear()
    _LOG.update(geoms=set(), tc=[], simt=set())
    rep, count, failures = {}, {}, []
    g = torch.Generator().manual_seed(2027)
    for name, args in uniq:
        count[name] = count.get(name, 0) + 1
        try:
            REPLAY[name](lib, g, name, args[0] if len(args) == 1 else args, rep)
        except AssertionError as e:          # report every failing launch of the config, not just the first
            failures.append(f"{name}: {e}".splitlines()[0])
        torch.cuda.synchronize()
    for f in failures:
        print(f"  FAIL {tag}: {f}")
    assert not failures, f"{tag}: {len(failures)} launches failed their checks"
    assert set(rep) == kinds, (tag, sorted(kinds - set(rep)))     # every kind the plan issued was checked
    assert Ls and max(Ls) <= lc.L_MAX, (min(Ls, default=None), max(Ls, default=None))
    print(f"\n{tag}: {len(calls)} launches, {len(uniq)} unique, {len(kinds)} kinds, all replayed; "
          f"{new} unique keys not in the C5 b6 training census; L in [{min(Ls)}, {max(Ls)}]")
    for name in sorted(rep):
        print(f"  {tag:32s} {name:26s} {count[name]:4d} unique, worst err/bound {max(rep[name]):.3f}")


# ---------------------------------------------------------------------------------------------------------------- batch positions
def test_cin256_v2_batch_100_forward_positions_match_fp64_oracle():
    """The no-grad cin256-v2 plan at batch 100 as DDIMSampler builds it for sample_for_FID's guided sampling at batch_size 50: context
    [uc x 50; 50 distinct class contexts], t = 500, one run_forward; eps_hat of images {0, 1, 49, 50, 98, 99} against ldm_oracle's
    unet_forward in float64 on those images alone, max-rel < 1e-4 each (the criterion of the full-width LDM pass)."""
    from oracle import ldm_oracle as lorc
    from diff_pruning_b200.engine import frozen_weights, get_plan
    ld, cfg = _c5_ld()
    unet = ld.model.diffusion_model.eval()
    B = 50
    labels = torch.randperm(1000, generator=torch.Generator().manual_seed(63))[:B]
    c, uc = _conds(ld, labels, torch.full((B,), 1000))
    ctx = torch.cat([uc, c])
    x = torch.randn(2 * B, 3, 64, 64, generator=torch.Generator().manual_seed(64)).cuda()
    t = torch.full((2 * B,), 500, dtype=torch.long, device="cuda")
    with torch.no_grad(), frozen_weights(unet):
        plan = get_plan(unet, 2 * B, 64, 64, x.device, need_grad=False)
        plan.ensure_packed()
        plan.load_context(ctx)
        plan.load_input_nchw(x, t)
        plan.run_forward()
        out = plan.output_nchw()
        torch.cuda.synchronize()
    del plan
    gc.collect()
    torch.cuda.empty_cache()
    idx = [0, 1, 49, 50, 98, 99]
    sd = {k: v.detach().double() for k, v in unet.state_dict().items()}
    with torch.no_grad():
        ref = lorc.unet_forward(sd, cfg, x[idx].double(), t[idx], ctx[idx].double())
    errs = {i: max_rel(out[i], ref[j]) for j, i in enumerate(idx)}
    print("\ncin256-v2 batch 100 forward, eps_hat max-rel per image: " + ", ".join(f"{i}: {e:.2e}" for i, e in errs.items()))
    assert all(e < 1e-4 for e in errs.values()), errs
