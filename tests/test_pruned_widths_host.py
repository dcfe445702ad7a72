"""The pruned networks the GPU tests of test_pruned_census_gpu.py run, built on the host: C1 (CIFAR-10 DDPM) and C3 (LSUN-256 DDPM)
pruned by the reference's call sequence (ddpm_prune.py:79-116 on the compat `torch_pruning` names: MagnitudePruner, local pruning, one
iterative step, seed-0 init, ignored_layers=[conv_out]).  Quotas do not depend on the importance, so Taylor pruning gives the same
shapes.  Each ratio gives different channel widths, and widths are where the engine has special cases: activation pitches rounded up
to 4 floats, the fused q / k / v buffer with its per-part pitch, flat-extent SiLU / loss kernels running over pads, N / C tails of
the tensor-core tiles, GroupNorm with an odd number of channels per group, padded weight rows and bf16 pitches rounded to 8.

Pinned here: the parameter count and the set of (in, out) widths of every convolution / linear layer of each network, and what the
sweep covers (a non-GroupNorm width in every residue class mod 4, the channels-per-group values).  If the sweep is edited, these
tests say what it stopped covering.  Also here: poisoned_alloc, the allocation hook of the poisoned-plan tests, and its self-test.
"""
import contextlib
import functools
import math
import os
import sys
from unittest import mock

import pytest
import torch
import torch.nn as nn

from conftest import ROOT
import diff_pruning_b200 as dp

# (family, ratio) of every network of the sweep; the reference's scripts prune at 0.05 - 0.5 (prune_cifar_ddpm_ssim.sh,
# prune_bedroom_ddpm.sh: C3 at 0.3 ...), 0.7 adds widths 76 / 153
SWEEP = [("C1", 0.05), ("C1", 0.15), ("C1", 0.2), ("C1", 0.3), ("C1", 0.5), ("C1", 0.7), ("C3", 0.3)]


def _compat():
    path = os.path.join(ROOT, "diff-pruning_b200", "compat")
    if path not in sys.path:
        sys.path.insert(0, path)
    import torch_pruning as tp
    from diffusers.models.resnet import Downsample2D, Upsample2D
    return tp, (Downsample2D, Upsample2D)


def build_pruned(family: str, ratio: float) -> nn.Module:
    """A fresh seed-0 C1 / C3 UNet on the host, pruned at `ratio` by magnitude through the compat call sequence (ratio 0: unpruned)."""
    cfg, hw = {"C1": (dp.CIFAR10_DDPM_CONFIG, 32), "C3": (dp.LSUN256_DDPM_CONFIG, 256)}[family]
    torch.manual_seed(0)
    m = dp.UNet2DModel(**cfg).eval()
    if ratio:
        tp, resamplers = _compat()
        ex = {"sample": torch.randn(1, 3, hw, hw), "timestep": torch.ones((1,)).long()}
        pr = tp.pruner.MagnitudePruner(m, ex, importance=tp.importance.MagnitudeImportance(), iterative_steps=1, channel_groups={},
                                       ch_sparsity=ratio, ignored_layers=[m.conv_out])
        for g in pr.step(interactive=True):
            g.prune()
        for mod in m.modules():                      # ddpm_prune.py:112-116
            if isinstance(mod, resamplers):
                mod.channels = mod.conv.in_channels
    return m


@functools.lru_cache(maxsize=None)
def _built(family, ratio):
    return build_pruned(family, ratio)


def widths(m: nn.Module):
    """(set of (in, out) widths of the convolutions / linears, set of GroupNorm widths, set of channels per GroupNorm group)."""
    io = set()
    for mod in m.modules():
        if isinstance(mod, nn.Conv2d):
            io.add((mod.in_channels, mod.out_channels))
        elif isinstance(mod, nn.Linear):
            io.add((mod.in_features, mod.out_features))
    gns = [mod for mod in m.modules() if isinstance(mod, nn.GroupNorm)]
    return io, {g.num_channels for g in gns}, {g.num_channels // g.num_groups for g in gns}


# parameter count, (in, out) widths of every convolution / linear, channels per GroupNorm group
PINNED = {
    ("C1", 0.05): (35373909, {(3, 128), (128, 3), (128, 128), (128, 256), (128, 486), (243, 256), (256, 128), (256, 243), (256, 256),
                              (384, 128), (384, 256), (486, 128), (486, 256), (486, 486), (512, 243), (512, 256)},
                   {4, 8, 12, 16}),
    ("C1", 0.15): (27824216, {(3, 128), (128, 3), (128, 128), (128, 224), (128, 435), (217, 224), (224, 217), (224, 224), (256, 128),
                              (352, 128), (352, 224), (435, 128), (435, 224), (435, 435), (448, 217), (448, 224)},
                   {4, 7, 8, 11, 14}),
    ("C1", 0.2): (27496590, {(3, 128), (128, 3), (128, 128), (128, 224), (128, 409), (204, 224), (224, 204), (224, 224), (256, 128),
                             (352, 128), (352, 224), (409, 128), (409, 224), (409, 409), (448, 204), (448, 224)},
                  {4, 7, 8, 11, 14}),
    ("C1", 0.3): (19851157, {(3, 96), (96, 3), (96, 96), (96, 192), (128, 358), (179, 192), (192, 96), (192, 179), (192, 192),
                             (288, 96), (288, 192), (358, 96), (358, 192), (358, 358), (384, 179), (384, 192)},
                  {3, 6, 9, 12}),
    ("C1", 0.5): (8968451, {(3, 64), (64, 3), (64, 64), (64, 128), (128, 64), (128, 128), (128, 256), (192, 64), (192, 128), (256, 64),
                            (256, 128), (256, 256)},
                  {2, 4, 6, 8}),
    ("C1", 0.7): (5120462, {(3, 64), (64, 3), (64, 64), (64, 96), (76, 96), (96, 76), (96, 96), (128, 64), (128, 153), (153, 64),
                            (153, 96), (153, 153), (160, 64), (160, 96), (192, 76), (192, 96)},
                  {2, 3, 4, 5, 6}),
    ("C3", 0.3): (63205897, {(3, 96), (89, 96), (96, 3), (96, 89), (96, 96), (96, 192), (128, 358), (179, 192), (192, 89), (192, 96),
                             (192, 179), (192, 192), (192, 384), (288, 96), (288, 179), (288, 192), (358, 96), (358, 192), (358, 358),
                             (358, 384), (384, 179), (384, 192), (384, 358), (384, 384), (576, 192), (576, 384), (768, 358), (768, 384)},
                  {3, 6, 9, 12, 18, 24}),
}


@pytest.mark.parametrize("family,ratio", SWEEP)
def test_pruned_network_widths_are_pinned(family, ratio):
    m = _built(family, ratio)
    n, io_ref, cpg_ref = PINNED[(family, ratio)]
    io, gn_w, cpg = widths(m)
    assert sum(p.numel() for p in m.parameters()) == n
    assert io == io_ref, sorted(io ^ io_ref)
    assert cpg == cpg_ref, sorted(cpg)
    for g in (mod for mod in m.modules() if isinstance(mod, nn.GroupNorm)):
        assert g.num_channels % g.num_groups == 0 and g.num_channels % 32 == 0, (g.num_channels, g.num_groups)


def test_sweep_covers_every_pitch_residue_and_the_odd_group_widths():
    """Across the sweep: a width that feeds no GroupNorm (attention inner dimension, time-embedding MLP) in each residue class 1 / 2 / 3
    mod 4 (pad columns of 3 / 2 / 1 floats in a pitch-4 buffer), and GroupNorm groups of 2, 3, 5, 7, 11, 14 and 18 channels, which the
    unpruned networks do not have.  The 0.5 network has no pad at all: the control."""
    residues, cpgs = set(), set()
    for fam, r in SWEEP:
        io, gn_w, cpg = widths(_built(fam, r))
        residues |= {w % 4 for pair in io for w in pair if w not in gn_w}
        cpgs |= cpg
    assert {1, 2, 3} <= residues, sorted(residues)
    assert {2, 3, 5, 7, 11, 14, 18} <= cpgs, sorted(cpgs)
    io, gn_w, _ = widths(_built("C1", 0.5))
    assert all(w % 4 == 0 for pair in io for w in pair if w != 3), sorted(io)      # only the 3-channel image ends are not 4-aligned


# ---------------------------------------------------------------------------------------------------------------------- poisoning
INT_POISON = 0xA5          # byte pattern of every integer allocation under poisoned_alloc


class _Count:
    n = 0


def _poison(t: torch.Tensor, value: float, count: _Count) -> torch.Tensor:
    if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():   # a fill inside a capture would be replayed
        return t
    if t.is_floating_point():
        v = value
        if math.isfinite(v) and abs(v) > torch.finfo(t.dtype).max:
            v = math.copysign(math.inf, v)           # 1e30 in an fp16 buffer: its largest magnitude beyond range
        t.fill_(v)
    else:
        t.untyped_storage().fill_(INT_POISON)
    count.n += 1
    return t


@contextlib.contextmanager
def poisoned_alloc(value: float):
    """Every tensor torch.empty / empty_like / empty_strided / Tensor.new_empty return inside the block comes back filled: floating
    tensors with `value`, integer tensors with the byte pattern INT_POISON; nothing is filled while the current stream captures a
    CUDA graph.  Yields a counter whose .n is the number of tensors poisoned.  Explicit zero_() calls after the allocation still run,
    so the poison reaches exactly the memory the code never initialised."""
    count = _Count()
    wrapped = {}
    for name in ("empty", "empty_like", "empty_strided"):
        fn = getattr(torch, name)
        wrapped[name] = fn
        setattr(torch, name, functools.wraps(fn)(lambda *a, _fn=fn, **k: _poison(_fn(*a, **k), value, count)))
    own = "new_empty" in torch.Tensor.__dict__
    new_empty = torch.Tensor.new_empty
    torch.Tensor.new_empty = lambda self, *a, **k: _poison(new_empty(self, *a, **k), value, count)
    try:
        yield count
    finally:
        for name, fn in wrapped.items():
            setattr(torch, name, fn)
        if own:
            torch.Tensor.new_empty = new_empty
        else:
            del torch.Tensor.new_empty


def test_poisoned_alloc_fills_counts_and_steps_aside_while_capturing():
    x = torch.zeros(3, 5)
    with poisoned_alloc(float("nan")) as c:
        floats = [torch.empty(7, 9), torch.empty_like(x), torch.empty_strided((4, 3), (1, 4)), x.new_empty((2, 6)),
                  torch.empty(5, dtype=torch.float16), torch.empty(5, dtype=torch.bfloat16)]
        ints = [torch.empty(11, dtype=torch.int32), torch.empty_like(x, dtype=torch.int64), torch.empty(3, dtype=torch.uint8)]
        assert c.n == len(floats) + len(ints)
        with mock.patch.object(torch.cuda, "is_available", return_value=True), \
                mock.patch.object(torch.cuda, "is_current_stream_capturing", return_value=True), \
                mock.patch.object(torch.Tensor, "fill_", side_effect=AssertionError("filled while capturing")):
            [torch.empty(64), torch.empty_like(x), torch.empty_strided((8,), (1,)), x.new_empty(9), torch.empty(2, dtype=torch.int32)]
        assert c.n == len(floats) + len(ints)                    # nothing counted while capturing
    assert all(bool(t.isnan().all()) for t in floats)
    for t in ints:
        assert bool((t.view(-1).view(torch.uint8) == INT_POISON).all()), t.dtype
    torch.empty(4), x.new_empty(4)
    assert c.n == len(floats) + len(ints) and "new_empty" not in torch.Tensor.__dict__    # unhooked after the block
    with poisoned_alloc(1e30) as c:
        a, h = torch.empty(4), torch.empty(4, dtype=torch.float16)
    assert bool((a == 1e30).all()) and bool((h == math.inf).all()) and c.n == 2
    with poisoned_alloc(0.0):
        assert bool((torch.empty(6, 6) == 0).all())
