"""Applying channel pruning to the module tree (host side, integer/index work).

Replaces the slicing done by torch_pruning's layer pruners — ddpm_exp/torch_pruning/pruner/function.py:85-146
(ConvPruner), :168-207 (LinearPruner), :274-302 (GroupNormPruner): keep-index selection on weight / bias and on the
accumulated ``.grad`` (so later groups of the same prune pass score the already-sliced tensors, exactly like the
reference's interactive loop ddpm_prune.py:108-109), plus the static-attribute fix of ddpm_prune.py:112-116.
Slicing runs on whatever device the parameters live on (torch.index_select on the GPU for the product path).
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Sequence, Tuple

import torch
import torch.nn as nn

from .models import Downsample2D, Upsample2D


def _keep(n: int, drop: Sequence[int], device) -> torch.Tensor:
    mask = torch.ones(n, dtype=torch.bool)
    mask[torch.as_tensor(sorted(set(int(i) for i in drop)), dtype=torch.long)] = False
    return torch.nonzero(mask).flatten().to(device)


def _slice_param(p: nn.Parameter, keep: torch.Tensor, dim: int) -> nn.Parameter:
    new = nn.Parameter(torch.index_select(p.data, dim, keep).contiguous(), requires_grad=p.requires_grad)
    if p.grad is not None:
        new.grad = torch.index_select(p.grad, dim, keep).contiguous()
    return new


def prune_out_channels(layer: nn.Module, drop: Sequence[int]) -> None:
    """Conv2d / Linear output channels or GroupNorm channels (function.py:88-105, 171-185, 277-294)."""
    if isinstance(layer, nn.GroupNorm):
        keep = _keep(layer.num_channels, drop, layer.weight.device)
        layer.num_channels = int(keep.numel())          # num_groups is NOT touched (function.py:274-294)
        layer.weight = _slice_param(layer.weight, keep, 0)
        layer.bias = _slice_param(layer.bias, keep, 0)
        return
    n = layer.weight.shape[0]
    keep = _keep(n, drop, layer.weight.device)
    layer.weight = _slice_param(layer.weight, keep, 0)
    if layer.bias is not None:
        layer.bias = _slice_param(layer.bias, keep, 0)
    if isinstance(layer, nn.Conv2d):
        layer.out_channels = int(keep.numel())
    else:
        layer.out_features = int(keep.numel())


def prune_in_channels(layer: nn.Module, drop: Sequence[int]) -> None:
    """Conv2d / Linear input channels (function.py:107-126, 187-199); bias untouched."""
    n = layer.weight.shape[1]
    keep = _keep(n, drop, layer.weight.device)
    layer.weight = _slice_param(layer.weight, keep, 1)
    if isinstance(layer, nn.Conv2d):
        layer.in_channels = int(keep.numel())
    else:
        layer.in_features = int(keep.numel())


def apply_group(modules: Dict[str, nn.Module], items: Iterable[Tuple[str, str, Sequence[int]]], selected: Sequence[int],
                channels: int) -> None:
    """Prune one group: `items` are (layer_name, kind in {out,in,gn}, full index list) where index lists map the root's
    channels positionally (a layer fed by both halves of a concat carries the two maps merged: len = parts*channels);
    `selected` are root-channel positions to remove."""
    for name, kind, idxs in items:
        idxs = list(idxs)
        parts = len(idxs) // channels
        assert parts * channels == len(idxs), (name, len(idxs), channels)
        drop = [idxs[q * channels + j] for q in range(parts) for j in selected]
        layer = modules[name]
        if kind == "in":
            prune_in_channels(layer, drop)
        else:
            prune_out_channels(layer, drop)


def fix_static_attributes(model: nn.Module) -> None:
    """ddpm_prune.py:112-116."""
    for m in model.modules():
        if isinstance(m, (Upsample2D, Downsample2D)):
            m.channels = m.conv.in_channels
            m.out_channels = m.conv.out_channels


# ==============================================================================================================
# Structural pruning groups of UNet2DModel (what torch_pruning's DependencyGraph derives by tracing — dependency.py:295-527 —
# obtained here directly from the architecture).  A "space" is a set of channel dimensions that must be pruned together:
#   residual stream   conv_in / conv_shortcut / downsampler outputs, every conv2 / to_out.0 added onto it, and all consumers
#                     (norm1 gamma, conv1 / conv_shortcut / downsampler / to_q,k,v inputs — through concat offsets on the up path)
#   block interior    conv1 out + time_emb_proj out + norm2 gamma + conv2 in
#   attention inner   to_q / to_k / to_v out + to_out.0 in
#   time embedding    linear_1 out + linear_2 in ;  linear_2 out + every time_emb_proj in
# Group order = order in which named_modules() first meets a producer of the space (dependency.py:498-527), because the
# reference scores groups interactively on already-sliced layers.
# ==============================================================================================================
class _Spaces:
    def __init__(self):
        self.parent: List[int] = []
        self.members: Dict[int, list] = {}

    def new(self) -> int:
        self.parent.append(len(self.parent))
        self.members[len(self.parent) - 1] = []
        return len(self.parent) - 1

    def find(self, a: int) -> int:
        while self.parent[a] != a:
            self.parent[a] = self.parent[self.parent[a]]
            a = self.parent[a]
        return a

    def union(self, a: int, b: int) -> int:
        a, b = self.find(a), self.find(b)
        if a != b:
            self.parent[b] = a
            self.members[a] += self.members.pop(b)
        return a

    def add(self, space, item):
        if space is not None:
            self.members[self.find(space)].append(item)


def traced_module_order(model) -> List[str]:
    """Order in which the reference's tracer inserts modules into its module2node table (dependency.py:631-705 hooks +
    :707-811 stack walk over out.grad_fn.next_functions, LIFO): one batch-1 trace-mode forward, forward hooks map
    grad_fn -> leaf module, then the same non-recursive walk.  Group order and group roots follow from it
    (dependency.py:498-527), and because groups are scored interactively the order is part of the result."""
    from .models import trace_mode
    leaves = {m: n for n, m in model.named_modules() if isinstance(m, (nn.Conv2d, nn.Linear, nn.GroupNorm))}
    fn2mod = {}
    hooks = [m.register_forward_hook(lambda mod, i, o: fn2mod.__setitem__(o.grad_fn, mod)) for m in leaves]
    cfg = model.config
    p0 = next(model.parameters())
    was_training = model.training
    model.eval()
    with torch.enable_grad(), trace_mode():
        if _is_ddim_model(model):       # prune.py:190: example_inputs {'x': randn(1, 3, S, S), 't': torch.ones(1)}
            # the trace input comes from a generator of its own: the reference's tracer draws nothing, and RandomImportance's draws
            # later in prune.py must see the global generator where the reference leaves it
            size = cfg.data.image_size
            x = torch.randn(1, model.in_channels, size, size, generator=torch.Generator().manual_seed(0)).to(p0.device)
            out = model(x, torch.ones(1, device=p0.device))
        else:
            size = cfg.sample_size if isinstance(cfg.sample_size, int) else 32
            out = model(torch.randn(1, cfg.in_channels, size, size, device=p0.device),
                        torch.ones(1, dtype=torch.long, device=p0.device)).sample
    for h in hooks:
        h.remove()
    model.train(was_training)
    order, seen_mod, visited = [], set(), set()

    def touch(fn):
        mod = fn2mod.get(fn)
        if mod is not None and mod not in seen_mod:
            seen_mod.add(mod)
            order.append(leaves[mod])

    stack = [out.grad_fn]
    while stack:
        fn = stack.pop()
        if fn in visited:
            continue
        touch(fn)
        for nxt, _ in getattr(fn, "next_functions", ()):
            if nxt is None or "accumulategrad" in nxt.name().lower():
                continue
            touch(nxt)
            stack.append(nxt)
        visited.add(fn)
    return order


def _is_ddim_model(model) -> bool:
    """ddpm_exp's DDIM-codebase Model (ddpm_exp.py), which the planner recognises the same way."""
    return hasattr(model, "temb") and hasattr(model, "mid")


def build_groups(model, ignored_layers: Sequence[nn.Module] = (), module_order: Sequence[str] = None) -> List[dict]:
    """Current pruning groups of a UNet2DModel or of ddpm_exp's Model: [{root, ch_groups, channels, items: [(layer_name, kind, idxs)]}]
    in the reference's group order.  `idxs` map the root's channel positions to each member's own indices (concat offsets);
    a member fed twice by the same space carries the merged map (len = 2*channels) like the reference."""
    from types import SimpleNamespace as NS
    from .models import UNet2DModel
    ddim = _is_ddim_model(model)
    assert ddim or isinstance(model, UNet2DModel)
    names = {m: n for n, m in model.named_modules()}
    if module_order is None:
        module_order = traced_module_order(model)
    order = {n: i for i, n in enumerate(module_order)}
    sp = _Spaces()
    ignored = {id(m) for m in ignored_layers}

    def produce(layer, space=None):       # layer's out-channels join `space` (or open a new one)
        s = sp.new() if space is None else space
        sp.add(s, ("out", layer, 0, layer.weight.shape[0]))
        return s

    def consume(layer, segs, kind="in"):  # layer's in-channels (or GN channels) read the concatenated segments
        off = 0
        for s, n in segs:
            sp.add(s, (kind, layer, off, n))
            off += n

    def resnet(m, segs, temb_space):        # ResnetBlock2D, or a ddpm_exp ResnetBlock in its attribute vocabulary
        consume(m.norm1, segs, "gn")
        consume(m.conv1, segs)
        a = produce(m.conv1)
        consume(m.time_emb_proj, [(temb_space, m.time_emb_proj.in_features)])
        produce(m.time_emb_proj, a)
        consume(m.norm2, [(a, m.conv1.out_channels)], "gn")
        consume(m.conv2, [(a, m.conv1.out_channels)])
        if m.conv_shortcut is not None:
            consume(m.conv_shortcut, segs)
            b = produce(m.conv_shortcut)
            produce(m.conv2, b)
        else:
            assert len(segs) == 1
            b = produce(m.conv2, segs[0][0])
        return [(b, m.conv2.out_channels)]

    def attention(m, segs):                 # Attention, or a ddpm_exp AttnBlock (1x1 convolutions) in its attribute vocabulary
        assert len(segs) == 1
        s, n = segs[0]
        consume(m.group_norm, segs, "gn")
        for lin in (m.to_q, m.to_k, m.to_v):
            consume(lin, segs)
        v = produce(m.to_q)
        produce(m.to_k, v)
        produce(m.to_v, v)
        consume(m.to_out[0], [(v, m.to_q.weight.shape[0])])
        produce(m.to_out[0], s)
        return segs

    if ddim:
        _ddim_spaces(model, produce, consume, resnet, attention, NS)
    else:
        _unet2d_spaces(model, produce, consume, resnet, attention)
    sp.add(sp.new(), ("out", model.conv_out, 0, model.conv_out.out_channels))
    return _groups_of(sp, names, order, ignored)


def _unet2d_spaces(model, produce, consume, resnet, attention):
    te = model.time_embedding
    t1 = produce(te.linear_1)
    consume(te.linear_2, [(t1, te.linear_1.out_features)])
    t2 = produce(te.linear_2)
    x = [(produce(model.conv_in), model.conv_in.out_channels)]
    skips = [x]
    for blk in model.down_blocks:
        for j, r in enumerate(blk.resnets):
            x = resnet(r, x, t2)
            if getattr(blk, "has_attention", False):
                x = attention(blk.attentions[j], x)
            skips.append(x)
        if blk.downsamplers is not None:
            conv = blk.downsamplers[0].conv
            consume(conv, x)
            x = [(produce(conv), conv.out_channels)]
            skips.append(x)
    mb = model.mid_block
    x = resnet(mb.resnets[0], x, t2)
    if mb.attentions[0] is not None:
        x = attention(mb.attentions[0], x)
    x = resnet(mb.resnets[1], x, t2)
    for blk in model.up_blocks:
        for j, r in enumerate(blk.resnets):
            x = resnet(r, x + skips.pop(), t2)
            if getattr(blk, "has_attention", False):
                x = attention(blk.attentions[j], x)
        if blk.upsamplers is not None:
            conv = blk.upsamplers[0].conv
            consume(conv, x)
            x = [(produce(conv), conv.out_channels)]
    consume(model.conv_norm_out, x, "gn")
    consume(model.conv_out, x)


def _ddim_spaces(model, produce, consume, resnet, attention, NS):
    """Model.forward (ddpm_exp models/diffusion.py:268-300): temb.dense, conv_in, the down levels with their hs entries, mid, the up levels
    over torch.cat([h, hs.pop()]), norm_out and conv_out.  A ResnetBlock applies nin_shortcut when it was built with in_channels !=
    out_channels; q / k / v / proj_out are 1x1 convolutions."""
    def rb(m, segs, t):
        return resnet(NS(norm1=m.norm1, conv1=m.conv1, time_emb_proj=m.temb_proj, norm2=m.norm2, conv2=m.conv2,
                         conv_shortcut=m.nin_shortcut if m.in_channels != m.out_channels else None), segs, t)

    def ab(m, segs):
        return attention(NS(group_norm=m.norm, to_q=m.q, to_k=m.k, to_v=m.v, to_out=[m.proj_out]), segs)
    d0, d1 = model.temb.dense
    t1 = produce(d0)
    consume(d1, [(t1, d0.out_features)])
    t2 = produce(d1)
    x = [(produce(model.conv_in), model.conv_in.out_channels)]
    hs = [x]
    for lvl in model.down:
        for i, m in enumerate(lvl.block):
            x = rb(m, x, t2)
            if len(lvl.attn) > 0:
                x = ab(lvl.attn[i], x)
            hs.append(x)
        if hasattr(lvl, "downsample"):
            conv = lvl.downsample.conv
            consume(conv, x)
            x = [(produce(conv), conv.out_channels)]
            hs.append(x)
    x = rb(model.mid.block_2, ab(model.mid.attn_1, rb(model.mid.block_1, x, t2)), t2)
    for i_level in reversed(range(len(model.up))):
        lvl = model.up[i_level]
        for i, m in enumerate(lvl.block):
            x = rb(m, x + hs.pop(), t2)
            if len(lvl.attn) > 0:
                x = ab(lvl.attn[i], x)
        if hasattr(lvl, "upsample"):
            conv = lvl.upsample.conv
            consume(conv, x)
            x = [(produce(conv), conv.out_channels)]
    consume(model.norm_out, x, "gn")
    consume(model.conv_out, x)


def _groups_of(sp, names, order, ignored) -> List[dict]:
    groups = []
    for root_space, members in sp.members.items():
        prods = [mem for mem in members if mem[0] == "out"]
        if not prods or any(id(mem[1]) in ignored for mem in prods):
            continue
        root = min(prods, key=lambda mem: order[names[mem[1]]])
        channels = root[3]
        merged: Dict[Tuple[str, str], List[int]] = {}
        seq: List[Tuple[str, str]] = []
        for kind, layer, off, n in members:
            assert n == channels, (names[layer], kind, n, channels)
            key = (names[layer], kind)
            if key not in merged:
                merged[key] = []
                seq.append(key)
            merged[key] += list(range(off, off + n))
        gn = [layer for kind, layer, _, _ in members if kind == "gn"]
        groups.append({"root": names[root[1]], "channels": channels, "ch_groups": gn[0].num_groups if gn else 1,
                       "items": [(n, k, merged[(n, k)]) for (n, k) in seq], "_order": order[names[root[1]]]})
    groups.sort(key=lambda g: g["_order"])
    return groups


def group_of_root(model, root: str, ignored_layers: Sequence[nn.Module] = (), module_order: Sequence[str] = None):
    """The CURRENT group rooted at `root` (the reference re-derives every group from the live graph right before it is pruned,
    metapruner.py:208), or None when it must be skipped: the reference's `_check_sparsity` (metapruner.py:172-194) refuses a group
    one of whose members is down to a single channel."""
    for g in build_groups(model, ignored_layers, module_order):
        if g["root"] == root:
            mods = dict(model.named_modules())
            for name, kind, _ in g["items"]:
                w = mods[name].weight
                if (w.shape[1] if kind == "in" else w.shape[0]) == 1:
                    return None
            return g
    raise KeyError(f"diff_pruning_b200: pruning group rooted at {root!r} no longer exists in the model (was the module tree edited "
                   "between MagnitudePruner(...) and step()?)")


def taylor_prune(model, ratio: float, variant: str = "taylor", ignored_layers: Sequence[nn.Module] = (), round_to=None) -> List[dict]:
    """ddpm_prune.py:79-116 without torch_pruning: for each group in the reference's order, score it ON DEVICE from the
    accumulated Parameter.grad (dp_taylor_reduce), select the lowest-importance channels (metapruner.py:225-249), slice
    weights + grads, go on to the next group (which therefore sees the sliced layers — the interactive semantics of the
    reference), finally fix the static attributes.  Returns the per-group record (root, importance, pruned positions)."""
    from .scoring import group_importance, select_pruning_idxs
    morder = traced_module_order(model)
    init = {g["root"]: g["channels"] for g in build_groups(model, ignored_layers, morder)}
    record = []
    for root in list(init):
        g = group_of_root(model, root, ignored_layers, morder)
        if g is None:
            continue
        mods = dict(model.named_modules())
        n_pruned = g["channels"] - int(init[root] * (1 - ratio))
        if round_to:
            n_pruned -= n_pruned % round_to
        if n_pruned <= 0:
            continue
        named_w = {n + ".weight": mods[n].weight for n, _, _ in g["items"]}
        named_g = {n + ".weight": mods[n].weight.grad for n, _, _ in g["items"]}
        imp = group_importance(g["items"], named_w, named_g, variant)
        sel = select_pruning_idxs(imp, g["ch_groups"], n_pruned)
        apply_group(mods, g["items"], sel, g["channels"])
        record.append({"root": root, "imp": imp, "idxs": sel, "channels": g["channels"], "ch_groups": g["ch_groups"]})
    fix_static_attributes(model)
    return record
