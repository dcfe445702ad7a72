"""`import torch_pruning as tp` surface used by ddpm_prune.py:41-118, on diff_pruning_b200.pruning / scoring.

tp.importance.TaylorImportance(multivariable=True|False)   ddpm_prune.py:60,66   (device-side dp_taylor_reduce)
tp.importance.MagnitudeImportance / RandomImportance       ddpm_prune.py:62,64
tp.pruner.MagnitudePruner(model, example_inputs, importance=, iterative_steps=, channel_groups=, ch_sparsity=, ignored_layers=)
    .step(interactive=True) -> iterable of groups with .prune()                 ddpm_prune.py:79-87,108-109
tp.utils.count_ops_and_params(model, example_inputs)                            ddpm_prune.py:89,118
"""
from types import SimpleNamespace

import torch
import torch.nn as nn

from diff_pruning_b200 import pruning as _pr
from diff_pruning_b200 import scoring as _sc
from diff_pruning_b200.models import trace_mode as _trace_mode


class _Importance:
    variant = None

    def __call__(self, group, ch_groups=1):
        raise NotImplementedError


class TaylorImportance(_Importance):
    def __init__(self, group_reduction="mean", normalizer="mean", multivariable=False, variant=None):
        # multivariable=True: |sum_k w dw| ("taylor"); False: sum_k |w dw| ("diff-pruning"); variant="vendored": sum (w dw)^2
        self.variant = variant or ("taylor" if multivariable else "diff")

    def __call__(self, group, ch_groups=1):
        mods = group.modules
        named_w = {n + ".weight": mods[n].weight for n, _, _ in group.items}
        named_g = {n + ".weight": mods[n].weight.grad for n, _, _ in group.items}
        return _sc.group_importance(group.items, named_w, named_g, self.variant)


class FullTaylorImportance(TaylorImportance):
    """ddpm_exp/torch_pruning/importance.py:438-548 (order 1 or 2)."""

    def __init__(self, order=1, group_reduction="mean", normalizer="mean"):
        if order not in (1, 2):
            raise NotImplementedError(order)
        self.variant = f"full{order}"


class AbsTaylorImportance(TaylorImportance):
    """ddpm_exp/torch_pruning/importance.py:553-670 (the per-layer criterion; its accum_abs_grad helper is an experiment-side loop)."""

    def __init__(self, order=1, group_reduction="mean", normalizer="mean"):
        self.variant = "abs"


class FisherImportance(TaylorImportance):
    """ddpm_exp/torch_pruning/importance.py:672-781."""

    def __init__(self, group_reduction="mean", normalizer="mean"):
        self.variant = "fisher"


class MagnitudeImportance(_Importance):
    """L2 norm of the weights per channel, summed over the group's equally-sized members (importance.py:18-126, p=2)."""

    def __init__(self, p=2, **unused):
        self.p = p

    def __call__(self, group, ch_groups=1):
        imps = []
        for name, kind, idxs in group.items:
            w = group.modules[name].weight.detach()
            idx = torch.as_tensor(sorted(idxs), device=w.device)
            if kind == "gn":
                continue
            v = (w.flatten(1) if kind == "out" else w.transpose(0, 1).flatten(1))[idx].abs().pow(self.p).sum(1)
            imps.append(v)
        size = len(imps[0])
        return torch.stack([i for i in imps if len(i) == size]).sum(0)


class RandomImportance(_Importance):
    def __call__(self, group, ch_groups=1):
        return torch.rand(group.channels)


importance = SimpleNamespace(TaylorImportance=TaylorImportance, MagnitudeImportance=MagnitudeImportance,
                             RandomImportance=RandomImportance, Importance=_Importance, FullTaylorImportance=FullTaylorImportance,
                             AbsTaylorImportance=AbsTaylorImportance, FisherImportance=FisherImportance)


class _Group:
    def __init__(self, model, g, idxs):
        self.modules = dict(model.named_modules())
        self.items, self.channels, self.root, self.idxs = g["items"], g["channels"], g["root"], idxs

    def prune(self):
        _pr.apply_group(self.modules, self.items, self.idxs, self.channels)


class MagnitudePruner:
    """metapruner.py:20-254 (local pruning, one iterative step) over the structural UNet groups."""

    def __init__(self, model, example_inputs=None, importance=None, iterative_steps=1, channel_groups=None, ch_sparsity=0.5,
                 ignored_layers=None, round_to=None, **unused):
        self.model, self.importance, self.ch_sparsity, self.round_to = model, importance, ch_sparsity, round_to
        self.ignored_layers = list(ignored_layers or [])
        self._order = _pr.traced_module_order(model)
        self._init = {g["root"]: g["channels"] for g in _pr.build_groups(model, self.ignored_layers, self._order)}

    def step(self, interactive=False):
        def gen():
            for root in list(self._init):
                g = _pr.group_of_root(self.model, root, self.ignored_layers, self._order)
                if g is None:
                    continue
                n_pruned = g["channels"] - int(self._init[root] * (1 - self.ch_sparsity))
                if self.round_to:
                    n_pruned -= n_pruned % self.round_to
                if n_pruned <= 0:
                    continue
                grp = _Group(self.model, g, [])
                imp = self.importance(grp, ch_groups=g["ch_groups"])
                if imp is None:
                    continue
                grp.idxs = _sc.select_pruning_idxs(imp, g["ch_groups"], n_pruned)
                grp.imp, grp.ch_groups, grp.n_pruned = imp, g["ch_groups"], n_pruned     # what the selection was made from
                yield grp
        if interactive:
            return gen()
        for grp in gen():
            grp.prune()


pruner = SimpleNamespace(MagnitudePruner=MagnitudePruner, MetaPruner=MagnitudePruner)


def count_ops_and_params(model, example_inputs):
    """The reference counter's conventions (utils/op_counter.py:53-110,250-284): Conv2d = k*k*Cin*Cout/groups per output
    position + one bias add per output element, Linear = in*out per row + out, GroupNorm = 2 per element (affine);
    attention bmm / softmax are not counted there either.  One hooked trace-mode forward at the example batch."""
    ops = [0]

    def hook(mod, inp, out):
        x = inp[0]
        if isinstance(mod, nn.Conv2d):
            pos = out.shape[0] * out.shape[2] * out.shape[3]
            ops[0] += pos * mod.kernel_size[0] * mod.kernel_size[1] * mod.in_channels * (mod.out_channels // mod.groups)
            ops[0] += pos * mod.out_channels if mod.bias is not None else 0
        elif isinstance(mod, nn.Linear):
            ops[0] += x.numel() * out.shape[-1] + (out.shape[-1] if mod.bias is not None else 0)
        elif isinstance(mod, nn.GroupNorm):
            ops[0] += x.numel() * (2 if mod.affine else 1)
    hs = [m.register_forward_hook(hook) for m in model.modules() if isinstance(m, (nn.Conv2d, nn.Linear, nn.GroupNorm))]
    with torch.no_grad(), _trace_mode():
        model(**example_inputs) if isinstance(example_inputs, dict) else model(*example_inputs)
    for h in hs:
        h.remove()
    return float(ops[0]), float(sum(p.numel() for p in model.parameters()))


utils = SimpleNamespace(count_ops_and_params=count_ops_and_params)
