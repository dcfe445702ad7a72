"""FID evaluation on the device: the Inception-v3 feature pass of the reference's fid_score.py / inception.py (pytorch-fid), fp64 feature
moments on the GPU, and the Fréchet distance on the host.

InceptionV3      the reference wrapper's module tree (`blocks.*` state-dict keys, BLOCK_INDEX_BY_DIM, output_blocks / resize_input /
                 normalize_input); loads the pytorch-fid weight file (torchvision names, `fc.*` ignored).  Its forward runs the device plan.
FeaturePlan      forward-only launch list for one batch size and input format: BatchNorm folded into the convolutions on the host (fp64,
                 rounded once), every buffer allocated up front, branches writing their channel range of the concatenated output, the
                 whole pass replayed as one CUDA graph.  Convolutions run with the ReLU epilogue (DP_CONV_RELU) on the exact-fp32 kernel.
get_activations / calculate_activation_statistics / compute_statistics_of_path / calculate_frechet_distance / calculate_fid_given_paths /
save_fid_stats   fid_score.py's functions; statistics come from device moments (dp_feature_moments), so the [n, dims] activation matrix
                 never has to reach the host.
statistics_of_pipeline   FID statistics of DDIMPipeline samples straight from device memory, bit-identical to writing the PNGs first.

The weight file is never downloaded: pass a path, set DPB200_FID_WEIGHTS, or place it in torch.hub's checkpoint directory."""
from __future__ import annotations

import ctypes
import gc
import os
import pathlib
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import _lib as L
from .engine import View, _stream, capture_graphs

WEIGHTS_FILE = "pt_inception-2015-12-05-6726825d.pth"
WEIGHTS_ENV = "DPB200_FID_WEIGHTS"
IMAGE_EXTENSIONS = {"bmp", "jpg", "jpeg", "pgm", "png", "ppm", "tif", "tiff", "webp"}
BN_EPS = 0.001
DP_CONV_FORCE_SIMT, DP_CONV_RELU, DP_CONV_ANY_GEOMETRY = 2, 4, 8

# ------------------------------------------------------------------------------------------------ architecture
# A convolution: (name, source, out channels, (kh, kw), stride, (pad_h, pad_w)); source "x" is the block input, "pool" the block's pool.
# torchvision's inception_v3 with the FID patches of inception.py:224-341 (average pools that do not count padding; max pool in E_2).
def _a(pf):
    return dict(pool=("avg", 1, 1), convs=[
        ("branch1x1", "x", 64, (1, 1), 1, (0, 0)),
        ("branch5x5_1", "x", 48, (1, 1), 1, (0, 0)), ("branch5x5_2", "branch5x5_1", 64, (5, 5), 1, (2, 2)),
        ("branch3x3dbl_1", "x", 64, (1, 1), 1, (0, 0)), ("branch3x3dbl_2", "branch3x3dbl_1", 96, (3, 3), 1, (1, 1)),
        ("branch3x3dbl_3", "branch3x3dbl_2", 96, (3, 3), 1, (1, 1)),
        ("branch_pool", "pool", pf, (1, 1), 1, (0, 0))],
        out=["branch1x1", "branch5x5_2", "branch3x3dbl_3", "branch_pool"])


_B = dict(pool=("max", 2, 0), convs=[
    ("branch3x3", "x", 384, (3, 3), 2, (0, 0)),
    ("branch3x3dbl_1", "x", 64, (1, 1), 1, (0, 0)), ("branch3x3dbl_2", "branch3x3dbl_1", 96, (3, 3), 1, (1, 1)),
    ("branch3x3dbl_3", "branch3x3dbl_2", 96, (3, 3), 2, (0, 0))],
    out=["branch3x3", "branch3x3dbl_3", "pool"])


def _c(c7):
    return dict(pool=("avg", 1, 1), convs=[
        ("branch1x1", "x", 192, (1, 1), 1, (0, 0)),
        ("branch7x7_1", "x", c7, (1, 1), 1, (0, 0)), ("branch7x7_2", "branch7x7_1", c7, (1, 7), 1, (0, 3)),
        ("branch7x7_3", "branch7x7_2", 192, (7, 1), 1, (3, 0)),
        ("branch7x7dbl_1", "x", c7, (1, 1), 1, (0, 0)), ("branch7x7dbl_2", "branch7x7dbl_1", c7, (7, 1), 1, (3, 0)),
        ("branch7x7dbl_3", "branch7x7dbl_2", c7, (1, 7), 1, (0, 3)), ("branch7x7dbl_4", "branch7x7dbl_3", c7, (7, 1), 1, (3, 0)),
        ("branch7x7dbl_5", "branch7x7dbl_4", 192, (1, 7), 1, (0, 3)),
        ("branch_pool", "pool", 192, (1, 1), 1, (0, 0))],
        out=["branch1x1", "branch7x7_3", "branch7x7dbl_5", "branch_pool"])


_D = dict(pool=("max", 2, 0), convs=[
    ("branch3x3_1", "x", 192, (1, 1), 1, (0, 0)), ("branch3x3_2", "branch3x3_1", 320, (3, 3), 2, (0, 0)),
    ("branch7x7x3_1", "x", 192, (1, 1), 1, (0, 0)), ("branch7x7x3_2", "branch7x7x3_1", 192, (1, 7), 1, (0, 3)),
    ("branch7x7x3_3", "branch7x7x3_2", 192, (7, 1), 1, (3, 0)), ("branch7x7x3_4", "branch7x7x3_3", 192, (3, 3), 2, (0, 0))],
    out=["branch3x3_2", "branch7x7x3_4", "pool"])


def _e(pool_kind):
    return dict(pool=(pool_kind, 1, 1), convs=[
        ("branch1x1", "x", 320, (1, 1), 1, (0, 0)),
        ("branch3x3_1", "x", 384, (1, 1), 1, (0, 0)), ("branch3x3_2a", "branch3x3_1", 384, (1, 3), 1, (0, 1)),
        ("branch3x3_2b", "branch3x3_1", 384, (3, 1), 1, (1, 0)),
        ("branch3x3dbl_1", "x", 448, (1, 1), 1, (0, 0)), ("branch3x3dbl_2", "branch3x3dbl_1", 384, (3, 3), 1, (1, 1)),
        ("branch3x3dbl_3a", "branch3x3dbl_2", 384, (1, 3), 1, (0, 1)), ("branch3x3dbl_3b", "branch3x3dbl_2", 384, (3, 1), 1, (1, 0)),
        ("branch_pool", "pool", 192, (1, 1), 1, (0, 0))],
        out=["branch1x1", "branch3x3_2a", "branch3x3_2b", "branch3x3dbl_3a", "branch3x3dbl_3b", "branch_pool"])


# (torchvision name, wrapper key, layer): a layer is ("conv", cin, cout, k, stride, pad), ("maxpool",) or ("mixed", cin, spec)
LAYERS = [
    ("Conv2d_1a_3x3", "0.0", ("conv", 3, 32, (3, 3), 2, (0, 0))),
    ("Conv2d_2a_3x3", "0.1", ("conv", 32, 32, (3, 3), 1, (0, 0))),
    ("Conv2d_2b_3x3", "0.2", ("conv", 32, 64, (3, 3), 1, (1, 1))),
    (None, "0.3", ("maxpool",)),
    ("Conv2d_3b_1x1", "1.0", ("conv", 64, 80, (1, 1), 1, (0, 0))),
    ("Conv2d_4a_3x3", "1.1", ("conv", 80, 192, (3, 3), 1, (0, 0))),
    (None, "1.2", ("maxpool",)),
    ("Mixed_5b", "2.0", ("mixed", 192, _a(32))),
    ("Mixed_5c", "2.1", ("mixed", 256, _a(64))),
    ("Mixed_5d", "2.2", ("mixed", 288, _a(64))),
    ("Mixed_6a", "2.3", ("mixed", 288, _B)),
    ("Mixed_6b", "2.4", ("mixed", 768, _c(128))),
    ("Mixed_6c", "2.5", ("mixed", 768, _c(160))),
    ("Mixed_6d", "2.6", ("mixed", 768, _c(160))),
    ("Mixed_6e", "2.7", ("mixed", 768, _c(192))),
    ("Mixed_7a", "3.0", ("mixed", 768, _D)),
    ("Mixed_7b", "3.1", ("mixed", 1280, _e("avg"))),
    ("Mixed_7c", "3.2", ("mixed", 2048, _e("max"))),
    (None, "3.3", ("avgpool",)),
]


class BasicConv2d(nn.Module):
    """Conv2d without bias + eval BatchNorm2d(eps=0.001) + ReLU: the parameter container of one convolution."""

    def __init__(self, cin, cout, kernel_size, stride=1, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, kernel_size, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(cout, eps=BN_EPS)


class Mixed(nn.Module):
    def __init__(self, cin, spec):
        super().__init__()
        self.spec, self.cin = spec, cin
        width = {"x": cin, "pool": cin}
        for name, src, cout, k, s, p in spec["convs"]:
            self.add_module(name, BasicConv2d(width[src], cout, k, s, p))
            width[name] = cout


def _module(layer):
    if layer[0] == "conv":
        return BasicConv2d(*layer[1:])
    if layer[0] == "maxpool":
        return nn.MaxPool2d(kernel_size=3, stride=2)
    if layer[0] == "avgpool":
        return nn.AdaptiveAvgPool2d((1, 1))
    return Mixed(layer[1], layer[2])


def find_weights(path: Optional[str] = None) -> str:
    """The pytorch-fid weight file: `path`, else $DPB200_FID_WEIGHTS, else torch.hub.get_dir()/checkpoints/<file> (where the reference's
    load_state_dict_from_url caches it).  Nothing is downloaded."""
    tried = []
    for cand in (path, os.environ.get(WEIGHTS_ENV) or None, os.path.join(torch.hub.get_dir(), "checkpoints", WEIGHTS_FILE)):
        if cand is None:
            continue
        if os.path.isfile(cand):
            return cand
        tried.append(cand)
    raise FileNotFoundError(
        f"Inception weights {WEIGHTS_FILE} not found (looked at: {', '.join(tried)}). This package never downloads them: place the "
        f"file from pytorch-fid's release 'fid_weights' at one of those paths, pass its path, or set {WEIGHTS_ENV}.")


def convert_torchvision_state_dict(sd: Dict[str, torch.Tensor], last_block: int = 3) -> Dict[str, torch.Tensor]:
    """torchvision / pytorch-fid names (Conv2d_1a_3x3.conv.weight, Mixed_5b.branch1x1.bn.running_mean, fc.*, ...) -> wrapper keys
    (blocks.0.0.conv.weight, blocks.2.0.branch1x1.bn.running_mean, ...) for blocks 0..last_block; `fc.*` and
    `num_batches_tracked` are dropped."""
    prefix = {tv: "blocks." + key for tv, key, _ in LAYERS if tv is not None and int(key[0]) <= last_block}
    out = {}
    for k, v in sd.items():
        head, _, rest = k.partition(".")
        if head in prefix and not k.endswith("num_batches_tracked"):
            out[prefix[head] + "." + rest] = v
    return out


class InceptionV3(nn.Module):
    """inception.py's InceptionV3 (FID variant): same constructor, BLOCK_INDEX_BY_DIM and state-dict keys.  `weights` may be a
    state dict (torchvision or wrapper names), a path, or None (the weight file lookup of find_weights); weights=False leaves the
    parameters at their initial values (for loading a state dict afterwards)."""

    DEFAULT_BLOCK_INDEX = 3
    BLOCK_INDEX_BY_DIM = {64: 0, 192: 1, 768: 2, 2048: 3}

    def __init__(self, output_blocks=(DEFAULT_BLOCK_INDEX,), resize_input=True, normalize_input=True, requires_grad=False,
                 use_fid_inception=True, weights=None):
        super().__init__()
        if not use_fid_inception:
            raise NotImplementedError("only the FID Inception (use_fid_inception=True) is implemented")
        self.resize_input, self.normalize_input = resize_input, normalize_input
        self.output_blocks = sorted(output_blocks)
        self.last_needed_block = max(output_blocks)
        assert self.last_needed_block <= 3, "Last possible output block index is 3"
        self.blocks = nn.ModuleList()
        for b in range(self.last_needed_block + 1):
            self.blocks.append(nn.Sequential(*[_module(layer) for _, key, layer in LAYERS if int(key[0]) == b]))
        if weights is not False:
            if weights is None or isinstance(weights, (str, os.PathLike)):
                weights = torch.load(find_weights(weights), map_location="cpu", weights_only=True)
            self.load_weights(weights)
        for p in self.parameters():
            p.requires_grad = requires_grad
        self.eval()
        self._plan: Optional["FeaturePlan"] = None

    def load_weights(self, sd: Dict[str, torch.Tensor]):
        if not any(k.startswith("blocks.") for k in sd):
            sd = convert_torchvision_state_dict(sd, self.last_needed_block)
        sd = {k: v for k, v in sd.items() if not k.endswith("num_batches_tracked")}
        self.load_state_dict(sd, strict=False)
        missing = [k for k in self.state_dict() if not k.endswith("num_batches_tracked") and k not in sd]
        if missing:
            raise KeyError(f"Inception state dict lacks {len(missing)} tensors, e.g. {missing[:3]}")

    def plan(self, batch: int, src: str, hw, quantize: bool = False) -> "FeaturePlan":
        """The feature plan for this batch size and input format.  Only the most recent plan is kept (one at batch 256 holds several GB
        of activations): a different request frees it before the new one is built."""
        key = (batch, src, tuple(int(v) for v in hw), bool(quantize))
        if self._plan is None or self._plan.key != key:
            if self._plan is not None:
                self._plan = None
                gc.collect()          # the launch list refers back to its plan
            self._plan = FeaturePlan(self, batch, src, hw, quantize)
        return self._plan

    @torch.no_grad()
    def forward(self, inp: torch.Tensor) -> List[torch.Tensor]:
        """inception.py:129-163 on the device: inp [N, 3, H, W] fp32 in [0, 1] (CUDA); returns the selected block outputs as NCHW
        tensors (block 3: [N, 2048, 1, 1])."""
        if not inp.is_cuda:
            raise RuntimeError("diff_pruning_b200: the Inception feature pass runs on a CUDA device (no CPU fallback)")
        plan = self.plan(inp.shape[0], "f32", inp.shape[2:])
        plan.load(inp)
        plan.run()
        out = []
        for b in self.output_blocks:
            if b == 3:     # the final adaptive average pool is the plan's feature step
                out.append(plan.feat[3].clone()[:, :, None, None])
            else:
                out.append(plan.block_out[b].torch().permute(0, 3, 1, 2).clone())
        return out


def fold_bn(mod: BasicConv2d):
    """conv -> eval BN as one convolution: w' = w * g / sqrt(v + eps), b' = beta - m * g / sqrt(v + eps), in fp64, rounded once."""
    w = mod.conv.weight.detach().double().cpu()
    bn = mod.bn
    scale = bn.weight.detach().double().cpu() / torch.sqrt(bn.running_var.detach().double().cpu() + bn.eps)
    bias = bn.bias.detach().double().cpu() - bn.running_mean.detach().double().cpu() * scale
    return (w * scale[:, None, None, None]).float(), bias.float()


class FeaturePlan:
    """Forward-only Inception pass for a fixed batch size and input format.  src "u8": uint8 NHWC [B, H, W, 3] (decoded image files);
    "f32": fp32 NCHW [B, 3, H, W] in [0, 1], or in [-1, 1] with quantize=True (DDIM samples, taken through the PNG quantisation).
    `feat[b]` holds the [B, C] pooled features of every output block the model returns.
    Convolutions run on the general-geometry tensor-core kernel (DP_CONV_ANY_GEOMETRY; the library keeps the C = 3 stem on SIMT), with
    amax slots that every launch of the pass fills for the next; force_simt=True puts all of them on the exact-fp32 SIMT kernel (the
    benchmark's comparison)."""

    MAX_SLOTS = 256

    def __init__(self, model: InceptionV3, batch: int, src: str, hw, quantize: bool = False, use_graph: bool = True,
                 force_simt: bool = False):
        assert src in ("u8", "f32") and not (src == "u8" and quantize)
        self.key = (batch, src, (int(hw[0]), int(hw[1])), bool(quantize))
        self.model, self.B, self.src, self.quantize = model, batch, src, quantize
        self.conv_flags = DP_CONV_RELU | (DP_CONV_FORCE_SIMT if force_simt else DP_CONV_ANY_GEOMETRY)
        self.Hs, self.Ws = int(hw[0]), int(hw[1])
        self.use_graph = use_graph
        dev = torch.device("cuda", torch.cuda.current_device())
        self.dev = dev
        B = batch
        self.inp = (torch.empty(B, self.Hs, self.Ws, 3, dtype=torch.uint8, device=dev) if src == "u8" else
                    torch.empty(B, 3, self.Hs, self.Ws, dtype=torch.float32, device=dev))
        H, W = (299, 299) if model.resize_input else (self.Hs, self.Ws)
        self.x0 = View(torch.zeros(B, H, W, 4, device=dev), 0, 3)    # 4-channel pitch: 16-byte pixel rows
        self.steps = []          # launch list: callables enqueuing on the current stream
        self.weights = []        # (module, packed weight, bias) repacked when the parameters change
        self.macs = 0            # multiply-accumulates of the convolutions per pass
        self.buffers = []        # every activation buffer: the launch list holds raw pointers into them
        self.slots = torch.zeros(self.MAX_SLOTS, dtype=torch.int32, device=dev)   # amax slot per buffer, zeroed at the start of a pass
        self._slot_of: Dict[int, int] = {}
        self.conv_args = []
        self.block_out: Dict[int, View] = {}
        self.feat: Dict[int, torch.Tensor] = {}
        lib = L.load()
        Hs, Ws, resize, norm = self.Hs, self.Ws, int(model.resize_input), int(model.normalize_input)
        u8, q = int(src == "u8"), int(quantize)
        x0 = self.x0
        slots = self.slots
        self.steps.append(lambda: L.check(lib.dp_zero_u32(slots.data_ptr(), slots.numel(), _stream()), "zero amax slots"))
        s0 = self._slot(x0)
        self.steps.append(lambda: L.check(lib.dp_fid_input(self.inp.data_ptr(), u8, q, B, Hs, Ws, x0.ptr, x0.ld, x0.H, x0.W, resize, norm,
                                                           s0, _stream()), "fid_input"))
        x = x0
        for b, block in enumerate(model.blocks):
            for m in block:
                x = self._layer(m, x)
            self.block_out[b] = x
            if b in model.output_blocks:
                f = torch.empty(B, x.C, device=dev)
                self.feat[b] = f
                self.steps.append(lambda x=x, f=f: L.check(lib.dp_global_mean(x.ptr, x.ld, f.data_ptr(), f.shape[1], B, x.H, x.W, x.C,
                                                                              _stream()), "global_mean"))
        # one split-K workspace for all convolutions (they run one after the other)
        need = max([lib.dp_conv_splitk_workspace_floats(ctypes.byref(a), 0) for a in self.conv_args] + [0])
        self.workspace = torch.empty(max(need, 1), device=dev)
        for a in self.conv_args:
            a.workspace = self.workspace.data_ptr() if need > 0 else None
        self._sig = None
        self._graph = None

    # ---- plan construction
    def _slot(self, v: View) -> int:
        """Device address of the amax slot of the buffer a view lives in (all channel slices of a concat share it)."""
        i = self._slot_of.setdefault(v.t.data_ptr(), len(self._slot_of))
        assert i < self.MAX_SLOTS
        return self.slots.data_ptr() + 4 * i

    def _buf(self, H, W, C):
        t = torch.empty(self.B, H, W, C, device=self.dev)
        self.buffers.append(t)
        return View(t)

    def _conv(self, m: BasicConv2d, x: View, y: View):
        conv = m.conv
        K, C, R, S = conv.weight.shape
        assert C == x.C and K == y.C
        (sh, sw), (ph, pw) = conv.stride, conv.padding
        assert sh == sw
        P, Q = (x.H + 2 * ph - R) // sh + 1, (x.W + 2 * pw - S) // sh + 1
        assert (P, Q) == (y.H, y.W)
        self.macs += self.B * P * Q * K * C * R * S
        lib = L.load()
        cp = lib.dp_tc_weight_row(C)
        pk = dict(w=torch.empty(R * S * C * K, device=self.dev), bias=torch.empty(K, device=self.dev),
                  hi=torch.empty(R * S * K * cp, dtype=torch.float16, device=self.dev),
                  lo=torch.empty(R * S * K * cp, dtype=torch.float16, device=self.dev), slot=torch.zeros(1, dtype=torch.int32, device=self.dev))
        self.weights.append((m, pk))
        a = L.ConvArgs()
        a.N, a.H, a.W, a.C, a.P, a.Q, a.K, a.R, a.S, a.stride, a.pad_t, a.pad_l = self.B, x.H, x.W, C, P, Q, K, R, S, sh, ph, pw
        a.flags, a.splits = self.conv_flags, 1
        a.x, a.ldx, a.y, a.ldy, a.w, a.bias = x.ptr, x.ld, y.ptr, y.ld, pk["w"].data_ptr(), pk["bias"].data_ptr()
        a.w_tc_hi, a.w_tc_lo, a.amax_w = pk["hi"].data_ptr(), pk["lo"].data_ptr(), pk["slot"].data_ptr()
        a.amax_x, a.amax_out = self._slot(x), self._slot(y)
        self.conv_args.append(a)
        self.steps.append(lambda a=a: L.check(lib.dp_conv2d_fprop(ctypes.byref(a), _stream()), "inception conv"))

    def _out_hw(self, x: View, k, s, p):
        return (x.H + 2 * p[0] - k[0]) // s + 1, (x.W + 2 * p[1] - k[1]) // s + 1

    def _pool(self, x: View, y: View, stride, pad, mode):
        lib = L.load()
        B, sy = self.B, self._slot(y)
        self.steps.append(lambda: L.check(lib.dp_pool3x3(x.ptr, x.ld, y.ptr, y.ld, B, x.H, x.W, x.C, stride, pad, mode, sy, _stream()),
                                          "pool"))

    def _layer(self, m, x: View) -> View:
        if isinstance(m, BasicConv2d):
            H, W = self._out_hw(x, m.conv.kernel_size, m.conv.stride[0], m.conv.padding)
            y = self._buf(H, W, m.conv.out_channels)
            self._conv(m, x, y)
            return y
        if isinstance(m, nn.MaxPool2d):
            y = self._buf((x.H - 3) // 2 + 1, (x.W - 3) // 2 + 1, x.C)
            self._pool(x, y, 2, 0, 0)
            return y
        if isinstance(m, nn.AdaptiveAvgPool2d):
            return x          # the global mean of the last block is the feature step every output block gets
        return self._mixed(m, x)

    def _mixed(self, m: Mixed, x: View) -> View:
        spec = m.spec
        kind, pstride, ppad = spec["pool"]
        widths = {name: cout for name, _, cout, _, _, _ in spec["convs"]}
        widths["pool"] = x.C
        # output grid: every output branch has the same extent; take it from the first
        first = spec["out"][0]
        if first == "pool":
            H, W = (x.H + 2 * ppad - 3) // pstride + 1, (x.W + 2 * ppad - 3) // pstride + 1
        else:
            c = getattr(m, first).conv
            H, W = self._out_hw(x, c.kernel_size, c.stride[0], c.padding)
        out_t = torch.empty(self.B, H, W, sum(widths[n] for n in spec["out"]), device=self.dev)
        self.buffers.append(out_t)
        views, off = {}, 0
        for n in spec["out"]:
            views[n] = View(out_t, off, widths[n])
            off += widths[n]
        views["x"] = x
        if "pool" in views:          # B / D: the strided max pool is an output branch, written into its channel range
            self._pool(x, views["pool"], pstride, ppad, 0)
        else:
            views["pool"] = self._buf(x.H, x.W, x.C)
            self._pool(x, views["pool"], pstride, ppad, 0 if kind == "max" else 1)
        for name, src, cout, k, s, p in spec["convs"]:
            mod = getattr(m, name)
            if name not in views:
                Ho, Wo = self._out_hw(views[src], k, s, p)
                views[name] = self._buf(Ho, Wo, cout)
            self._conv(mod, views[src], views[name])
        return View(out_t)

    # ---- execution
    def _signature(self):
        return tuple((p.data_ptr(), p._version) for p in self.model.state_dict().values())

    def ensure_packed(self, force: bool = False):
        """Fold BatchNorm and pack every convolution weight when the module's tensors changed since the last pack."""
        sig = self._signature()
        if not force and sig == self._sig:
            return
        lib = L.load()
        for m, pk in self.weights:
            w, b = fold_bn(m)
            K, C, R, S = w.shape
            wd = w.to(self.dev).contiguous()
            L.check(lib.dp_pack_conv_weight(wd.data_ptr(), K, C, R, S, pk["w"].data_ptr(), None, _stream()), "pack")
            L.check(lib.dp_pack_conv_weight_tc(wd.data_ptr(), K, C, R, S, pk["hi"].data_ptr(), pk["lo"].data_ptr(), None, None,
                                               pk["slot"].data_ptr(), _stream()), "pack tc")
            pk["bias"].copy_(b.to(self.dev))
        torch.cuda.current_stream().synchronize()
        self._sig = sig

    def load(self, x: torch.Tensor, rows: Optional[int] = None):
        """Copy a batch into the plan's input buffer.  With rows < B the tail is zeroed: its features are ignored, and it must not carry
        the previous batch into the per-tensor operand scales of the tensor-core convolutions (features depend only on this batch)."""
        n = x.shape[0] if rows is None else rows
        assert n <= self.B and tuple(x.shape[1:]) == tuple(self.inp.shape[1:]) and x.dtype == self.inp.dtype
        self.inp[:n].copy_(x[:n], non_blocking=True)
        if n < self.B:
            self.inp[n:].zero_()

    def run_eager(self):
        for s in self.steps:
            s()

    def run(self):
        self.ensure_packed()
        if not self.use_graph:
            self.run_eager()
            return
        if self._graph is None:
            self._graph, = capture_graphs(self.dev, self.run_eager)
        self._graph.replay()


# ------------------------------------------------------------------------------------------------ moments and statistics
class Moments:
    """n, sum d and the upper triangle of sum d d^T of a feature stream, d = x - shift, in fp64 on the device.  The shift is the fp32
    mean of the first batch added (dp_global_mean over its rows), so the covariance does not cancel against mu mu^T when features sit far
    from zero.  Moments about one shift add: batches, padded final batches (only the valid rows enter) and, later, devices sharing the
    shift combine by plain sums (share_shift, then all_reduce)."""

    def __init__(self, dims: int, device=None):
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.D, self.n = dims, 0
        self.shift = torch.zeros(dims, dtype=torch.float32, device=dev)
        self.shift_set = False
        self.s = torch.zeros(dims, dtype=torch.float64, device=dev)
        self.sxx = torch.zeros(dims, dims, dtype=torch.float64, device=dev)

    def add(self, feat: torch.Tensor, rows: Optional[int] = None):
        rows = feat.shape[0] if rows is None else rows
        assert feat.dtype == torch.float32 and feat.is_cuda and feat.stride(1) == 1 and feat.shape[1] == self.D
        lib = L.load()
        if not self.shift_set and rows > 0:      # [rows][D] as one image of rows x 1 pixels
            L.check(lib.dp_global_mean(feat.data_ptr(), feat.stride(0), self.shift.data_ptr(), self.D, 1, rows, 1, self.D, _stream()),
                    "moments shift")
            self.shift_set = True
        L.check(lib.dp_feature_moments(feat.data_ptr(), feat.stride(0), rows, self.D, self.shift.data_ptr(), self.s.data_ptr(),
                                       self.sxx.data_ptr(), _stream()), "feature_moments")
        self.n += rows

    def share_shift(self, src: int = 0):
        """Every rank of the default process group takes rank `src`'s shift (one broadcast).  Called by all ranks, after rank src added
        its first rows and before any other rank added any."""
        import torch.distributed as dist
        if dist.get_rank() != src and self.n:
            raise RuntimeError("share_shift: this rank already added rows about a shift of its own")
        dist.broadcast(self.shift, src)
        self.shift_set = True

    def all_reduce(self):
        """Sums n, s and sxx over the ranks of the default process group, which must share the shift (share_shift): every rank then
        holds the moments of all their rows."""
        import torch.distributed as dist
        n = torch.tensor([self.n], dtype=torch.int64, device=self.s.device)
        for t in (n, self.s, self.sxx):
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
        self.n = int(n.item())

    def finalize(self):
        """(mu, sigma) as np.mean(act, 0) and np.cov(act, rowvar=False) define them, float64."""
        if self.n < 2:
            raise ValueError("need at least two feature rows for a covariance")
        s, sxx = self.s.cpu().numpy(), self.sxx.cpu().numpy()
        sxx = np.triu(sxx) + np.triu(sxx, 1).T
        d = s / self.n
        mu = self.shift.double().cpu().numpy() + d
        sigma = (sxx - self.n * np.outer(d, d)) / (self.n - 1)
        return mu, sigma


def _image_files(path) -> list:
    path = pathlib.Path(path)
    return sorted(f for ext in IMAGE_EXTENSIONS for f in path.glob("**/*.{}".format(ext)))


def _decode(files) -> torch.Tensor:
    from PIL import Image
    arrs = [np.asarray(Image.open(f).convert("RGB")) for f in files]
    shape = arrs[0].shape
    if any(a.shape != shape for a in arrs):
        raise NotImplementedError("images of different sizes in one batch (the reference's DataLoader cannot stack them either)")
    return torch.from_numpy(np.stack(arrs))


def _block_of(model: InceptionV3, dims: int) -> int:
    b = InceptionV3.BLOCK_INDEX_BY_DIM[dims]
    if b not in model.output_blocks:
        raise ValueError(f"model does not return block {b} ({dims} dims)")
    return b


def _run_files(files, model, batch_size, dims, consume):
    """Decode `files` on the host in batches, run the plan, hand (features [B, dims] on the device, valid rows) to `consume`."""
    b = _block_of(model, dims)
    for start in range(0, len(files), batch_size):
        x = _decode(files[start:start + batch_size])
        plan = model.plan(batch_size, "u8", x.shape[1:3])
        plan.load(x.to(plan.dev))
        plan.run()
        consume(plan.feat[b], x.shape[0])


def _check_device(device):
    if device is not None and torch.device(device).type != "cuda":
        raise NotImplementedError("the Inception feature pass runs on a CUDA device only")


def get_activations(files, model, batch_size=50, dims=2048, device="cuda", num_workers=1, res=None, dataset_name=None):
    """fid_score.py:100-179: [len(files), dims] float64 pool features of the image files (host copy of the device features)."""
    _check_device(device)
    if res is not None or dataset_name is not None:
        raise NotImplementedError("--res / --dataset_name crop transforms are not implemented")
    if batch_size > len(files):
        print("Warning: batch size is bigger than the data size. Setting batch size to data size")
        batch_size = len(files)
    out = np.empty((len(files), dims))
    pos = [0]

    def take(f, n):
        out[pos[0]:pos[0] + n] = f[:n].cpu().numpy()
        pos[0] += n
    _run_files(files, model, batch_size, dims, take)
    return out


def calculate_activation_statistics(files, model, batch_size=50, dims=2048, device="cuda", num_workers=1, res=None, dataset_name=None):
    """fid_score.py:239-261 with the moments accumulated on the device: (mu, sigma) float64."""
    _check_device(device)
    if res is not None or dataset_name is not None:
        raise NotImplementedError("--res / --dataset_name crop transforms are not implemented")
    batch_size = min(batch_size, len(files))
    mom = Moments(dims)
    _run_files(files, model, batch_size, dims, mom.add)
    return mom.finalize()


def compute_statistics_of_path(path, model, batch_size, dims, device="cuda", num_workers=1, num_samples=None, res=None,
                               dataset_name=None):
    """fid_score.py:264-282: a .npz with mu / sigma, or a folder of images (searched recursively, sorted)."""
    path = str(path)
    if path.endswith(".npz"):
        with np.load(path) as f:
            return f["mu"][:], f["sigma"][:]
    files = _image_files(path)
    if num_samples is not None:
        files = files[:num_samples]
    print("Found %d files." % len(files))
    return calculate_activation_statistics(files, model, batch_size, dims, device, num_workers, res=res, dataset_name=dataset_name)


def calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """d^2 = |mu1 - mu2|^2 + tr(sigma1) + tr(sigma2) - 2 tr((sigma1 sigma2)^(1/2)) in float64 (scipy.linalg.sqrtm).  A product whose
    square root is not finite is retried with eps added to both diagonals; an imaginary part is dropped when the diagonal's is within
    1e-3 of zero, else it is an error."""
    from scipy import linalg
    mu1, mu2 = np.atleast_1d(mu1), np.atleast_1d(mu2)
    sigma1, sigma2 = np.atleast_2d(sigma1), np.atleast_2d(sigma2)
    if mu1.shape != mu2.shape:
        raise ValueError("mean vectors have different lengths")
    if sigma1.shape != sigma2.shape:
        raise ValueError("covariances have different dimensions")
    root = linalg.sqrtm(sigma1 @ sigma2)
    if not np.isfinite(root).all():
        print("fid calculation produces singular product; adding %s to diagonal of cov estimates" % eps)
        eye = np.eye(sigma1.shape[0]) * eps
        root = linalg.sqrtm((sigma1 + eye) @ (sigma2 + eye))
    if np.iscomplexobj(root):
        if not np.allclose(np.diagonal(root).imag, 0, atol=1e-3):
            raise ValueError("Imaginary component {}".format(np.max(np.abs(root.imag))))
        root = root.real
    d = mu1 - mu2
    return d.dot(d) + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(root)


def _model_for(dims, weights=None):
    return InceptionV3([InceptionV3.BLOCK_INDEX_BY_DIM[dims]], weights=weights).cuda()


def calculate_fid_given_paths(paths, batch_size, device="cuda", dims=2048, num_workers=1, num_samples=None, res=None, dataset_name=None,
                              weights=None):
    """fid_score.py:285-301."""
    _check_device(device)
    for p in paths:
        if not os.path.exists(p):
            raise RuntimeError("Invalid path: %s" % p)
    model = _model_for(dims, weights)
    m1, s1 = compute_statistics_of_path(paths[0], model, batch_size, dims, device, num_workers, num_samples, res, dataset_name)
    m2, s2 = compute_statistics_of_path(paths[1], model, batch_size, dims, device, num_workers, num_samples, res, dataset_name)
    return calculate_frechet_distance(m1, s1, m2, s2)


def save_stats(path, mu, sigma):
    """An .npz with `mu` / `sigma`, interchangeable with fid_score.py --save-stats files."""
    np.savez_compressed(path, mu=mu, sigma=sigma)


def save_fid_stats(paths, batch_size, device="cuda", dims=2048, num_workers=1, num_samples=None, res=None, dataset_name=None, weights=None):
    """fid_score.py:304-321."""
    _check_device(device)
    if not os.path.exists(paths[0]):
        raise RuntimeError("Invalid path: %s" % paths[0])
    if os.path.exists(paths[1]):
        raise RuntimeError("Existing output file: %s" % paths[1])
    model = _model_for(dims, weights)
    print(f"Saving statistics for {paths[0]}")
    m1, s1 = compute_statistics_of_path(paths[0], model, batch_size, dims, device, num_workers, num_samples, res, dataset_name)
    save_stats(paths[1], m1, s1)


@torch.no_grad()
def statistics_of_pipeline(pipeline, total_samples, batch_size, num_inference_steps, seed=0, dims=2048, model=None, weights=None,
                           return_features=False):
    """FID statistics (mu, sigma) of `total_samples // batch_size` batches of DDIM samples drawn as ddpm_sample.py:57-74 draws them (one
    generator on the pipeline's device seeded with `seed`, one pipeline call per batch).  Each batch stays on the device and goes
    through the quantising input kernel, which reproduces the PNG the sampler would have written: the features equal those of
    compute_statistics_of_path on the saved folder.  return_features=True also returns the [n, dims] float64 features."""
    model = model if model is not None else _model_for(dims, weights)
    b = _block_of(model, dims)
    generator = torch.Generator(device=pipeline.device).manual_seed(seed)
    mom, feats = Moments(dims), []
    for _ in range(total_samples // batch_size):
        x = pipeline(batch_size=batch_size, num_inference_steps=num_inference_steps, generator=generator, output_type="device").images
        plan = model.plan(batch_size, "f32", x.shape[2:], quantize=True)
        plan.load(x)
        plan.run()
        mom.add(plan.feat[b])
        if return_features:
            feats.append(plan.feat[b].double().cpu().numpy())
    mu, sigma = mom.finalize()
    return (mu, sigma, np.concatenate(feats)) if return_features else (mu, sigma)
