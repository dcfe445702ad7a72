"""Amax-slot audit read from the launch arguments (test_slot_audit_gpu.py; its table is checked against the exported entry points by
test_slot_audit_host.py).

Every fp32-grade tensor-core launch scales an operand by the power of two taken from its amax slot: a device uint32 that must hold the
bit pattern of an upper bound of max|operand| (conv_tc.cu, amax_exponent).  A slot below the operand's maximum lets s * v pass 2^14 and
the fp16 hi half overflow, silently.  SlotAudit is an on_call sink for launch_census.wrap_launches: before each launch that reads an input
slot it synchronises the device, reads the slot word and takes max|.| over exactly the view the launch's own arguments describe (base
pointer, pitch, rows, columns, batch stride), not the view the planner meant.  It asserts the slot is a finite, non-negative float bit
pattern and >= that maximum, and records the looseness slot / max.  In raise mode a violation raises before the library is called, so
the launch never runs; in record mode it is kept and the launch runs as usual.
"""
from __future__ import annotations

import struct

import torch

DP_CONV_FORCE_SIMT = 2          # dpb200.h: the launch never takes the tensor-core path, so it reads no slot

# (entry point, slot field or argument name) -> the operand view the slot bounds (dpb200.h, conv_tc.cu conv_launch / dp_gemm_nt_tc)
AUDITED = {
    ("dp_conv2d_fprop", "amax_x"): "x: N*H*W rows x C, pitch ldx",
    ("dp_conv2d_dgrad", "amax_y"): "dy: N*P*Q rows x K, pitch ldy",
    ("dp_conv2d_wgrad", "amax_x"): "x: N*H*W rows x C, pitch ldx",
    ("dp_conv2d_wgrad", "amax_y"): "dy: N*P*Q rows x K, pitch ldy",
    ("dp_gemm_nt_tc", "amax_a"): "A: batch*H*W rows x Kg, pitch ld_a",
    ("dp_split_h3", "amax"): "x: [batch][rows][cols], batch stride bs, pitch ld",
}
_OUT = "output: the launch accumulates the maximum of what it writes into it (dp_amax semantics)"
EXEMPT = {
    ("dp_conv2d_fprop", "amax_w"): "weight slot, written by dp_pack_conv_weight_tc, which the launch census checks to equal max|w|",
    ("dp_conv2d_dgrad", "amax_w"): "weight slot, written by dp_pack_conv_weight_tc, which the launch census checks to equal max|w|",
    ("dp_conv2d_wgrad", "amax_w"): "not read: the weight gradient's operands are x and dy",
    ("dp_conv2d_fprop", "amax_y"): "not read: y is fprop's output (conv_launch takes amax_x for the A operand)",
    ("dp_conv2d_dgrad", "amax_x"): "not read: x is dgrad's output dx (conv_launch takes amax_y for the A operand)",
    ("dp_conv2d_fprop", "amax_out"): _OUT,
    ("dp_conv2d_dgrad", "amax_out"): _OUT,
    ("dp_conv2d_wgrad", "amax_out"): "not read or written by the weight gradient",
    ("dp_gemm_nt_tc", "amax_b"): "slot of the matrix dp_split_h3 split into b_hi / b_lo: audited at that split",
    ("dp_gemm_nt_tc", "amax_out"): _OUT,
    ("dp_groupnorm_fwd", "amax_y"): _OUT,
    ("dp_groupnorm_fwd", "amax_dx"): "not read or written by the forward",
    ("dp_groupnorm_bwd", "amax_y"): "not read or written by the backward",
    ("dp_groupnorm_bwd", "amax_dx"): _OUT,
    ("dp_groupnorm_bwd_param", "amax_y"): "not read or written by the parameter gradient",
    ("dp_groupnorm_bwd_param", "amax_dx"): "not read or written by the parameter gradient",
    ("dp_amax", "slot"): _OUT,
    ("dp_zero_u32", "p"): "output: zeroes slots at the start of a pass",
    ("dp_pack_conv_weight_tc", "amax_w"): "output: the weight's own slot, checked exactly by the launch census",
    ("dp_softmax_bwd", "amax_ds"): _OUT,
    ("dp_fid_input", "amax_out"): _OUT,
    ("dp_pool3x3", "amax_out"): _OUT,
}
SPLIT_SLOT_ARG = 7              # dp_split_h3(x, ld, bs, batch, rows, cols, transpose, amax, hi, lo, stream)


class _Dev:
    """A raw device range as torch sees it (__cuda_array_interface__): no copy, no ownership."""

    def __init__(self, ptr: int, shape, strides, typestr="<f4"):
        self.__cuda_array_interface__ = {"data": (int(ptr), False), "shape": tuple(shape), "strides": tuple(strides),
                                         "typestr": typestr, "version": 2}


def device_view(ptr: int, batch: int, rows: int, cols: int, ld: int, bs: int) -> torch.Tensor:
    """The fp32 elements ptr[b * bs + r * ld + c], b < batch, r < rows, c < cols, as a [batch, rows, cols] tensor."""
    return torch.as_tensor(_Dev(ptr, (batch, rows, cols), (4 * bs, 4 * ld, 4)), device="cuda")


def slot_bits(ptr: int) -> int:
    return int(torch.as_tensor(_Dev(ptr, (1,), (4,), "<i4"), device="cuda").item()) & 0xFFFFFFFF


def input_views(name: str, args):
    """[(slot name, slot address, (ptr, batch, rows, cols, ld, batch stride))] of every input slot the launch names."""
    out = []
    if name in ("dp_conv2d_fprop", "dp_conv2d_dgrad", "dp_conv2d_wgrad"):
        a = args[0]
        if name != "dp_conv2d_dgrad" and a.amax_x:
            out.append(("amax_x", a.amax_x, (a.x, 1, a.N * a.H * a.W, a.C, a.ldx, 0)))
        if name != "dp_conv2d_fprop" and a.amax_y:
            out.append(("amax_y", a.amax_y, (a.y, 1, a.N * a.P * a.Q, a.K, a.ldy, 0)))
    elif name == "dp_gemm_nt_tc":
        a = args[0]
        if a.amax_a:
            out.append(("amax_a", a.amax_a, (a.A, a.batch, a.H * a.W, a.Kg, a.ld_a, a.H * a.W * a.ld_a)))
    elif name == "dp_split_h3":
        x, ld, bs, batch, rows, cols = args[:6]
        if args[SPLIT_SLOT_ARG]:
            out.append(("amax", args[SPLIT_SLOT_ARG], (x, batch, rows, cols, ld, bs)))
    return out


class SlotAudit:
    """on_call sink of launch_census.wrap_launches (see the module docstring).  raise_now=True raises at the first violation, before the
    library runs the launch; otherwise violations go to .failures and the launch runs.

    .launches: launches that name an input slot; .simt: of those, the ones flagged DP_CONV_FORCE_SIMT (they read no slot, so they are
    not audited); .checks: [(looseness slot / max, description)] of every audited slot whose operand is not all zero; .zero: audited
    slots whose operand is all zero (looseness undefined); .kinds: entry points audited."""

    def __init__(self, raise_now: bool = False):
        self.raise_now = raise_now
        self.launches = self.simt = self.zero = self.audited = 0
        self.checks, self.failures, self.kinds = [], [], set()

    def __call__(self, name, args, stream):
        views = input_views(name, args)
        if not views:
            return
        self.launches += 1
        if name.startswith("dp_conv2d") and args[0].flags & DP_CONV_FORCE_SIMT:
            self.simt += 1
            return
        torch.cuda.synchronize()        # every launch enqueued before this one (on any stream) has finished
        self.audited += 1
        self.kinds.add(name)
        for field, slot, (ptr, batch, rows, cols, ld, bs) in views:
            what = f"{name} #{self.launches} {field}: view ptr {ptr:#x} batch {batch} rows {rows} cols {cols} ld {ld} bs {bs}"
            bits = slot_bits(slot)
            bound = struct.unpack("<f", struct.pack("<I", bits))[0]
            top = float(device_view(ptr, batch, rows, cols, ld, bs).abs().amax()) if batch * rows * cols else 0.0
            msg = None
            if bits >= 0x7F800000:
                msg = f"{what}: slot bits {bits:#010x} are not a finite non-negative float"
            elif not bound >= top:
                msg = f"{what}: slot {bound!r} below the operand's maximum {top!r}"
            if msg is not None:
                if self.raise_now:
                    raise AssertionError(msg)
                self.failures.append(msg)
            elif top > 0:
                self.checks.append((bound / top, what))
            else:
                self.zero += 1

    def worst(self):
        return max(self.checks, default=(0.0, "none"))
