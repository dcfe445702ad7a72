"""The slot audit's table (slot_audit.py) on the host: every amax slot an exported launch takes, as a struct field or as an argument, is
either audited against the operand view the launch's arguments describe or exempt with a reason, so a new kernel cannot slip past the
audit; and the views it reads are the ones dpb200.h documents."""
import ctypes as C
import os
import re

import slot_audit as sa
from diff_pruning_b200 import _lib as L

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dpb200.h")


def _header():
    text = open(HEADER).read()
    text = re.sub(r"/\*.*?\*/", " ", text, flags=re.S)
    return re.sub(r"//[^\n]*", " ", text)


def _param(decl: str):
    """'const uint32_t* amax' -> ('constuint32_t*', 'amax')."""
    m = re.fullmatch(r"(.*?)(\w+)", decl.strip(), flags=re.S)
    return re.sub(r"\s+", "", m.group(1)), m.group(2)


def _prototypes():
    """{entry point: [(type, name)]} of every function dpb200.h declares."""
    out = {}
    for m in re.finditer(r"\b(dp_\w+)\s*\(([^()]*)\)\s*;", _header()):
        params = [p for p in m.group(2).split(",") if p.strip() and p.strip() != "void"]
        out[m.group(1)] = [_param(p) for p in params]
    return out


def _is_slot_type(t: str) -> bool:
    return t in ("uint32_t*", "constuint32_t*")


def _slots_of_exports():
    """{(entry point, slot name)} over every exported launch (the entry points taking a stream last; the rest are host queries that
    launch nothing): the amax fields of its argument structs and its uint32_t* arguments."""
    protos = _prototypes()
    found = set()
    for name, (_, argtypes) in L._SIGS.items():
        if not argtypes or argtypes[-1] is not C.c_void_p:
            continue
        for t in argtypes:
            if isinstance(t, type) and issubclass(t, C._Pointer) and issubclass(t._type_, C.Structure):
                found |= {(name, f) for f, _ in t._type_._fields_ if f.startswith("amax")}
        found |= {(name, n) for t, n in protos[name] if _is_slot_type(t)}
    return found


def test_every_slot_of_every_export_is_audited_or_exempt():
    found = _slots_of_exports()
    table = set(sa.AUDITED) | set(sa.EXEMPT)
    assert not set(sa.AUDITED) & set(sa.EXEMPT), sorted(set(sa.AUDITED) & set(sa.EXEMPT))
    assert found - table == set(), f"amax slots neither audited nor exempt: {sorted(found - table)}"
    assert table - found == set(), f"table rows naming no slot of an exported launch: {sorted(table - found)}"
    assert all(len(r) > 20 for r in sa.EXEMPT.values())
    print(f"\n{len(found)} slots over {len({n for n, _ in found})} entry points: {len(sa.AUDITED)} audited, {len(sa.EXEMPT)} exempt")


def test_header_and_bindings_agree_on_the_arguments():
    """The header parse sees exactly the arguments the ctypes binding passes (so no uint32_t* argument hides from the check above),
    and dp_split_h3's slot is the argument the audit reads."""
    protos = _prototypes()
    assert set(L._SIGS) <= set(protos), sorted(set(L._SIGS) - set(protos))
    for name, (_, argtypes) in L._SIGS.items():
        assert len(protos[name]) == len(argtypes), (name, protos[name], argtypes)
    t, n = protos["dp_split_h3"][sa.SPLIT_SLOT_ARG]
    assert _is_slot_type(t) and n == "amax", (t, n)


def test_every_slot_field_of_the_header_structs_is_named_amax():
    """The binding-side rule above finds struct slots by name: every uint32_t* field of a dpb200.h struct is an amax_* field."""
    fields = []
    for body in re.findall(r"typedef\s+struct\s+\w*\s*\{(.*?)\}", _header(), flags=re.S):
        for decl in body.split(";"):
            if "uint32_t" in decl and "*" in decl:
                fields.append(_param(decl)[1])
    assert fields and all(f.startswith("amax") for f in fields), fields


def test_views_follow_the_launch_arguments():
    """input_views reads each view from the arguments as dpb200.h lays it out: conv x [N*H*W][C] / dy [N*P*Q][K] by pitch, NT-GEMM A
    [batch*H*W][Kg] (batch stride H*W*ld_a), split [batch][rows][cols] with its own batch stride; a launch forced onto SIMT still names
    its slots (the audit counts and skips it)."""
    a = L.ConvArgs()
    a.N, a.H, a.W, a.C, a.P, a.Q, a.K = 2, 8, 6, 5, 4, 3, 7
    a.x, a.ldx, a.y, a.ldy = 0x1000, 12, 0x2000, 9
    a.amax_x, a.amax_y, a.amax_w, a.amax_out = 0x10, 0x14, 0x18, 0x1C
    assert sa.input_views("dp_conv2d_fprop", [a]) == [("amax_x", 0x10, (0x1000, 1, 96, 5, 12, 0))]
    assert sa.input_views("dp_conv2d_dgrad", [a]) == [("amax_y", 0x14, (0x2000, 1, 24, 7, 9, 0))]
    assert sa.input_views("dp_conv2d_wgrad", [a]) == [("amax_x", 0x10, (0x1000, 1, 96, 5, 12, 0)), ("amax_y", 0x14, (0x2000, 1, 24, 7, 9, 0))]
    a.amax_x = None
    assert sa.input_views("dp_conv2d_fprop", [a]) == []
    g = L.GemmNtArgs()
    g.batch, g.H, g.W, g.Kg, g.N, g.A, g.ld_a, g.amax_a, g.amax_b = 3, 4, 32, 40, 128, 0x3000, 44, 0x20, 0x24
    assert sa.input_views("dp_gemm_nt_tc", [g]) == [("amax_a", 0x20, (0x3000, 3, 128, 40, 44, 128 * 44))]
    split = [0x4000, 44, 5000, 3, 128, 40, 1, 0x28, 0x5000, 0x6000]
    assert sa.input_views("dp_split_h3", split) == [("amax", 0x28, (0x4000, 3, 128, 40, 44, 5000))]
    assert sa.input_views("dp_amax", [0x4000, 44, 128, 40, 0x28]) == []
