"""Host checks of the stream-order audit (footprint.py, stream_order.py): region intersection against brute-force byte sets,
happens-before semantics, and a synthetic two-stream backward with the engine's schedule shape in which every hazard the schedule's
invariants rule out is planted, one at a time, and must be reported at exactly its pair of launches."""
import random

import pytest

import footprint as fp
import stream_order as so


# ---------------------------------------------------------------------------------------------------------------- region algebra
def _bytes(r: fp.Region):
    return {r.ptr + i * r.pitch + b for i in range(r.rows) for b in range(r.cols * r.esz)}


def _brute_first(a: fp.Region, b: fp.Region):
    bb = _bytes(b)
    for i in range(a.rows):
        for e in range(a.cols):
            s = a.ptr + i * a.pitch + e * a.esz
            if any(s + k in bb for k in range(a.esz)):
                return i, e
    return None


def _rand_region(rng, base, esz=None, same=None):
    esz = esz or rng.choice((2, 4, 8))
    if same is not None:
        ld = same.ld * same.esz // esz if (same.ld * same.esz) % esz == 0 else same.ld
    else:
        ld = rng.randint(1, 12)
    cols = rng.randint(1, ld)
    rows = rng.randint(1, 9)
    ptr = base + rng.randint(0, 120)          # off the 16-byte phase on purpose
    return fp.Region(ptr, esz, rows, ld, cols)


def test_intersection_matches_brute_force_on_random_regions():
    rng = random.Random(7)
    hits = 0
    for n in range(6000):
        a = _rand_region(rng, 1 << 20)
        b = _rand_region(rng, 1 << 20, same=a if n % 2 else None, esz=a.esz if n % 3 == 0 else None)
        want = _brute_first(a, b)
        got = fp.first_overlap(a, b)
        assert (got is None) == (want is None), (a, b, got, want)
        if want is not None:
            hits += 1
            # the reported element overlaps b, and none of a before it does
            assert got == want, (a, b, got, want)
        assert fp.overlaps(b, a) == (want is not None)
    assert 1000 < hits < 5000            # both outcomes are exercised


@pytest.mark.parametrize("esz", [2, 4, 8])
def test_concat_halves_are_disjoint_and_pitch_padding_is_not_a_channel(esz):
    """The h half and the skip half of a torch.cat([h, skip]) buffer interleave row by row; a view over the pitch padding touches
    neither, while a view that reaches one channel into the other half does."""
    rows, Ch, Cs, pad = 37, 5, 7, 3
    ld = Ch + Cs + pad
    base = 0x7000 + 6                      # off the 16-byte phase
    h = fp.view(base, rows, ld, Ch, esz)
    skip = fp.view(base + esz * Ch, rows, ld, Cs, esz)
    padding = fp.view(base + esz * (Ch + Cs), rows, ld, pad, esz)
    assert fp.first_overlap(h, skip) is None and fp.first_overlap(skip, h) is None
    assert fp.first_overlap(h, padding) is None and fp.first_overlap(skip, padding) is None
    wide = fp.view(base, rows, ld, Ch + 1, esz)           # one channel into the skip half
    assert fp.first_overlap(wide, skip) == (0, Ch)
    assert fp.first_overlap(skip, wide) == (0, 0)
    whole = fp.view(base, rows, ld, ld, esz)               # dense: a flat range
    assert whole.rows == 1 and fp.first_overlap(whole, padding) == (0, Ch + Cs)
    last = fp.flat(base + esz * ((rows - 1) * ld + Ch), 1, esz)   # first skip element of the last row
    assert fp.first_overlap(skip, last) == (rows - 1, 0) and fp.first_overlap(h, last) is None


def test_different_pitch_and_element_size():
    a = fp.Region(0x1000, 4, 8, 16, 4)          # [8][16] floats, 4 channels
    b = fp.Region(0x1000 + 64 * 3 + 8, 2, 5, 8, 2)   # bf16 rows of another pitch inside row 3 of a
    assert fp.first_overlap(a, b) == (3, 2) == _brute_first(a, b)
    c = fp.Region(0x1000 + 20, 2, 4, 32, 2)      # in the padding of every row of a
    assert fp.first_overlap(a, c) is None and _brute_first(a, c) is None


# ----------------------------------------------------------------------------------------------------------------- happens-before
M, S, T = 0x100, 0x200, 0x300
BUF = 0x1000_0000


def L(stream, *accs, label=""):
    return so.Launch("k", None, stream, label, [fp.Access(f"f{i}", r, m) for i, (r, m) in enumerate(accs)])


def buf(i, n=64):
    return fp.flat(BUF + 0x10000 * i, n)


def _pairs(log):
    rep = so.check_races(log, {S, T})
    return {(r.a.label, r.b.label) for r in rep.races}, rep


def test_a_wait_covers_only_work_enqueued_before_it():
    a, b, c = L(S, (buf(0), fp.W), label="a"), L(S, (buf(1), fp.W), label="b"), L(M, (buf(0), fp.R), (buf(1), fp.R), label="c")
    log = so.clocks([a, so.Wait(M, S), b, c])
    assert so.hb(a, c) and not so.hb(b, c)
    pairs, rep = _pairs(log)
    assert pairs == {("b", "c")} and rep.ordered == 1


def test_ordering_is_transitive_through_a_third_stream():
    a, c = L(S, (buf(0), fp.W), label="a"), L(M, (buf(0), fp.R), label="c")
    log = so.clocks([a, so.Wait(T, S), so.Wait(M, T), c])
    assert so.hb(a, c)
    log2 = so.clocks([L(S, (buf(0), fp.W), label="a"), so.Wait(M, T), so.Wait(T, S), L(M, (buf(0), fp.R), label="c")])
    assert _pairs(log2)[0] == {("a", "c")}       # the waits in the other order do not chain


def test_host_synchronisation_orders_everything_before_it():
    a, b, c = L(S, (buf(0), fp.W), label="a"), L(T, (buf(1), fp.W), label="b"), L(M, (buf(0), fp.R), (buf(1), fp.R), label="c")
    assert _pairs(so.clocks([a, b, so.Sync(None), c]))[0] == set()
    a, b, c = L(S, (buf(0), fp.W), label="a"), L(T, (buf(1), fp.W), label="b"), L(M, (buf(0), fp.R), (buf(1), fp.R), label="c")
    assert _pairs(so.clocks([a, b, so.Sync(S), c]))[0] == {("b", "c")}       # a stream synchronisation covers that stream only


def test_events_order_like_waits():
    a, c = L(S, (buf(0), fp.W), label="a"), L(M, (buf(0), fp.R), label="c")
    assert _pairs([a, so.Record(1, S), so.WaitEvent(M, 1), c])[0] == set()
    a, b, c = L(S, (buf(0), fp.W), label="a"), L(S, (buf(0), fp.W), label="b"), L(M, (buf(0), fp.R), label="c")
    assert _pairs([a, so.Record(1, S), b, so.WaitEvent(M, 1), c])[0] == {("b", "c")}


def test_atomic_max_commits_commute_but_not_with_zeroing_or_reading():
    slot = fp.flat(BUF, 1)
    assert _pairs([L(S, (slot, fp.A), label="a"), L(M, (slot, fp.A), label="b")])[0] == set()
    assert _pairs([L(S, (slot, fp.A), label="a"), L(M, (slot, fp.W), label="z")])[0] == {("a", "z")}
    assert _pairs([L(S, (slot, fp.R), label="r"), L(M, (slot, fp.A), label="a")])[0] == {("r", "a")}
    other = fp.flat(BUF + 4, 1)                 # the next slot of the same array
    assert _pairs([L(S, (slot, fp.R), label="r"), L(M, (other, fp.A), label="a")])[0] == set()


def test_reads_never_conflict():
    assert _pairs([L(S, (buf(0), fp.R), label="a"), L(M, (buf(0), fp.R), label="b")])[0] == set()


# ------------------------------------------------------------------------------------------------------ synthetic engine schedule
def slot(i):
    return fp.flat(0x8000_0000 + 4 * i, 1)


DY = fp.view(0x1_0000_0000, 64, 8, 8)             # a per-tensor gradient buffer (dy of a convolution)
X = fp.view(0x2_0000_0000, 64, 8, 8)              # its forward input
DX = fp.view(0x3_0000_0000, 64, 8, 8)             # the next gradient down the main chain
CAT = 0x4_0000_0000
H_HALF = fp.view(CAT, 64, 12, 4)                  # h half of a concat buffer's gradient (channels 0..3 of 12)
SKIP = fp.view(CAT + 16, 64, 12, 6)               # its skip half (channels 4..9; 10, 11 are pitch padding)
SPLITK, SPLITK_SIDE = fp.flat(0x5_0000_0000, 4096), fp.flat(0x5_1000_0000, 4096)
GN_WS, FIN = fp.flat(0x6_0000_0000, 1024), fp.flat(0x6_1000_0000, 16)
WG_WS_SIDE = fp.flat(0x7_0000_0000, 4096)
ARENA = 0x9_0000_0000
DW1, DGAMMA, DW2, DW3 = (fp.flat(ARENA + 0x10000 * i, 64) for i in range(4))
SEG_SIDE, DTEMB = fp.flat(0xA_0000_0000, 16), fp.flat(0xA_1000_0000, 16)
SLOTS = fp.flat(0x8000_0000, 64)


def K(stream, label, *accs, name="k"):
    return so.Launch(name, None, stream, label, [fp.Access(f, r, m) for f, r, m in accs])


def schedule(plant=None):
    """One pass of the engine's backward shape, then the first launches of the next pass.  Launch labels name the pairs."""
    p = plant or ""
    ws_side = SPLITK if p == "shared split-K scratch" else SPLITK_SIDE
    param_reads = [("workspace", GN_WS, fp.R)] if p == "param reads gn_ws" else []
    log = [
        K(M, "zero slots", ("p", SLOTS, fp.W)), so.Sync(None, what="device"),
        K(M, "dgrad1", ("y", X, fp.R), ("x", DY, fp.W), ("amax_out", slot(0), fp.A)),
        so.Wait(S, M, "lead"),
        K(S, "wgrad1", ("x", X, fp.R), ("y", DY, fp.R), ("amax_y", slot(0), fp.R), ("workspace", WG_WS_SIDE, fp.W)),
        K(S, "reduce1", ("workspace", WG_WS_SIDE, fp.R), ("dw", DW1, fp.RW)),
        K(M, "gn bwd", ("dy", DY, fp.R), ("dx", DX, fp.W), ("workspace", GN_WS, fp.W), ("fin", FIN, fp.W), ("amax_dx", slot(1), fp.A)),
    ]
    if p == "main rewrites dy":
        log.append(K(M, "dy rewrite", ("x", DY, fp.W)))
    if p == "main commits into the side's slot":
        log.append(K(M, "skip writer", ("x", SKIP, fp.W), ("amax_out", slot(0), fp.A)))
    if p == "main zeroes the side's slot":
        log.append(K(M, "slot zero", ("p", slot(0), fp.W)))
    log += [
        so.Wait(S, M, "lead"),
        K(S, "gn param", ("fin", FIN, fp.R), ("dgamma", DGAMMA, fp.RW), *param_reads),
        K(M, "dgrad2", ("y", DX, fp.R), ("x", H_HALF, fp.W), ("workspace", SPLITK, fp.W)),
        K(M, "gn fwd2", ("workspace", GN_WS, fp.W)),
        so.Wait(S, M, "lead"),
        K(S, "temb colsum", ("x", H_HALF, fp.R), ("out", SEG_SIDE, fp.W)),
        K(S, "temb dgrad", ("y", SEG_SIDE, fp.R), ("x", DTEMB, fp.RW), ("workspace", ws_side, fp.W)),
        K(M, "skip write", ("y", DX, fp.R), ("x", SKIP, fp.RW)),            # interleaves with the h half the side is reading
        K(M, "dgrad3", ("y", DX, fp.R), ("x", fp.view(0x3_1000_0000, 64, 8, 8), fp.W), ("workspace", SPLITK, fp.W)),
    ]
    if p != "join dropped":
        log.append(so.Wait(M, S, "join"))
    log += [
        K(M, "silu bwd", ("dy", DTEMB, fp.R), ("dx", fp.flat(0xB_0000_0000, 16), fp.W)),
        so.Wait(S, M, "lead"),
        K(S, "wgrad in", ("x", X, fp.R), ("y", DY, fp.R), ("amax_y", slot(2), fp.R), ("workspace", WG_WS_SIDE, fp.W)),
        K(S, "reduce in", ("workspace", WG_WS_SIDE, fp.R), ("dw", DW3, fp.RW)),
    ]
    if p != "final join dropped":
        log.append(so.Wait(M, S, "final"))
    log += [K(M, "next zero slots", ("p", SLOTS, fp.W)), K(M, "next grad zero", ("self", fp.flat(ARENA, 0x40000 // 4), fp.W))]
    if p == "group lead dropped":
        i = next(k for k, e in enumerate(log) if isinstance(e, so.Launch) and e.label == "wgrad1")
        assert isinstance(log[i - 1], so.Wait)
        del log[i - 1]
    return log


PLANTED = {
    "group lead dropped": {("dgrad1", "wgrad1")},
    "main rewrites dy": {("wgrad1", "dy rewrite")},
    "main commits into the side's slot": {("wgrad1", "skip writer")},
    "main zeroes the side's slot": {("wgrad1", "slot zero")},
    "shared split-K scratch": {("temb dgrad", "dgrad3")},
    "param reads gn_ws": {("gn param", "gn fwd2")},
    "join dropped": {("temb dgrad", "silu bwd")},
    "final join dropped": {("wgrad in", "next zero slots"), ("reduce in", "next grad zero")},
}


def test_clean_schedule_reports_nothing_and_orders_its_conflicts():
    rep = so.check_races(schedule(), {S})
    assert rep.races == []
    assert rep.ordered >= 8              # the waits do order conflicting cross-stream pairs
    assert rep.side == 7
    assert so.check_aliasing(schedule()) == []


@pytest.mark.parametrize("hazard", sorted(PLANTED))
def test_planted_hazard_is_reported_at_its_pair(hazard):
    rep = so.check_races(schedule(hazard), {S})
    got = {(r.a.label, r.b.label) for r in rep.races}
    assert got == PLANTED[hazard], [str(r) for r in rep.races]
    assert all(r.hit is not None for r in rep.races)


def test_intra_launch_aliasing_and_the_in_place_allowlist():
    buf_ = fp.view(0x1000, 16, 8, 8)
    ok = so.Launch("dp_groupnorm_bwd", None, M, "", [fp.Access("dx", buf_, fp.W), fp.Access("dx_add", buf_, fp.R)])
    bad = so.Launch("dp_groupnorm_bwd", None, M, "", [fp.Access("dx", buf_, fp.W), fp.Access("dx_add2", buf_, fp.R)])
    shifted = so.Launch("dp_groupnorm_bwd", None, M, "", [fp.Access("dx", buf_, fp.W),
                                                         fp.Access("dx_add", fp.view(0x1004, 16, 8, 8), fp.R)])
    halves = so.Launch("dp_conv2d_dgrad", None, M, "", [fp.Access("x", fp.view(0x1000, 16, 8, 4), fp.W),
                                                       fp.Access("y", fp.view(0x1010, 16, 8, 4), fp.R)])
    msgs = so.check_aliasing([ok, bad, shifted, halves])
    assert len(msgs) == 2 and "dx_add2" in msgs[0] and "dx_add " in msgs[1] + " "


def test_lifetime_of_side_regions():
    a = K(S, "side", ("x", fp.flat(0x5000, 64), fp.R))
    a.t_us = 100
    w = so.Wait(M, S, "final", t_us=200)
    log = [so.Wait(S, M, "lead", t_us=50), a, w]
    assert so.check_lifetime(log, [(300, 0x5000, 512)], {S}) == []              # freed after the join
    msgs = so.check_lifetime(log, [(150, 0x4F00, 512)], {S})                     # freed before it
    assert len(msgs) == 1 and "side" in msgs[0]
    assert so.check_lifetime(log, [(150, 0x6000, 512)], {S}) == []              # another block


def test_footprints_of_every_kind_are_declared():
    """Every launching entry point of the C ABI has a footprint (the GPU test additionally checks each against the kernel)."""
    import ast
    import os
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "diff-pruning_b200", "_lib.py")).read()
    tree = ast.parse(src)
    names = set()
    for node in ast.walk(tree):
        if isinstance(node, ast.Dict):
            for k, v in zip(node.keys, node.values):
                if isinstance(k, ast.Constant) and isinstance(k.value, str) and k.value.startswith("dp_") and isinstance(v, ast.Tuple):
                    args = v.elts[1]
                    if isinstance(args, ast.List) and args.elts and isinstance(args.elts[-1], ast.Name) and args.elts[-1].id == "vp":
                        names.add(k.value)
    assert names and names <= set(fp.KINDS), sorted(names - set(fp.KINDS))
