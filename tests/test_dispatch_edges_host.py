"""Host checks of the dispatch-edge sweep: every threshold the kernels' host code dispatches on, read from the CUDA sources, has a case
of test_dispatch_edges_gpu.py at it and one across it (at 132 SMs, an H100 SXM), and the Python restatements the sweep predicts paths
with agree with the census's mirrors and with the C++ rules they restate."""
import itertools

import pytest

import dispatch_edges as de
import launch_census as lc

T = de.T
SMS = 132


def _conv(op=None, kernel=None):
    out = []
    for c in de.CONV:
        p = de.conv_path(c, SMS)
        if (op is None or c["op"] == op) and (kernel is None or p["kernel"] == kernel):
            out.append((c, p))
    return out


def _gemm_in(c):
    """(Kg, Nout) of a fprop / dgrad case's GEMM."""
    return (c["C"], c["K"]) if c["op"] == "fprop" else (c["K"], c["C"])


def test_thresholds_read_from_the_sources():
    assert T["ANY_MIN_C"] > 1 and T["PS_MAX_SPLIT_STAGES"] > 8 and T["BM"] > 0 and T["BK"] > 0 and T["PS_BN"] > 0
    assert T["NT"] * T["MAXCPT"] < T["LN_MAX_C"], "the LayerNorm row kernels are what admits channels beyond the GroupNorm map"
    assert T["GN_FOLD_BWD"] < T["GN_FOLD_FWD"]


def test_conv_box_and_simt_fallback():
    tc = _conv("fprop", "box")
    assert any(c["W"] == T["BM"] and p["box"] == (T["BM"], 1, 1) for c, p in tc), "W == BM"
    assert any(c["W"] == 2 * T["BM"] and p["box"] == (T["BM"], 1, 1) for c, p in tc), "BM divides W"
    assert any(p["box"][2] == 1 and p["box"][1] > 1 for c, p in tc), "W divides BM, H takes the rest"
    past = [(c, p) for c, p in _conv() if p["box"] and p["box"][2] > 1 and c["N"] % p["box"][2]]
    assert {c["op"] for c, _ in past} >= {"fprop", "dgrad", "wgrad"}, "a box running past the batch, per op"
    assert any(de.out_extent(c)[0] * de.out_extent(c)[1] * p["box"][2] == T["WG_KPIX"] for c, p in past if c["op"] == "wgrad")
    simt_w = {c["W"] for c, p in _conv("fprop", "simt") if de.box_geometry(c) and not c.get("flags") and al_ok(c)}
    assert simt_w >= {12, 24, 48, 192}, simt_w
    assert any(c["W"] == 32 and c["H"] == 6 for c, _ in _conv("fprop", "simt")), "W = 32, H = 6"
    assert _conv("dgrad", "simt") and _conv("wgrad", "simt") and _conv("wgrad", "wgrad_tc")
    assert any(p["box"][2] == 1 and de.out_extent(c)[0] * de.out_extent(c)[1] == T["WG_KPIX"] for c, p in _conv("wgrad", "wgrad_tc"))


def al_ok(c):
    return de.al16(c.get("px", 0), c["C"] + c.get("xe", 0))


def test_conv_kg_nout_and_wrow_tails():
    tc = _conv(kernel="box") + _conv(kernel="any")
    kg = {_gemm_in(c)[0] for c, _ in tc}
    nout = {_gemm_in(c)[1] for c, _ in tc}
    assert kg >= {T["BK"], T["BK"] + 1, 2 * T["BK"] - 1, 2 * T["BK"]}, sorted(kg)
    assert nout >= {T["PS_BN"], T["PS_BN"] + 1, 2 * T["PS_BN"], 2 * T["PS_BN"] + 1}, sorted(nout)
    assert kg >= {T["WROW_SPLIT"], T["WROW_SPLIT"] + 1} and any(k < T["WROW_SPLIT"] and k % T["WROW_SHORT"] == 0 for k in kg)
    # long rows pad to whole 64-element (128-byte) TMA box rows of one pipeline stage, short rows to the 16-byte TMA stride rule
    assert T["WROW_LONG"] == T["BK"] and T["WROW_SHORT"] * 2 == 16


def test_conv_ksplit_branches():
    rows = [(c, p, g) for c, p in _conv(kernel="box") + _conv(kernel="any") for g in p["gemms"] if c.get("ws", True)]
    iters = {}
    for c, p, g in rows:
        Kg = _gemm_in(c)[0]
        taps = c["R"] * c.get("S", c["R"])
        if c["op"] == "fprop" or c.get("stride", 1) == 1:
            iters[id(c)] = taps * de.cdiv(Kg, T["BK"])
    seen = set()
    for c, p, g in rows:
        ks, ips, work = g
        it = iters.get(id(c))
        tiles = work // ks
        if it is None:
            continue
        if tiles * 2 > SMS and ks == 1 and it <= T["PS_MAX_SPLIT_STAGES"]:
            seen.add("no split: tiles fill half the SMs" + (" at the chain limit" if it == T["PS_MAX_SPLIT_STAGES"] else ""))
        if tiles * 2 > SMS and it == T["PS_MAX_SPLIT_STAGES"] + 1:
            assert ks == 2
            seen.add("forced chain split, M filling the machine")
        if tiles * 2 <= SMS and it == 7:
            assert ks == 1
            seen.add("iters 7")
        if tiles * 2 <= SMS and it == 8:
            assert ks == 2
            seen.add("iters 8: capped at iters / 4")
        if tiles * 2 <= SMS and it >= 8 and min(SMS // tiles, it // 4) > 16:
            seen.add("capped at 16")
    assert seen >= {"no split: tiles fill half the SMs", "no split: tiles fill half the SMs at the chain limit",
                    "forced chain split, M filling the machine", "iters 7", "iters 8: capped at iters / 4", "capped at 16"}, seen


@pytest.mark.parametrize("sms", [114, 132])
def test_conv_persistent_rounds(sms):
    work = {g[2] for c in de.CONV for g in de.conv_path(c, sms)["gemms"] if g[0] == 1 and de.conv_path(c, sms)["kernel"] == "box"}
    assert work >= {sms - 1, sms, sms + 1, 2 * sms + 1}, sorted(work)


def test_conv_epilogue_alignment():
    box = [c for c, p in _conv("fprop", "box") if not p["vec4"]]
    assert any(c.get("ye") for c in box) and any(c.get("py") for c in box)
    for key in ("pb", "pr", "ps"):
        assert any(c.get(key) for c in box), f"a case with only {key} off its 16-byte phase"
        assert any(c.get(key) and not c.get("ws", True) for c in box) or key == "pb", key
    assert any(p["vec4"] and c.get("residual") and c.get("rowadd") and c.get("bias") for c, p in _conv("fprop", "box"))
    assert any(not p["vec4"] for c, p in _conv("fprop", "box") if any(g[0] > 1 for g in p["gemms"]))
    assert any(c.get("flags", 0) & de.ACC for c, _ in _conv("fprop", "box")) and any(c.get("flags", 0) & de.ACC for c, _ in _conv("dgrad", "box"))
    assert any(not p["vec4"] for c, p in _conv("dgrad", "box"))


def test_conv_dgrad_parity_classes():
    s2 = [(c, p) for c, p in _conv("dgrad", "box") if c.get("stride", 1) == 2]
    assert {c["pad"] for c, _ in s2} == {0, 1}
    assert {de.out_extent(c)[0] % 2 for c, _ in s2} == {0, 1}, "P odd and even on the tensor cores"
    assert all(len(p["gemms"]) == 4 for _, p in s2)


def test_conv_general_geometry():
    anyf = [c for c in de.CONV if c.get("flags", 0) & de.ANY]
    paths = {(c["C"], de.conv_path(c, SMS)["kernel"]) for c in anyf}
    assert (T["ANY_MIN_C"] - 1, "simt") in paths and (T["ANY_MIN_C"], "any") in paths, paths
    shapes = {(c["R"], c.get("S", c["R"])) for c in anyf if de.conv_path(c, SMS)["kernel"] == "any"}
    assert shapes >= {(1, 7), (7, 1), (5, 5)}, shapes
    run = [(c, de.conv_path(c, SMS)) for c in anyf]
    assert any(p["kernel"] == "any" and c.get("stride") == 2 and c.get("pad") == 0 for c, p in run)
    assert any(p["kernel"] == "any" and c["flags"] & de.RELU for c, p in run)
    assert any(p["kernel"] == "any" and any(g[0] > 1 for g in p["gemms"]) for c, p in run), "the flat split-K epilogue"
    assert any(p["kernel"] == "any" and not p["vec4"] for c, p in run)
    assert any(p["kernel"] == "simt" and c.get("rowadd") for c, p in run) and any(p["kernel"] == "box" and c.get("rowadd") for c, p in run)
    assert any(c.get("flags") == de.RELU and de.conv_path(c, SMS)["kernel"] == "simt" and de.box_geometry(c) for c in de.CONV)


def test_bf16_tiles_and_refusals():
    plans = [(c, de.bf16_plan(c)) for c in de.BF16]
    for c, (ok, _, _) in plans:
        assert ok == ("refuse" not in c), c["tag"]
    conv = [(c, tile) for c, (ok, tile, _) in plans if ok and c["op"] != "wgrad"]
    assert {tile for _, tile in conv} >= {64, 128, 192, 256}
    nouts = {(c["K"] if c["op"] == "fprop" else c["C"]) for c, _ in conv}
    assert nouts >= {T["BF_NTILE"], T["BF_NTILE"] + 1}, nouts
    assert any(c["C"] == 7 and "refuse" in c for c in de.BF16) and any(c["C"] == 8 and "refuse" not in c for c in de.BF16)
    assert any((c["C"] + c.get("xe", 0)) % 8 and "refuse" in c for c in de.BF16)
    wg = [(c, box) for c, (ok, _, box) in plans if c["op"] == "wgrad"]
    assert any("refuse" in c and box and box[2] > 1 and c["N"] % box[2] and de.out_extent(c)[0] * de.out_extent(c)[1] * box[2] == T["WG_PIX"]
               for c, box in wg)
    assert any("refuse" not in c and box and de.out_extent(c)[0] * de.out_extent(c)[1] == T["WG_PIX"] for c, box in wg)


def test_groupnorm_thresholds():
    run = [(c, de.gn_path(c)) for c in de.GN if "refuse" not in c]
    for c in de.GN:
        assert ("refuse" in de.gn_path(c)) == ("refuse" in c), c["tag"]
        if "refuse" in c:
            assert de.gn_path(c)["refuse"] == c["refuse"], c["tag"]
    gn = [(c, p) for c, p in run if not p["ln"]]
    for op in ("gn_fwd", "gn_bwd"):
        cs = {c["C"] for c, _ in gn if c["op"] == op}
        assert cs >= {32, T["NT"] - 1, T["NT"] + 1, T["NT"] * T["MAXCPT"]} and any(c < T["NT"] // 2 for c in cs), (op, cs)
    assert {c["C"] for c, _ in gn if c["op"] == "gn_fwd"} >= {64, 128, T["NT"]}
    assert any(c["C"] > T["NT"] * T["MAXCPT"] and c["op"] == "gn_fwd" and not ln for c, ln in ((c, de.ln_fast(c)) for c in de.GN if "refuse" in c))
    fwd = {p["nchunks"] for c, p in gn if c["op"] == "gn_fwd"}
    assert {T["GN_FOLD_FWD"], T["GN_FOLD_FWD"] + 1} <= fwd, fwd
    for v4 in (True, False):
        assert {T["GN_FOLD_FWD"], T["GN_FOLD_FWD"] + 1} <= {p["nchunks"] for c, p in gn if c["op"] == "gn_fwd" and p["v4"] == v4}, v4
    bwd = {p["nchunks"] for c, p in gn if c["op"] == "gn_bwd"}
    assert {T["GN_FOLD_BWD"], T["GN_FOLD_BWD"] + 1} <= bwd, bwd
    assert any(c.get("fin") for c, p in gn if p["reduce"]) and any(c.get("add") for c, p in gn if p["reduce"])
    assert any(c.get("alias") for c, _ in gn) and any(c.get("add") and not c.get("alias") for c, _ in gn)
    # every float4 condition on its own: exactly one view off, the rest aligned
    for op, keys in (("gn_fwd", ("px", "xe", "py", "ye")), ("gn_bwd", ("px", "dye", "pdx", "padd", "add2e"))):
        for k in keys:
            assert any(c["op"] == op and c.get(k) and not p["v4"] and c["C"] % 4 == 0 for c, p in gn), (op, k)
    # G <= 1024 is checked with the channel limit, but G divides C, so G > 1024 only comes with C > NT * MAXCPT, which refuses first:
    # the limit cannot be reached on its own.  The table runs G = 1024 and refuses a G beyond it.
    assert T["NT"] * T["MAXCPT"] <= 1024
    assert any(c["G"] == 1024 for c, _ in gn) and any(c["G"] > 1024 for c in de.GN if "refuse" in c)


def test_layernorm_admission():
    ln = [c for c in de.GN if c["HW"] == 1 and c["G"] == 1]
    runs = lambda c: "refuse" not in c and de.gn_path(c).get("ln")
    assert any(runs(c) and c["C"] == T["LN_MAX_C"] and c["op"] == op for c in ln for op in ("gn_fwd", "gn_bwd"))
    assert any(c["C"] == T["LN_MAX_C"] + 1 and "refuse" in c for c in ln)
    assert any(runs(c) and T["NT"] * T["MAXCPT"] < c["C"] < T["LN_MAX_C"] for c in ln)
    assert any(runs(c) and c["N"] > 65535 for c in ln)
    # above NT * MAXCPT each condition of the row kernels alone refuses: gamma, beta, x, y pitch, y missing; backward gamma, dx
    big = [c for c in ln if c["C"] > T["NT"] * T["MAXCPT"] and "refuse" in c and c["C"] <= T["LN_MAX_C"]]
    for op, k in (("gn_fwd", "pg"), ("gn_fwd", "pbeta"), ("gn_fwd", "px"), ("gn_fwd", "ye"), ("gn_fwd", "no_y"), ("gn_bwd", "pg"),
                  ("gn_bwd", "pdx"), ("gn_bwd", "padd2")):
        assert any(c["op"] == op and c.get(k) for c in big), (op, k)
    # off the row kernels below the limit: the GroupNorm kernels, which take one image per grid row
    assert any("refuse" not in c and not de.gn_path(c)["ln"] and c.get("pg") for c in ln)
    assert {c["refuse"] for c in ln if c["N"] > 65535 and "refuse" in c} == {de.DP_ERR_SHAPE}


@pytest.mark.parametrize("C", range(T["NT"] * T["MAXCPT"] + 4, T["LN_MAX_C"] + 1, 4))
def test_float4_map_has_no_pixel_lane_beyond_maxcpt(C):
    """Why validation refuses C > NT * MAXCPT off the row kernels: make_map4 has CT >= 2 NT thread slots per pixel there, so PL = 0
    pixel lanes and zero bytes of statistics shared memory (and the scalar map's MAXCPT channels per thread stop short of C)."""
    CT, PL, _, _ = de.make_map4(1, C)
    assert CT > T["NT"] and PL == 0
    assert de.make_map(1, C)[0] * T["MAXCPT"] < C


def test_rows_cases():
    cols = {a[1] for n, a in de.ROWS if n == "dp_softmax_fwd"}
    assert cols >= {1, 31, 32, 33, 4096, 4097}
    amax = [a for n, a in de.ROWS if n == "dp_amax"]
    dense = lambda a: a[1] == a[3]
    vec = lambda a: a[0] == 0 and (a[2] * a[3] if dense(a) else a[3]) % 4 == 0 and (dense(a) or a[1] % 4 == 0)
    assert {(dense(a), vec(a)) for a in amax} == {(True, True), (True, False), (False, True), (False, False)}
    cs = [a for n, a in de.ROWS if n == "dp_colsum"]
    assert any(a[0] == 0 and a[1] % 4 == 0 for a in cs) and any(a[0] or a[1] % 4 for a in cs)
    assert any(a[2] % a[4] for a in cs) and any(a[5] for a in cs)
    sp = [a for n, a in de.ROWS if n == "dp_split_h3"]
    vec = lambda a: a[0] == 0 and a[1] % 4 == 0 and a[2] % 4 == 0
    for tr in (0, 1):
        assert {vec(a) for a in sp if a[6] == tr} == {True, False}, tr
    assert any(a[0] for a in sp if not a[6]) and any(a[1] % 4 for a in sp if not a[6]) and any(a[2] % 4 for a in sp if not a[6])
    assert any(a[5] % 8 for a in sp if not a[6]) and any(a[4] % 8 for a in sp if a[6])
    tp = [a for n, a in de.ROWS if n == "dp_transpose_batched"]
    assert {a[1] % 4 == 0 and a[2] % 4 == 0 for a in tp} == {True, False} and any(a[1] % 64 and a[2] % 64 for a in tp)
    gm = [a for n, a in de.ROWS if n == "dp_gemm_batched"]
    assert {(a[4], a[5]) for a in gm} == {(0, 0), (0, 1), (1, 0), (1, 1)} and any(a[6] for a in gm)
    assert {a[1] for a in gm} >= {128, 129, 127} and {a[2] for a in gm} >= {128, 129} and {a[3] for a in gm} >= {15, 16, 17}


@pytest.mark.parametrize("sms", [114, 132])
def test_ksplit_mirrors_agree(sms):
    for tiles, iters in itertools.product(range(1, 300, 3), range(1, 400, 7)):
        assert lc.pick_ksplit(tiles, iters, sms) == de.pick_ksplit(tiles, iters, sms), (tiles, iters, sms)
    for c in de.CONV:
        if de.conv_path(c, sms)["kernel"] == "any":
            P, Q = de.out_extent(c)
            assert de.conv_path(c, sms)["gemms"][0][:2] == lc.general_split(c["N"], P, Q, c["K"], c["C"], c["R"], c.get("S", c["R"]), sms)


def test_pick_box_restatement():
    """pick_box against its meaning: boxes of npix pixels that tile whole rows of the grid, then whole images (the last box may run past
    the batch), found whenever such a box exists."""
    for npix in (64, 128):
        for H, W in itertools.product(range(1, 70), [1, 2, 3, 4, 6, 8, 12, 16, 24, 32, 48, 64, 96, 128, 192, 256, 384]):
            box = de.pick_box(npix, H, W)
            want = None
            if W % npix == 0:
                want = (npix, 1, 1)
            elif npix % W == 0 and H % (npix // W) == 0:
                want = (W, npix // W, 1)
            elif npix % W == 0 and (npix // W) % H == 0:
                want = (W, H, npix // (W * H))
            assert box == want, (npix, H, W, box, want)
