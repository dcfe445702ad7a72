"""Race audit of the two-stream backward (DESIGN.md §5): every plan that forks work onto the side stream is recorded — library launches
with their streams and footprints (footprint.py), aten ops, waits, host synchronisations, allocator frees — and checked by
stream_order.py for cross-stream races, intra-launch aliasing and side-stream lifetime.  Single-stream paths are checked for one stream
and aliasing.  Planted edits of the recorded C1 / C5 logs (never executed) show the check has teeth.
"""
import ctypes as C

import pytest
import torch

import footprint as fp
import launch_census as lc
import stream_order as so
from test_launch_census_gpu import S, _inputs, lib  # noqa: F401  (lib: the module-scoped fixture)

pytestmark = pytest.mark.gpu
ROWS = []


def _plans(model):
    return list(model.__dict__.get("_dpb200_plans", {}).values())


def _side_streams(plans):
    return {p._side_stream.cuda_stream for p in plans if p._side_stream is not None}


class Recorded:
    """What a test keeps of one recorded plan once the plan is gone: the recorder (log, frees, live blocks), the side streams, whether a
    plan forks, and the main stream's shared scratch (for the planted re-pointing)."""

    def __init__(self, rec, plans):
        self.rec, self.side = rec, _side_streams(plans)
        self.forks = any(p._has_side for p in plans)
        sc = plans[0]._scratch if plans else {}
        ws = sc.get("wgrad_ws", sc.get("splitk_ws"))
        self.main_ws = ws.data_ptr() if ws is not None else 0


def _record(lib, run):
    rec = so.Recorder(lib)
    with rec.record():
        keep = run()            # alive until the recording's allocation snapshot is taken
        torch.cuda.synchronize()
    del keep
    return rec


def _check(tag, r: Recorded, forks=True):
    """Asserts no race, no unallowed aliasing, no lifetime violation; that a forking plan did fork and the checker saw conflicting
    cross-stream pairs the waits order; prints the plan's row."""
    rec, side = r.rec, r.side
    launches = [e for e in so.executed(rec.log) if isinstance(e, so.Launch) and e.src == "lib"]
    for s in {e.stream for e in launches}:
        if s > 0:                 # 0: the legacy default stream; < 0: the branches of a CUDA-graph replay
            assert so.stream_nonblocking(s), f"{tag}: stream {s:#x} is blocking (implicit barrier with the legacy default stream)"
    rep = so.check_races(rec.log, side)
    alias = so.check_aliasing(rec.log)
    life = so.check_lifetime(rec.log, rec.frees, side)
    # the allocator's trace and the log share one clock: every free the trace holds falls inside the recording
    assert all(rec.t0 - 1_000_000 <= t <= rec.t1 + 1_000_000 for t, _, _ in rec.frees), (rec.t0, rec.t1, rec.frees[:3])
    ROWS.append((tag, len(launches), sum(e.stream in side for e in launches), rep.ordered, len(rep.unused_waits)))
    print(f"\n{tag:34s} launches {len(launches):6d}  side {ROWS[-1][2]:5d}  conflicting cross-stream pairs {rep.ordered:6d}, all ordered"
          f"  waits ordering no conflict {len(rep.unused_waits)}")
    for x in rep.races[:10]:
        print("  ", x)
    for m in (alias + life)[:10]:
        print("  ", m)
    assert not rep.races, f"{tag}: {len(rep.races)} cross-stream races"
    assert not alias, f"{tag}: intra-launch aliasing"
    assert not life, f"{tag}: side-stream lifetime"
    if forks:
        assert r.forks
        assert ROWS[-1][2] > 0 and rep.ordered > 0, f"{tag}: the plan forks but nothing was checked across streams"
    else:
        assert len({e.stream for e in launches}) == 1, f"{tag}: a single-stream path used several streams"
    return rep


# ---------------------------------------------------------------------------------------------------------------------- plans
def _c1():
    import diff_pruning_b200 as dp
    torch.manual_seed(0)
    return dp.UNet2DModel(**dp.CIFAR10_DDPM_CONFIG).eval().cuda()


def _scorer_passes(model, B, hw, n=2, **kw):
    from diff_pruning_b200.scoring import TaylorScorer
    clean, noise = _inputs(B, hw)
    sc = TaylorScorer(model, clean, noise, use_graph=False, **kw)
    for t in (7, 400)[:n]:
        sc.step(t)
    return sc


def _rec_c1(lib, out):
    """C1 at batch 128: two accumulated eager passes, then the same scorer captured into a CUDA graph and replayed twice.  TaylorScorer's
    pass body is bracketed by marks, so the captured pass can be compared with the eager one."""
    from diff_pruning_b200.scoring import TaylorScorer
    orig, cur = TaylorScorer._body, {}

    def body(self):
        cur["rec"].mark("body>")
        orig(self)
        cur["rec"].mark("<body")
    TaylorScorer._body = body
    try:
        m = _c1()
        rec = so.Recorder(lib)
        cur["rec"] = rec
        with rec.record():
            sc = _scorer_passes(m, 128, 32)
            torch.cuda.synchronize()
        rec2 = so.Recorder(lib)
        cur["rec"] = rec2
        with rec2.record():
            sc.use_graph = True
            for t in (7, 400):
                sc.step(t)
            torch.cuda.synchronize()
    finally:
        TaylorScorer._body = orig
    plans = _plans(m)
    out["C1"], out["C1 graph"] = Recorded(rec, plans), Recorded(rec2, plans)


def _rec_c3(lib):
    import diff_pruning_b200 as dp
    torch.manual_seed(0)
    m = dp.UNet2DModel(**dp.LSUN256_DDPM_CONFIG).eval().cuda()
    return Recorded(_record(lib, lambda: _scorer_passes(m, 4, 256)), _plans(m))


def _rec_c5(lib):
    from diff_pruning_b200 import ldm
    m, cfg = lc.c5_model()
    m = m.cuda()
    ctx = torch.randn(6, 1, cfg["context_dim"], generator=torch.Generator().manual_seed(9)).cuda()
    return Recorded(_record(lib, lambda: _scorer_passes(m, 6, 64, alphas_cumprod=ldm.ldm_alphas_cumprod(), context=ctx)), _plans(m))


def _rec_finetune(lib, compute):
    from diff_pruning_b200.scoring import FinetuneStepper
    from test_pruned_census_gpu import _fresh
    m = _fresh("C1", 0.3).train()

    def run():
        st = FinetuneStepper(m, use_graph=False, compute=compute)
        g = torch.Generator().manual_seed(5)
        for step in range(2):
            clean, noise = torch.randn(8, 3, 32, 32, generator=g).cuda(), torch.randn(8, 3, 32, 32, generator=g).cuda()
            st.step(clean, noise, (torch.arange(8) * 124 + 3 * step) % 1000)
        return st
    return Recorded(_record(lib, run), _plans(m))


def _rec_sweep(lib, family, ratio, B):
    from diff_pruning_b200.scoring import TaylorScorer
    from test_pruned_census_gpu import HW, _batch, _fresh
    m = _fresh(family, ratio)

    def run():
        clean, noise = _batch(B, HW[family])
        sc = TaylorScorer(m, clean, noise, use_graph=False, fused_scores=True)
        for t in (7, 400):
            sc.step(t)
        return sc
    return Recorded(_record(lib, run), _plans(m))


def _rec_ldm(lib):
    from test_ldm_sampling_gpu import _loop, _tiny_ld
    ld = _tiny_ld()
    return Recorded(_record(lib, lambda: _loop(ld, 2, 1, use_graph=True)), _plans(ld.model.diffusion_model))


def _rec_ddim(lib):
    from test_pruned_census_gpu import _ddim, _fresh
    m = _fresh("C1", 0.3)
    return Recorded(_record(lib, lambda: (m, _ddim(m, 8))), [])


def _rec_fid(lib):
    from diff_pruning_b200 import fid
    from test_eval_census_gpu import _seeded_inception
    model = _seeded_inception()
    x = torch.randint(0, 256, (50, 32, 32, 3), generator=torch.Generator().manual_seed(13), dtype=torch.uint8).cuda()

    def run():
        plan = fid.FeaturePlan(model, 50, "u8", (32, 32), quantize=False, use_graph=False)
        plan.load(x)
        plan.ensure_packed()
        plan.run_eager()
        return plan
    return Recorded(_record(lib, run), [])


def _rec_vq_ssim(lib):
    """VQ-f4 decode of two 16 x 16 latents (dp_vq_quantize + the decoder plan), the decoded images as saved (dp_decode_images), and SSIM
    of three image pairs."""
    from diff_pruning_b200.ssim import ssim
    from test_vq_decoder_gpu import _vq_f4
    m = _vq_f4().cuda()
    m.use_graph = False
    h = (torch.randn(2, 3, 16, 16, generator=torch.Generator().manual_seed(9)) * 2e-4).cuda()
    g = torch.Generator().manual_seed(4)
    X, Y = torch.rand(3, 3, 37, 45, generator=g).cuda(), torch.rand(3, 3, 37, 45, generator=g).cuda()

    def run():
        img = m.decode(h)
        y = img.permute(0, 2, 3, 1).contiguous()
        u8 = torch.empty(y.shape, dtype=torch.uint8, device="cuda")
        f = torch.empty_like(img)
        assert lib.dp_decode_images(y.data_ptr(), 3, 2, 3, y.shape[1], y.shape[2], u8.data_ptr(), f.data_ptr(),
                                    torch.cuda.current_stream().cuda_stream) == 0
        return img, y, u8, f, ssim(X, Y, data_range=1.0, size_average=False)
    return Recorded(_record(lib, run), [])


SWEEP = [("C1", 0.05, 16), ("C1", 0.3, 16), ("C1", 0.7, 16), ("C3", 0.3, 2)]
RECORD = {"C3": _rec_c3, "C5": _rec_c5, "finetune fp32": lambda lib: _rec_finetune(lib, "fp32"),
          "finetune bf16": lambda lib: _rec_finetune(lib, "bf16"), "LDMPruneScorer": _rec_ldm, "DDIM": _rec_ddim,
          "FID features": _rec_fid, "VQ decode + SSIM": _rec_vq_ssim}
RECORD.update({f"{f} {r} b{B}": (lambda lib, f=f, r=r, B=B: _rec_sweep(lib, f, r, B)) for f, r, B in SWEEP})


@pytest.fixture(scope="module")
def recorded(lib):
    """tag -> Recorded, each plan recorded once on first use (the planted-race and footprint tests need no other test to have run)."""
    import gc
    cache = {}

    def get(tag):
        if tag not in cache:
            if tag in ("C1", "C1 graph"):
                _rec_c1(lib, cache)
            else:
                cache[tag] = RECORD[tag](lib)
            gc.collect()                      # plans and their models form reference cycles
            torch.cuda.empty_cache()
        return cache[tag]
    get.all = lambda: [get(t) for t in ["C1", "C1 graph"] + list(RECORD)]
    return get


def test_c1_taylor_eager_and_captured(recorded):
    """The captured pass enqueues exactly the eager pass's events, up to stream handles; the replays run it with its branches joined."""
    eager_r, graph_r = recorded("C1"), recorded("C1 graph")
    _check("C1 b128 Taylor, 2 eager passes", eager_r)
    _check("C1 b128 Taylor, graph capture", graph_r)

    def bodies(log):
        out, cur_ = [], None
        for e in log:
            if isinstance(e, so.Mark) and e.text in ("body>", "<body"):
                cur_ = [] if e.text == "body>" else (out.append(cur_) or None)
            elif cur_ is not None and not isinstance(e, so.Mark):
                cur_.append(e)
        return out
    eager, captured = bodies(eager_r.rec.log), bodies(graph_r.rec.log)
    assert len(eager) == 2 and len(captured) == 2      # warm-up outside the capture, then the captured pass
    span = so.captured(graph_r.rec.log)
    assert len(span) == 1 and all(any(e is x for x in span[0]) for e in captured[-1])
    assert so.canonical(captured[-1]) == so.canonical(eager[-1])
    replayed = [e for e in so.executed(graph_r.rec.log) if isinstance(e, so.Launch) and e.src == "lib"]
    assert len(replayed) >= 3 * sum(isinstance(e, so.Launch) and e.src == "lib" for e in captured[-1])


def test_c3_taylor(recorded):
    _check("C3 b4 Taylor, 2 eager passes", recorded("C3"))


def test_c5_taylor(recorded):
    r = recorded("C5")
    _check("C5 b6 Taylor, 2 eager passes", r)
    # one-pixel LayerNorm rows keep dgamma / dbeta on the main stream
    ln = [e for e in r.rec.log if isinstance(e, so.Launch) and e.name == "dp_groupnorm_bwd" and e.args[0].HW == 1]
    assert ln and all(e.stream not in r.side and not e.args[0].fin for e in ln)


@pytest.mark.parametrize("compute", ["fp32", "bf16"])
def test_pruned_c1_finetune(recorded, compute):
    r = recorded(f"finetune {compute}")
    _check(f"pruned C1 finetune {compute}, 2 steps", r)
    assert [e.name for e in r.rec.log if isinstance(e, so.Launch)].count("dp_adam_clip_ema") == 2


@pytest.mark.parametrize("family,ratio,B", SWEEP)
def test_pruned_sweep_taylor(recorded, family, ratio, B):
    _check(f"{family} pruned {ratio} Taylor b{B}", recorded(f"{family} {ratio} b{B}"))


def test_ldm_prune_scorer_iteration(recorded):
    """One LDMPruneScorer iteration: sample graph, forward + loss graph, the stop rule's read-back, backward graph."""
    _check("LDMPruneScorer, 1 iteration (graphs)", recorded("LDMPruneScorer"))


@pytest.mark.parametrize("tag", ["DDIM", "FID features", "VQ decode + SSIM"])
def test_single_stream_paths(recorded, tag):
    """DDIM sampling (pruned C1), the FID Inception feature pass, VQ-f4 decoding with the saved-image conversion, and SSIM: every launch on
    one stream, no unallowed aliasing."""
    r = recorded(tag)
    _check(f"{tag} (single stream)", r, forks=False)
    kinds = {e.name for e in r.rec.log if isinstance(e, so.Launch) and e.src == "lib"}
    want = {"DDIM": {"dp_ddim_step"}, "FID features": {"dp_fid_input", "dp_pool3x3", "dp_global_mean"},
            "VQ decode + SSIM": {"dp_vq_quantize", "dp_decode_images", "dp_ssim"}}[tag]
    assert want <= kinds, sorted(want - kinds)


# ---------------------------------------------------------------------------------------------------------------------- teeth
def _backward_waits(log, side):
    """Indices of the waits run_backward issues: group leads (side waits main), mid-pass joins and final joins (main waits side; the
    final join is the one on run_backward's last wait line)."""
    tagged = [(i, e) for i, e in enumerate(log) if isinstance(e, so.Wait) and e.tag.startswith("run_backward:")]
    line = lambda e: int(e.tag.split(":")[1])
    leads = [i for i, e in tagged if e.waiter in side]
    mains = [(i, e) for i, e in tagged if e.waited in side and e.waiter not in side]
    last = max(line(e) for _, e in mains)
    return leads, [i for i, e in mains if line(e) != last], [i for i, e in mains if line(e) == last]


@pytest.mark.parametrize("net", ["C1", "C5"])
def test_planted_races_in_recorded_logs_are_reported(recorded, net):
    r = recorded(net)
    rec, side = r.rec, r.side
    log = list(rec.log)
    leads, joins, finals = _backward_waits(log, side)
    assert leads and joins and len(finals) == 2, (len(leads), len(joins), len(finals))
    reported = {}

    def run(what, edited, expect):
        rep = so.check_races(edited, side)
        assert rep.races, f"{net}: planted '{what}' not reported"
        hit = [x for x in rep.races if expect(x)]
        assert hit, f"{net}: '{what}' reported elsewhere: {rep.races[:3]}"
        reported[what] = hit[0]
        print(f"\n{net} planted {what}: {len(rep.races)} races, at the planted pair e.g. {hit[0]}")

    def first_after(i, pred):
        return next(e for e in log[i + 1:] if isinstance(e, so.Launch) and pred(e))

    # 1. drop the mid-pass join: the first main-stream reader of d silu(temb) after it races with the side stream's time-embedding branch
    j = joins[0]
    reader = first_after(j, lambda e: e.stream not in side and e.name == "dp_silu_bwd")
    run("join dropped", log[:j] + log[j + 1:], lambda x: x.b is reader and x.a.stream in side and x.a.pos < j)
    # 2. drop one side group's leading wait: the first group whose first launch then races with the main stream's earlier work
    for i in leads:
        first = first_after(i, lambda e: True)
        rep = so.check_races(log[:i] + log[i + 1:], side)
        hit = [x for x in rep.races if x.b is first and x.a.stream not in side and x.a.pos < i]
        if hit:
            reported["group lead dropped"] = hit[0]
            print(f"\n{net} planted group lead dropped: {len(rep.races)} races, at the planted pair e.g. {hit[0]}")
            break
    else:
        pytest.fail(f"{net}: dropping a group's leading wait was never reported at that group")
    # 3. drop the first pass's final join: the next pass's first launch on the main stream, the zeroing of every amax slot, races with
    #    the first pass's side work after its mid-pass join (weight gradients of the time-embedding MLP reading their dy slots)
    f = finals[0]
    zero = first_after(f, lambda e: e.stream not in side and e.name == "dp_zero_u32")
    assert zero.pos < first_after(f, lambda e: e.stream not in side and e.name == "dp_conv2d_fprop").pos   # before the next forward's work
    run("final join dropped", log[:f] + log[f + 1:], lambda x: x.b is zero and x.a.stream in side and j < x.a.pos < f)
    # 4. re-point one side weight gradient's workspace at the main stream's shared scratch
    k = next(i for i, e in enumerate(log) if isinstance(e, so.Launch) and e.name == "dp_conv2d_wgrad" and e.stream in side and
             any(isinstance(x, so.Launch) and x.stream not in side and any(a.field == "workspace" and a.region.ptr == r.main_ws
                                                                            for a in x.accs) for x in log[i:]))
    e = log[k]
    args = [type(e.args[0])()]
    C.memmove(C.byref(args[0]), C.byref(e.args[0]), C.sizeof(e.args[0]))
    args[0].workspace = r.main_ws
    moved = so.Launch(e.name, args, e.stream, e.label, fp.footprint(e.name, args, rec.ctx))
    run("side wgrad on the main scratch", log[:k] + [moved] + log[k + 1:],
        lambda x: x.a is moved and x.b.stream not in side and x.xa.field == "workspace")
    assert len(reported) == 4


# ---------------------------------------------------------------------------------------------------------- footprint validation
FILL = {"NaN": 0x7FC00000, "0": 0}
POSITIVE = {"rstd", "sumsq", "step_scalars"}
DTYPE = {"f32": torch.float32, "acp": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "f64": torch.float64,
         "i64": torch.int64, "seed": torch.int64, "u8": torch.uint8, "slot": torch.int32}


def _owner(live, allocs, p):
    """The allocation holding address p: the live one at the end of the recording, else the largest allocation the recording made there."""
    import bisect
    i = bisect.bisect_right(live, (p, 1 << 62)) - 1
    if i >= 0 and live[i][0] + live[i][1] > p:
        return live[i] + (True,)
    best = None
    for a, n in reversed(allocs[max(0, bisect.bisect_right(allocs, (p, 1 << 62)) - 256):bisect.bisect_right(allocs, (p, 1 << 62))]):
        if a + n > p and (best is None or n > best[1]):
            best = (a, n)
    return None if best is None else best + (False,)


def _pointers(name, args):
    """[(setter, value)] of every non-NULL pointer of a captured call (struct fields or arguments)."""
    out = []
    if name in fp.STRUCT_KINDS:
        a = args[0]
        for f, t in a._fields_:
            if t is C.c_void_p and getattr(a, f):
                out.append((f, getattr(a, f)))
    else:
        for i, (k, v) in enumerate(zip(lc.argkinds(name), args)):
            if k == "p" and v:
                out.append((i, int(v)))
    return out


def _rebind(name, args, remap):
    if name in fp.STRUCT_KINDS:
        b = type(args[0])()
        C.memmove(C.byref(b), C.byref(args[0]), C.sizeof(b))
        for f, v in _pointers(name, args):
            setattr(b, f, remap(v))
        return [b]
    out = list(args)
    for i, v in _pointers(name, args):
        out[i] = remap(v)
    return out


def _typed(buf, base, r: fp.Region, dtype):
    off = r.ptr - base
    assert off % r.esz == 0, (off, r)
    return torch.as_strided(buf.view(dtype), (r.rows, r.cols), (r.ld, 1), off // r.esz)


def _bytes(buf, base, r: fp.Region):
    return torch.as_strided(buf, (r.rows, r.cols * r.esz), (r.pitch, 1), r.ptr - base)


def _replay(lib, ctx, name, args, live, allocs):
    """Runs one captured launch on fresh buffers twice (undeclared bytes NaN, then 0).  Returns a list of failures."""
    ptrs = _pointers(name, args)
    owner = {}
    for _, v in ptrs:
        b = _owner(live, allocs, v)
        if b is None:
            return [f"{name}: pointer {v:#x} lies in no allocation of the recording"]
        owner[v] = b
    outs, bad = {}, []
    for fill, pattern in FILL.items():
        # an allocation known only from the allocator's trace (freed before the recording ended) may have been one of several at that
        # address: its buffer grows to hold the declared regions of the pointers in it.  A live allocation never grows.
        size = {b: b[1] for b in owner.values()}
        for x in fp.footprint(name, args, ctx):
            b = owner.get(x.region.ptr)
            if b is not None and not b[2]:
                size[b] = max(size[b], x.region.hi - b[0])
        bufs = {b: torch.empty(-(-size[b] // 8) * 8, dtype=torch.uint8, device="cuda") for b in size}
        for t in bufs.values():
            t.view(torch.int32).fill_(pattern)
        remap = lambda v: bufs[owner[v]].data_ptr() + (v - owner[v][0])
        new = _rebind(name, args, remap)
        accs = fp.footprint(name, new, ctx)

        def where(r):
            for b, t in bufs.items():
                if t.data_ptr() <= r.ptr and r.hi <= t.data_ptr() + t.numel():
                    return t
            raise AssertionError(f"{name}: a declared region at {r.ptr:#x} does not fit the allocation its pointer lies in")
        g = torch.Generator(device="cuda").manual_seed(97)
        for x in accs:                       # seeded inputs: everything read, accumulated into or raised by atomic max
            if x.mode == fp.W or x.kind == "slot":
                continue
            t = where(x.region)
            v = _typed(t, t.data_ptr(), x.region, DTYPE[x.kind])
            if x.kind in ("f32", "acp", "f16", "bf16", "f64"):
                lo, hi = (0.5, 1.5) if x.field in POSITIVE else ((0.01, 0.99) if x.kind == "acp" else (-1.0, 1.0))
                v.copy_(torch.empty(v.shape, device="cuda", dtype=torch.float64).uniform_(lo, hi, generator=g).to(v.dtype))
            elif x.kind == "i64":
                v.copy_(torch.randint(0, fp.T_TABLE, v.shape, device="cuda", generator=g))
            elif x.kind == "seed":
                v.copy_(torch.randint(0, 1 << 62, v.shape, device="cuda", generator=g))
            elif x.kind == "u8":
                v.copy_(torch.randint(0, 256, v.shape, device="cuda", generator=g, dtype=torch.uint8))
        for x in accs:                       # amax slots: max|operand| for a read slot, 0 for one the call raises or resets
            if x.kind != "slot" or x.mode == fp.W:
                continue
            t = where(x.region)
            val = 0.0
            if x.mode == fp.R:
                op = next((y for y in accs if y.field == x.of and y.kind == "f32"), None)
                val = float(_typed(where(op.region), where(op.region).data_ptr(), op.region, torch.float32).abs().max()) if op else 1.0
            _typed(t, t.data_ptr(), x.region, torch.int32).copy_(torch.tensor([val], dtype=torch.float32).view(torch.int32).cuda()
                                                                  .expand(x.region.rows, x.region.cols))
        before = {b: t.clone() for b, t in bufs.items()}
        fn = getattr(lib, name)
        rc = fn(C.byref(new[0]), S()) if name in fp.STRUCT_KINDS else fn(*new, S())
        torch.cuda.synchronize()
        if rc:
            return [f"{name}: the replay returned {rc}"]
        for b, t in bufs.items():            # writes within the declared W / RW / A regions only
            mask = torch.zeros_like(t, dtype=torch.bool)
            for x in accs:
                if x.mode in fp.WRITES and where(x.region) is t:
                    _bytes(mask, t.data_ptr(), x.region).fill_(True)
            stray = (t != before[b]) & ~mask
            if bool(stray.any()):
                i = int(stray.nonzero()[0])
                bad.append(f"{name} (F={fill}): byte {i} of a {b[1]}-byte allocation written outside the declared regions")
        outs[fill] = [(x.field, _bytes(where(x.region), where(x.region).data_ptr(), x.region).clone()) for x in accs
                      if x.mode in fp.WRITES and not x.scratch]
    nan = torch.tensor([FILL["NaN"]], dtype=torch.int32).view(torch.uint8).cuda()
    for (f, a), (_, b) in zip(outs["NaN"], outs["0"]):
        if not torch.equal(a, b):
            d = (a != b).nonzero()[0].tolist()
            unwritten = bool((a.view(-1)[: a.numel() // 4 * 4].view(-1, 4) == nan).all(1).any())
            bad.append(f"{name}: output {f} differs between the NaN and 0 fills at (row, byte) {tuple(d)} of {tuple(a.shape)}"
                       + (" (declared written, left unwritten)" if unwritten else " (reads undeclared bytes)"))
    return bad


def test_footprints_match_the_kernels(lib, recorded):
    """Every unique launch (launch_census.launch_key) of every recorded plan, replayed on fresh buffers that keep the offsets of its
    pointers inside their allocations (so in-place and concat aliasing survive) and are as large as those allocations: declared reads
    seeded, every other byte F.  With F = NaN and F = 0, no byte outside the declared writes may change, and the declared outputs must be
    bit-identical between the two fills."""
    ctx = fp.Ctx(lib)
    uniq = {}
    for r in recorded.all():
        live, allocs = sorted(r.rec.blocks), sorted({(a, n) for _, a, n in r.rec.allocs})
        for e in so.executed(r.rec.log):
            if isinstance(e, so.Launch) and e.src == "lib":
                key = lc.launch_key(e.name, lc.argkinds(e.name), e.args)
                uniq.setdefault(key, (e.name, e.args, live, allocs))
    failures, kinds = [], set()
    for name, args, live, allocs in uniq.values():
        kinds.add(name)
        try:
            failures += _replay(lib, ctx, name, args, live, allocs)
        except (AssertionError, RuntimeError) as err:
            failures.append(f"{name}: {str(err).splitlines()[0]}")
    torch.cuda.empty_cache()
    for f in failures[:30]:
        print("  FAIL", f)
    print(f"\nfootprint validation: {len(uniq)} unique launches of {len(kinds)} kinds replayed with undeclared bytes NaN and 0")
    assert not failures, f"{len(failures)} footprint failures"
    assert set(kinds) >= {"dp_conv2d_wgrad", "dp_groupnorm_bwd_param", "dp_softmax_fwd", "dp_softmax_bwd", "dp_ssim", "dp_vq_quantize"}


def test_print_table():
    if ROWS:
        print("\nplan                               launches   side  ordered conflicting pairs  waits ordering no conflict")
        for r in ROWS:
            print(f"{r[0]:34s} {r[1]:8d} {r[2]:6d} {r[3]:25d} {r[4]:27d}")
