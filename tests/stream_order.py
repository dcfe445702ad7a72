"""Stream-order audit: an event log of everything a plan enqueues (library launches with their stream, aten ops, stream / event waits,
host synchronisations, caching-allocator frees), happens-before over it by vector clocks, and three checks:

  1. cross-stream race: two accesses (footprint.py) that overlap in at least one byte, at least one of them a write, not both atomic-max
     commits of one amax slot, and neither ordered before the other;
  2. intra-launch aliasing: a read region of one operand overlapping a written region of another operand of the same launch, outside
     footprint.IN_PLACE;
  3. lifetime: no allocator block a side-stream launch touches is freed between that launch and the wait that orders it before the
     main stream.

Happens-before counts explicit orderings only: a.wait_stream(b) / wait_event orders everything enqueued on b so far before everything
enqueued on a afterwards (and nothing enqueued on b later); Event.record / wait likewise; a host synchronisation (device, stream or event
synchronize, .item(), a blocking device-to-host copy) orders everything enqueued before it on what it waited for.  The legacy default
stream's implicit barrier is not modelled: the GPU test asserts that every other stream the plans use is non-blocking, so there is none.
Checked on the host by test_stream_order_host.py, on the plans by test_stream_races_gpu.py.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import sys
import time
from typing import Dict, List, Optional

import numpy as np

import footprint as fp


# ------------------------------------------------------------------------------------------------------------------------ the log
class Launch:
    __slots__ = ("name", "args", "stream", "label", "accs", "src", "pos", "vc", "t_us")

    def __init__(self, name, args, stream, label="", accs=None, src="lib", t_us=0):
        self.name, self.args, self.stream, self.label, self.src, self.t_us = name, args, stream, label, src, t_us
        self.accs: List[fp.Access] = accs if accs is not None else []
        self.pos, self.vc = -1, None

    def __repr__(self):
        return f"#{self.pos} {self.name} [{self.label}] on stream {self.stream:#x}"


class Wait:
    """waiter.wait_stream(waited)."""
    __slots__ = ("waiter", "waited", "tag", "pos", "gain", "t_us")

    def __init__(self, waiter, waited, tag="", t_us=0):
        self.waiter, self.waited, self.tag, self.t_us = waiter, waited, tag, t_us
        self.pos, self.gain = -1, None

    def __repr__(self):
        return f"#{self.pos} wait {self.waiter:#x} <- {self.waited:#x} [{self.tag}]"


class Record:
    __slots__ = ("event", "stream", "pos", "t_us")

    def __init__(self, event, stream, t_us=0):
        self.event, self.stream, self.t_us, self.pos = event, stream, t_us, -1


class WaitEvent:
    __slots__ = ("stream", "event", "pos", "t_us")

    def __init__(self, stream, event, t_us=0):
        self.stream, self.event, self.t_us, self.pos = stream, event, t_us, -1


class Sync:
    """Host synchronisation: with stream None, the whole device; with event set, that event."""
    __slots__ = ("stream", "event", "what", "pos", "t_us")

    def __init__(self, stream=None, event=None, what="", t_us=0):
        self.stream, self.event, self.what, self.t_us, self.pos = stream, event, what, t_us, -1


class Mark:
    __slots__ = ("text", "pos", "t_us")

    def __init__(self, text, t_us=0):
        self.text, self.t_us, self.pos = text, t_us, -1


CAPTURE_BEGIN, CAPTURE_END = "capture>", "<capture"


def executed(log):
    """The events that execute where they stand: a CUDA-graph capture records its launches without running them (they run, remapped,
    at every replay, where the recorder appends them again)."""
    out, depth = [], 0
    for e in log:
        if isinstance(e, Mark) and e.text in (CAPTURE_BEGIN, CAPTURE_END):
            depth += 1 if e.text == CAPTURE_BEGIN else -1
        elif depth == 0:
            out.append(e)
    return out


def captured(log):
    """The spans recorded under CUDA-graph capture, as lists of events."""
    spans, cur = [], None
    for e in log:
        if isinstance(e, Mark) and e.text == CAPTURE_BEGIN:
            cur = []
        elif isinstance(e, Mark) and e.text == CAPTURE_END:
            spans.append(cur)
            cur = None
        elif cur is not None:
            cur.append(e)
    return spans


def number(log):
    for i, e in enumerate(log):
        e.pos = i
    return log


# ------------------------------------------------------------------------------------------------------------------ happens-before
def _join(a: Dict[int, int], b: Dict[int, int]):
    for k, v in b.items():
        if a.get(k, 0) < v:
            a[k] = v


def clocks(log):
    """Vector clocks: every launch gets vc (its stream's clock right after it, host orderings joined in); every Wait gets gain =
    (waited stream's component before, after), the launches of the waited stream the wait newly orders."""
    log = executed(log)
    clk: Dict[int, Dict[int, int]] = {}
    host: Dict[int, int] = {}
    ev: Dict[int, Dict[int, int]] = {}

    def cur(s):
        c = clk.setdefault(s, {})
        _join(c, host)
        return c
    for e in number(log):
        if isinstance(e, Launch):
            c = cur(e.stream)
            c[e.stream] = c.get(e.stream, 0) + 1
            e.vc = dict(c)
        elif isinstance(e, Wait):
            c, o = cur(e.waiter), cur(e.waited)
            before = c.get(e.waited, 0)
            _join(c, o)
            e.gain = (before, c.get(e.waited, 0))
        elif isinstance(e, Record):
            ev[e.event] = dict(cur(e.stream))
        elif isinstance(e, WaitEvent):
            _join(cur(e.stream), ev.get(e.event, {}))
        elif isinstance(e, Sync):
            if e.event is not None:
                _join(host, ev.get(e.event, {}))
            elif e.stream is not None:
                _join(host, cur(e.stream))
            else:
                for s in list(clk):
                    _join(host, cur(s))
    return log


def hb(a: Launch, b: Launch) -> bool:
    """a happens before b (both numbered and clocked)."""
    return a.pos < b.pos and a.vc[a.stream] <= b.vc.get(a.stream, 0)


# ------------------------------------------------------------------------------------------------------------------------- checks
class Race:
    def __init__(self, a, b, xa, xb, hit):
        self.a, self.b, self.xa, self.xb, self.hit = a, b, xa, xb, hit

    def __repr__(self):
        r = self.xa.region
        return (f"race: {self.a} {self.xa.field}:{self.xa.mode}  vs  {self.b} {self.xb.field}:{self.xb.mode}; "
                f"buffer {r.ptr:#x} (esz {r.esz}, ld {r.ld}), first overlap at row {self.hit[0]}, element {self.hit[1]}")


def _conflict_modes(ma: str, mb: str) -> bool:
    if ma == fp.A and mb == fp.A:        # atomic max commits into one slot commute
        return False
    return ma in fp.WRITES or mb in fp.WRITES


class Report:
    def __init__(self):
        self.races: List[Race] = []
        self.ordered = 0               # conflicting cross-stream pairs the waits order
        self.unused_waits: List[Wait] = []
        self.launches = self.side = 0


def check_races(log, side=(), limit: int = 50) -> Report:
    """Cross-stream races over a clocked log.  Candidate pairs come from a sweep over the accesses' byte ranges sorted by start; only
    pairs on different streams with conflicting modes are tested exactly (footprint.first_overlap) and then for happens-before."""
    log = clocks(log)
    rep = Report()
    launches = [e for e in log if isinstance(e, Launch)]
    rep.launches = len(launches)
    rep.side = sum(1 for e in launches if e.stream in side)
    items = [(e, x) for e in launches for x in e.accs]
    if not items:
        return rep
    sid = {s: i for i, s in enumerate(sorted({e.stream for e in launches}))}
    lo = np.array([x.region.lo for _, x in items], dtype=np.int64)
    hi = np.array([x.region.hi for _, x in items], dtype=np.int64)
    st = np.array([sid[e.stream] for e, _ in items], dtype=np.int64)
    wr = np.array([x.mode in fp.WRITES for _, x in items])
    at = np.array([x.mode == fp.A for _, x in items])
    order = np.argsort(lo, kind="stable")
    lo_s, hi_s = lo[order], hi[order]
    end = np.searchsorted(lo_s, hi_s, side="left")              # items k+1 .. end-1 start before item k ends
    cnt = np.maximum(end - np.arange(len(order)) - 1, 0)
    ia = np.repeat(np.arange(len(order)), cnt)
    ib = (np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)) + ia + 1
    a_idx, b_idx = order[ia], order[ib]
    keep = (st[a_idx] != st[b_idx]) & (wr[a_idx] | wr[b_idx]) & ~(at[a_idx] & at[b_idx])
    used = set()
    waits = [e for e in log if isinstance(e, Wait)]
    for i, j in zip(a_idx[keep].tolist(), b_idx[keep].tolist()):
        (ea, xa), (eb, xb) = items[i], items[j]
        if ea.pos > eb.pos:
            (ea, xa), (eb, xb) = (eb, xb), (ea, xa)
        if not _conflict_modes(xa.mode, xb.mode):
            continue
        hit = fp.first_overlap(xa.region, xb.region)
        if hit is None:
            continue
        if hb(ea, eb):
            rep.ordered += 1
            own = ea.vc[ea.stream]
            for w in waits:
                if w.waited == ea.stream and ea.pos < w.pos < eb.pos and w.gain[0] < own <= w.gain[1]:
                    used.add(w.pos)
        elif len(rep.races) < limit:
            rep.races.append(Race(ea, eb, xa, xb, hit))
    rep.unused_waits = [w for w in waits if w.pos not in used]
    return rep


def check_aliasing(log) -> List[str]:
    out = []
    for e in executed(log):
        if isinstance(e, Launch) and e.src == "lib":
            for rf, wf, hit in fp.aliasing(e.name, e.accs):
                out.append(f"{e}: read operand {rf} overlaps written operand {wf} at row {hit[0]}, element {hit[1]}")
    return out


def check_lifetime(log, frees, side) -> List[str]:
    """frees: [(t_us, addr, size)] of caching-allocator blocks.  Every launch on a side stream must keep its regions allocated until the
    first later wait or synchronisation that orders it before another stream (or the host).  Only frees are looked at: the allocator
    hands a block out again only after it was freed, so a block handed out again inside the window was freed inside it.  The frees are
    placed in the log's order by time: the allocator's trace and the log both stamp host wall-clock microseconds (the GPU test checks
    that every free of the trace falls inside the recording), so a free within a microsecond or so of a wait is placed approximately."""
    log = clocks(log)
    out = []
    if not frees:
        return out
    f = np.array(frees, dtype=np.int64).reshape(-1, 3)
    joins = [e for e in log if isinstance(e, (Wait, Sync))]
    for e in log:
        if not isinstance(e, Launch) or e.stream not in side:
            continue
        own = e.vc[e.stream]
        t_end = None
        for j in joins:
            if j.pos <= e.pos:
                continue
            if isinstance(j, Wait) and j.waited == e.stream and j.gain[1] >= own:
                t_end = j.t_us
                break
            if isinstance(j, Sync) and (j.stream is None or j.stream == e.stream):
                t_end = j.t_us
                break
        t_end = t_end if t_end is not None else sys.maxsize
        for x in e.accs:
            r = x.region
            sel = (f[:, 0] >= e.t_us) & (f[:, 0] < t_end) & (f[:, 1] < r.hi) & (f[:, 1] + f[:, 2] > r.lo)
            if sel.any():
                k = int(np.argmax(sel))
                out.append(f"{e} {x.field}: block {f[k, 1]:#x} (+{f[k, 2]}) freed at {f[k, 0]} us, before the wait that orders the "
                           f"launch ({t_end} us)")
    return out


# ------------------------------------------------------------------------------------------------------------------------ recorder
def _label(depth: int = 3) -> str:
    """`what` of the plan step that made this call (engine.Plan._rec closures keep it as a local), else ''."""
    f = sys._getframe(depth)
    for _ in range(4):
        if f is None:
            break
        w = f.f_locals.get("what")
        if isinstance(w, str):
            return w
        f = f.f_back
    return ""


def _info(name, args) -> str:
    a = args[0] if len(args) == 1 and hasattr(args[0], "_fields_") else None
    if a is not None and hasattr(a, "R") and hasattr(a, "P"):
        return f"{a.C}->{a.K} {a.R}x{a.S}" + (f" s{a.stride}" if a.stride != 1 else "") + f" @{a.P}x{a.Q}"
    return ""


def tensor_region(t) -> fp.Region:
    """Byte footprint of a CUDA tensor: exact for contiguous tensors and [rows][ld] row patterns, else its bounding range."""
    esz, n = t.element_size(), t.numel()
    if t.is_contiguous():
        return fp.flat(t.data_ptr(), n, esz)
    if t.dim() >= 2 and t.stride(-1) == 1:
        s = [d for d in zip(t.shape[:-1], t.stride()[:-1]) if d[0] > 1]
        if len(s) <= 1:
            rows, ld = (s[0] if s else (1, t.shape[-1]))
            return fp.view(t.data_ptr(), rows, ld, t.shape[-1], esz)
    span = 1 + sum((d - 1) * st for d, st in zip(t.shape, t.stride()))
    return fp.flat(t.data_ptr(), span, esz)


class Recorder:
    """Context manager: while active, every library launch (through launch_census.wrap_launches), aten op on a CUDA tensor, stream /
    event wait, Event.record and host synchronisation is appended to self.log; caching-allocator frees come from torch's memory
    history (self.frees).  Nothing is reordered or delayed: the log is the host's enqueue order."""

    NO_KERNEL = ("empty.memory_format", "empty_strided.default", "empty_like.default", "set_.source_Storage_storage_offset",
                 "record_stream.default", "lift_fresh.default", "_has_compatible_shallow_copy_type.default", "resize_.default")

    def __init__(self, lib, ctx: Optional[fp.Ctx] = None, aten: bool = True, memory: bool = True):
        self.lib, self.ctx = lib, ctx or fp.Ctx(lib)
        self.log: list = []
        self.frees: list = []
        self.blocks: list = []
        self.allocs: list = []
        self.aten, self.memory = aten, memory
        self._busy = 0
        self._events: Dict[int, int] = {}
        self._capture, self._graphs, self._replays = None, {}, 0

    @staticmethod
    def now() -> int:
        return time.time_ns() // 1000

    def mark(self, text):
        self.log.append(Mark(text, self.now()))

    # ---- library launches
    def _on_launch(self, name, args, stream):
        self.log.append(Launch(name, args, int(stream or 0), " ".join(x for x in (_label(3), _info(name, args)) if x),
                               fp.footprint(name, args, self.ctx), "lib", self.now()))

    # ---- aten ops
    def _on_aten(self, func, args, kwargs, out):
        import torch
        name = func._schema.name.split("::")[-1] + "." + (func._overloadname or "default")
        if func.is_view or name in self.NO_KERNEL:
            return
        accs, cuda = [], False
        sch = func._schema.arguments
        flat_args = list(args) + [kwargs.get(a.name) for a in sch[len(args):]]
        for a, v in zip(sch, flat_args):
            for t in (v if isinstance(v, (list, tuple)) else [v]):
                if isinstance(t, torch.Tensor) and t.is_cuda and t.numel():
                    cuda = True
                    w = a.alias_info is not None and a.alias_info.is_write
                    accs.append(fp.Access(a.name, tensor_region(t), fp.RW if w else fp.R, "aten"))
        outs = out if isinstance(out, (list, tuple)) else [out]
        written = {x.region.ptr for x in accs if x.mode == fp.RW}
        host_out = False
        for t in outs:
            if isinstance(t, torch.Tensor):
                if t.is_cuda and t.numel() and t.data_ptr() not in written:
                    cuda = True
                    accs.append(fp.Access("out", tensor_region(t), fp.W, "aten"))
                elif not t.is_cuda:
                    host_out = True
        if not cuda:
            return
        s = torch.cuda.current_stream().cuda_stream
        self.log.append(Launch("aten." + name, None, s, "", accs, "aten", self.now()))
        if name.startswith("_local_scalar_dense") or (host_out and any(x.mode == fp.R for x in accs)):
            self.log.append(Sync(s, what="aten." + name, t_us=self.now()))

    @contextlib.contextmanager
    def _patched(self):
        import torch
        from torch.utils._python_dispatch import TorchDispatchMode
        rec = self
        saved = []

        def patch(obj, attr, make):
            orig = getattr(obj, attr)
            saved.append((obj, attr, orig))
            setattr(obj, attr, make(orig))

        def guard(orig, before=None, after=None):
            def f(*a, **k):
                if rec._busy:
                    return orig(*a, **k)
                rec._busy += 1
                try:
                    if before:
                        before(*a, **k)
                    r = orig(*a, **k)
                    if after:
                        after(r, *a, **k)
                    return r
                finally:
                    rec._busy -= 1
            return f

        def sid(s):
            return int(s.cuda_stream) if s is not None else torch.cuda.current_stream().cuda_stream

        def wait_tag():
            f = sys._getframe(3)
            return f"{f.f_code.co_name}:{f.f_lineno}" if f else ""

        def eid(ev):
            return self._events.setdefault(id(ev), len(self._events) + 1)
        patch(torch.cuda.Stream, "wait_stream", lambda o: guard(o, before=lambda self_, other: rec.log.append(
            Wait(sid(self_), sid(other), wait_tag(), rec.now()))))
        patch(torch.cuda.Stream, "wait_event", lambda o: guard(o, after=lambda r, self_, ev: rec.log.append(
            WaitEvent(sid(self_), eid(ev), rec.now()))))
        patch(torch.cuda.Stream, "record_event", lambda o: guard(o, after=lambda ev, self_, event=None: rec.log.append(
            Record(eid(ev), sid(self_), rec.now()))))
        patch(torch.cuda.Event, "record", lambda o: guard(o, after=lambda r, ev, stream=None: rec.log.append(
            Record(eid(ev), sid(stream), rec.now()))))
        patch(torch.cuda.Event, "wait", lambda o: guard(o, after=lambda r, ev, stream=None: rec.log.append(
            WaitEvent(sid(stream), eid(ev), rec.now()))))
        patch(torch.cuda.Event, "synchronize", lambda o: guard(o, after=lambda r, ev: rec.log.append(
            Sync(event=eid(ev), what="event", t_us=rec.now()))))
        patch(torch.cuda.Stream, "synchronize", lambda o: guard(o, after=lambda r, self_: rec.log.append(
            Sync(sid(self_), what="stream", t_us=rec.now()))))
        patch(torch.cuda, "synchronize", lambda o: guard(o, after=lambda r, device=None: rec.log.append(
            Sync(None, what="device", t_us=rec.now()))))

        def begin(g, *a, **k):
            rec._capture = (id(g), torch.cuda.current_stream().cuda_stream, len(rec.log) + 1)
            rec.mark(CAPTURE_BEGIN)

        def end(r, g, *a, **k):
            gid, cs, i0 = rec._capture
            rec._graphs[gid] = (cs, rec.log[i0:])
            rec.mark(CAPTURE_END)
            rec._capture = None

        def replay(g, *a, **k):
            cs, body = rec._graphs[id(g)]
            rec._replays += 1
            s = torch.cuda.current_stream().cuda_stream
            branch = lambda x: s if x == cs else -(rec._replays << 20 | (x & 0xFFFFF))   # forked branches: streams of this replay
            for e in body:
                if isinstance(e, Launch):
                    rec.log.append(Launch(e.name, e.args, branch(e.stream), e.label, e.accs, e.src, rec.now()))
                elif isinstance(e, Wait):
                    rec.log.append(Wait(branch(e.waiter), branch(e.waited), e.tag, rec.now()))
        patch(torch.cuda.CUDAGraph, "capture_begin", lambda o: guard(o, before=begin))
        patch(torch.cuda.CUDAGraph, "capture_end", lambda o: guard(o, after=end))
        patch(torch.cuda.CUDAGraph, "replay", lambda o: guard(o, before=replay))

        class Aten(TorchDispatchMode):
            def __torch_dispatch__(self, func, types, args=(), kwargs=None):
                out = func(*args, **(kwargs or {}))
                if not rec._busy:
                    rec._on_aten(func, args, kwargs or {}, out)
                return out
        import launch_census as lc
        try:
            with lc.wrap_launches(self.lib, self._on_launch):
                if self.aten:
                    with Aten():
                        yield
                else:
                    yield
        finally:
            for obj, attr, orig in reversed(saved):
                setattr(obj, attr, orig)

    @contextlib.contextmanager
    def record(self):
        import torch
        if self.memory:
            torch.cuda.memory._record_memory_history(enabled="all", context=None, stacks="python", max_entries=2_000_000)
        self.t0 = self.now()
        try:
            with self._patched():
                yield self
        finally:
            self.t1 = self.now()
            if self.memory:
                snap = torch.cuda.memory._snapshot()
                dev = torch.cuda.current_device()
                for t in snap["device_traces"][dev]:
                    if t["action"] in ("free_requested", "free_completed", "segment_free"):
                        self.frees.append((int(t.get("time_us", 0)), int(t["addr"]), int(t["size"])))
                    elif t["action"] == "alloc":
                        self.allocs.append((int(t.get("time_us", 0)), int(t["addr"]), int(t["size"])))
                # the allocations alive at the end of the recording: every pointer a launch of the plans used lies in one of them
                self.blocks = sorted((int(b["address"]), int(b["size"])) for seg in snap["segments"] for b in seg["blocks"]
                                     if b["state"].startswith("active"))
                torch.cuda.memory._record_memory_history(enabled=None)


# ------------------------------------------------------------------------------------------------------------------ stream facts
def _cudart():
    import glob
    import os
    import torch
    here = os.path.dirname(os.path.dirname(torch.__file__))
    for p in glob.glob(os.path.join(here, "nvidia", "cuda_runtime", "lib", "libcudart.so*")) + ["libcudart.so.12", "libcudart.so"]:
        try:
            return C.CDLL(p)
        except OSError:
            continue
    return None


def stream_nonblocking(handle: int) -> bool:
    """cudaStreamGetFlags(handle) has cudaStreamNonBlocking: no implicit barrier with the legacy default stream."""
    rt = _cudart()
    assert rt is not None, "libcudart not found: cannot check the stream flags"
    flags = C.c_uint(0)
    rc = rt.cudaStreamGetFlags(C.c_void_p(handle), C.byref(flags))
    assert rc == 0, f"cudaStreamGetFlags: error {rc}"
    return bool(flags.value & 1)


def canonical(log):
    """The log as a sequence comparable across runs of the same plan: streams renamed by first appearance, times and numbering dropped."""
    names: Dict[int, int] = {}

    def n(s):
        return None if s is None else names.setdefault(s, len(names))
    out = []
    for e in log:
        if isinstance(e, Launch):
            out.append(("launch", e.name, n(e.stream), tuple(x[:3] for x in e.accs)))
        elif isinstance(e, Wait):
            out.append(("wait", n(e.waiter), n(e.waited)))
        elif isinstance(e, Sync):
            out.append(("sync", n(e.stream), e.what))
    return out
