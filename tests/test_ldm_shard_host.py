"""Host (CPU gloo, W = 2 and 3) checks of how LDMPruneScorer.run shards prune_ldm.py's loop over ranks: the round-wise replay of the stop
rule against PruneLDMStopRule run sequentially on the same losses, and the inputs each rank's iterations get against the single-process
random stream, with every rank seeded differently.  The per-iteration GPU work (sample, forward + loss, backward) is replaced by a stub
that returns a preset loss and adds a known per-iteration "gradient"; run()'s rounds, draws and collectives are the real ones."""
import datetime
import os
import random
import sys
import traceback
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, S, SHAPE, LOSS_SHAPE, ARENA = 3, 2, (2, 4, 4), (3, 2, 2, 2), 16
SEED_RANDOM, SEED_GEN = 1234, 99

NAN = float("nan")
# (pruner, iterations, eta, losses); iteration t's loss is losses[t]
CASES = {
    "diff-pruning, stop on a round's first rank": ("diff-pruning", 8, 0.0, [1.0, 2.0, 1.5, 1.2, 0.9, 0.8, 0.19, 0.01]),
    "diff-pruning, stop on a later rank": ("diff-pruning", 8, 0.5, [1.0, 2.0, 1.5, 1.2, 0.21, 0.199, 0.4, 0.3]),
    "diff-pruning, stop in the final partial round": ("diff-pruning", 7, 0.0, [1.0, 2.0, 1.5, 1.2, 0.9, 0.8, 0.15]),
    "diff-pruning, exactly at the threshold": ("diff-pruning", 5, 0.0, [0.5, 1.0, 0.1, 0.09999999, 0.3]),
    "diff-pruning, NaN and zero losses": ("diff-pruning", 7, 0.0, [NAN, 0.0, 3.0, NAN, 0.31, 0.29, 1.0]),
    "taylor, never stops": ("taylor", 7, 0.5, [1.0, 0.0, 1e-9, NAN, 5.0, 1e-30, 2.0]),
    "diff0, never stops on non-negative losses": ("diff0", 7, 0.0, [1.0, 0.0, 1e-30, NAN, 0.5, 0.0, 2.0]),
    "diff0, stops on a negative loss": ("diff0", 6, 0.0, [1.0, 0.5, 0.2, -1e-6, 0.1, 0.1]),
    "fewer iterations than ranks": ("taylor", 2, 0.5, [1.0, 0.5]),
}


def _sequential(pruner, losses):
    """PruneLDMStopRule over the losses one at a time: (losses seen, stopped_at, iterations whose backward ran)."""
    from diff_pruning_b200.ldm_sampling import PruneLDMStopRule
    rule = PruneLDMStopRule(pruner)
    for t, loss in enumerate(losses):
        if rule.stop(loss):
            return losses[:t + 1], t, list(range(t))
    return list(losses), None, list(range(len(losses)))


def _grad(t):
    return torch.randn(ARENA, generator=torch.Generator().manual_seed(1000 + t))


def _stub(losses, eta):
    from diff_pruning_b200.ldm_sampling import LDMPruneScorer
    sc = LDMPruneScorer.__new__(LDMPruneScorer)
    sc.model = SimpleNamespace(cond_stage_key="class_label", get_learned_conditioning=lambda d: d["class_label"].float()[:, None, None])
    sc.unet = torch.nn.Linear(2, 2)
    sc.dev = torch.device("cpu")
    sc.B, sc.S, sc.eta, sc.shape, sc.loss_shape = B, S, eta, SHAPE, LOSS_SHAPE
    sc.ts, sc.stopped_at = None, None
    arena = torch.zeros(ARENA)
    seen = {}

    def forward(t, d, uc):
        assert torch.equal(uc, torch.full((B, 1, 1), 1000.0))
        seen[t] = {k: v.clone() for k, v in d.items()}
        sc._last = t
        return torch.tensor([losses[t]], dtype=torch.float32)

    def backward():
        arena.add_(_grad(sc._last))
    sc._forward, sc._backward, sc._grad_arena = forward, backward, (lambda uc: arena)
    return sc, arena, seen


def _sampler_for(rank):
    """A stateful class sampler whose labels differ between ranks: only rank 0's may reach the iterations."""
    k = iter(range(1 << 20))
    return lambda n: [(37 * next(k) + 11 * i + 100 * rank) % 1000 for i in range(n)]


def _expected_draws(iterations, eta, own_sampler):
    """The single-process stream: per iteration the labels, then x_T, the eta > 0 step noise and the q_sample noise on the generator."""
    random.seed(SEED_RANDOM)
    g = torch.Generator().manual_seed(SEED_GEN)
    sampler = _sampler_for(0) if own_sampler else (lambda n: random.sample(range(1000), n))
    out = []
    for _ in range(iterations):
        d = {"labels": torch.tensor(sampler(B), dtype=torch.long), "x_T": torch.randn((B,) + SHAPE, generator=g)}
        if eta > 0:
            d["step_noise"] = torch.stack([torch.randn((B,) + SHAPE, generator=g) for _ in range(S)])
        d["noise"] = torch.randn(LOSS_SHAPE, generator=g)
        out.append(d)
    return out


def _run_case(name, own_sampler, rank):
    pruner, iterations, eta, losses = CASES[name]
    sc, arena, seen = _stub(losses, eta)
    random.seed(SEED_RANDOM + 7919 * rank)                       # ranks seeded differently, as torchrun processes usually are
    g = torch.Generator().manual_seed(SEED_GEN + 104729 * rank)
    got = sc.run(pruner, iterations=iterations, class_sampler=_sampler_for(rank) if own_sampler else None, generator=g)
    return got, sc.stopped_at, arena, seen


def _worker(rank, world, port, q):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    torch.set_num_threads(1)
    out = {}
    try:
        for name in CASES:
            for own in (False, True):
                got, stopped_at, arena, seen = _run_case(name, own, rank)
                out[(name, own)] = (got.tolist(), stopped_at, arena.tolist(), {t: {k: v.tolist() for k, v in d.items()} for t, d in seen.items()})
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def _check(name, own, world, per_rank):
    pruner, iterations, eta, losses = CASES[name]
    want_losses, want_stop, used = _sequential(pruner, losses[:iterations])
    want_arena = sum((_grad(t) for t in used), torch.zeros(ARENA))
    draws = _expected_draws(iterations, eta, own)
    ran = {}
    for rank, (got, stopped_at, arena, seen) in per_rank.items():
        np.testing.assert_array_equal(np.float32(got), np.float32(want_losses), err_msg=f"{name}, rank {rank}")
        assert stopped_at == want_stop, (name, rank, stopped_at, want_stop)
        assert torch.allclose(torch.tensor(arena), want_arena, rtol=0, atol=1e-5), (name, rank)
        assert arena == per_rank[0][2], (name, rank, "the arena differs between ranks")
        for t, d in seen.items():
            assert t % world == rank, (name, rank, t)
            assert set(d) == set(draws[t]), (name, t, sorted(d))
            for k, v in d.items():
                assert torch.equal(torch.tensor(v, dtype=draws[t][k].dtype), draws[t][k]), (name, rank, t, k)
            ran[t] = rank
    last = want_stop if want_stop is not None else iterations - 1
    # every iteration up to the last one the rule looked at ran exactly once, on its rank; none after the round that stopped
    assert sorted(ran) == list(range(min(iterations, (last // world + 1) * world))), (name, sorted(ran))


def _collect(q, procs, limit):
    """{rank: result} from the workers; stops early when one reports an error or exits without reporting."""
    import queue
    import time
    results, end = {}, time.monotonic() + limit
    while len(results) < len(procs) and time.monotonic() < end:
        try:
            rank, v = q.get(timeout=2)
            results[rank] = v
            if isinstance(v, str):
                break
        except queue.Empty:
            if any(p.exitcode not in (None, 0) for p in procs):
                break
    return results


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_run_equals_the_sequential_rule_and_stream(world):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000) + world
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = _collect(q, procs, 300)
        for p in procs:
            p.join(60)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    errors = [v for v in results.values() if isinstance(v, str)]
    assert not errors, errors[0]
    assert len(results) == world, f"ranks {sorted(results)} reported, the others exited with {[p.exitcode for p in procs]}"
    assert all(p.exitcode == 0 for p in procs)
    for (name, own) in results[0]:
        _check(name, own, world, {r: results[r][(name, own)] for r in range(world)})


def test_single_process_run_is_the_sequential_rule():
    """Without a process group the same rounds are of one iteration: the sequential rule, the stream in order, the arena in order."""
    sys.path.insert(0, ROOT)
    for name in CASES:
        pruner, iterations, eta, losses = CASES[name]
        got, stopped_at, arena, seen = _run_case(name, False, 0)
        want_losses, want_stop, used = _sequential(pruner, losses[:iterations])
        np.testing.assert_array_equal(got.numpy(), np.float32(want_losses), err_msg=name)
        assert stopped_at == want_stop, name
        want_arena = torch.zeros(ARENA)
        for t in used:
            want_arena += _grad(t)
        assert torch.equal(arena, want_arena), name
        draws = _expected_draws(iterations, eta, False)
        assert sorted(seen) == list(range(len(want_losses)))
        for t, d in seen.items():
            assert all(torch.equal(d[k], draws[t][k]) for k in draws[t]) and set(d) == set(draws[t]), (name, t)


def test_stop_cases_land_where_their_names_say():
    """The synthetic sequences stop where the cases claim (so the W = 2 / 3 runs cover a stop on rank 0 and on later ranks of a round,
    one in a final partial round, and none)."""
    sys.path.insert(0, ROOT)
    stops = {name: _sequential(c[0], c[3][:c[1]])[1] for name, c in CASES.items()}
    assert stops["diff-pruning, stop on a round's first rank"] == 6                    # rank 0 for W = 2 and 3
    assert stops["diff-pruning, stop on a later rank"] == 5                            # rank 1 for W = 2, rank 2 for W = 3
    assert stops["diff-pruning, stop in the final partial round"] == 6                 # 7 iterations: a last round of one
    assert stops["diff-pruning, exactly at the threshold"] == 3                        # 0.1 / 1.0 is not < fp32(0.1); 0.09999999 is
    assert stops["diff-pruning, NaN and zero losses"] == 5
    assert stops["taylor, never stops"] is None and stops["diff0, never stops on non-negative losses"] is None
    assert stops["diff0, stops on a negative loss"] == 3
