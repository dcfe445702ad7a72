"""prune_ldm.py's and sample_for_FID.py's loops sharded over two ranks against the same loops in one process, on the tiny LDM:

* two gloo processes sharing one GPU (the rounds, draws and collectives of the multi-GPU path, on one H100), and
* two NCCL processes on two GPUs (skipped with fewer).

Every rank seeds `random` and its generator differently; the single-process runs use rank 0's seeds.  LDMPruneScorer.run: taylor over an
odd number of iterations, diff-pruning with the stop on rank 1's iteration of the third round, and the encode_samples loop: the losses and stopped_at equal the
single-process run's, the accumulated gradient is within 1e-6 relative L2 of it and identical on both ranks.  sample_for_fid over an odd
number of batches with eta 0.5, PNG files and FID moments: the union of the files equals the single-process run's, names and bytes; mu and
sigma are within 1e-10 relative of it and identical on both ranks."""
import datetime
import hashlib
import os
import random
import sys
import traceback

import numpy as np
import pytest
import torch

from test_ldm_shard_host import _collect

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED_RANDOM, SEED_GEN = 4321, 31


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200 import _lib as L
    return L.load()


def _seeds(rank):
    random.seed(SEED_RANDOM + 7919 * rank)
    return SEED_GEN + 104729 * rank


def _prune(ld, pruner, iterations, rank, shard, encode=False):
    """LDMPruneScorer.run sharded (shard=True, this rank's seeds) or in this process alone (rank 0's seeds): losses, stopped_at, gradient."""
    from diff_pruning_b200.ldm_sampling import LDMPruneScorer
    unet = ld.model.diffusion_model
    unet.zero_grad()
    sc = LDMPruneScorer(ld, n_samples_per_class=2, ddim_steps=4, scale=3.0, encode_samples=encode)
    g = torch.Generator().manual_seed(_seeds(rank if shard else 0))
    losses = sc.run(pruner, iterations=iterations, generator=g, shard=shard)
    torch.cuda.synchronize()
    return losses.tolist(), sc.stopped_at, torch.cat([p.grad.flatten() for p in unet.parameters()]).cpu().numpy()


def _boost_for_stop_at(losses, j):
    """A factor for loss j - 1 that makes diff-pruning (loss / max_loss < 0.1) stop at iteration j: F * losses[j - 1] = 15 losses[j]
    becomes the running maximum, and losses[j] is a fifteenth of it.  Checked on PruneLDMStopRule over the boosted sequence."""
    from diff_pruning_b200.ldm_sampling import PruneLDMStopRule
    F = 15 * losses[j] / losses[j - 1]
    rule = PruneLDMStopRule("diff-pruning")
    stops = [rule.stop(l * F if i == j - 1 else l) for i, l in enumerate(losses)]
    assert stops.index(True) == j, (losses, F, stops)
    return F


def _prune_cases(rank):
    from diff_pruning_b200.ldm_sampling import PruneLDMStopRule
    from test_ldm_criterion_gpu import _tiny
    from test_ldm_sampling_gpu import _tiny_ld
    out = {}
    ld = _tiny_ld()
    out["taylor, 5 iterations"] = (_prune(ld, "taylor", 5, rank, True), _prune(ld, "taylor", 5, rank, False))
    j = 5                   # W = 2: rank 1 of the third of four rounds, after iterations 0-4 accumulated on both ranks
    F = _boost_for_stop_at(_prune(ld, "taylor", j + 1, rank, False)[0], j)
    orig = PruneLDMStopRule.stop

    def boosted(self, loss):
        n = self.__dict__.setdefault("_seen", 0)
        self._seen = n + 1
        return orig(self, loss * F if n == j - 1 else loss)
    PruneLDMStopRule.stop = boosted
    try:
        got = (_prune(ld, "diff-pruning", 8, rank, True), _prune(ld, "diff-pruning", 8, rank, False))
    finally:
        PruneLDMStopRule.stop = orig
    assert got[1][1] == j, (got[1][1], j)
    out[f"diff-pruning, stop at {j}"] = got
    ld = _tiny()
    out["taylor + encode, 3 iterations"] = (_prune(ld, "taylor", 3, rank, True, encode=True), _prune(ld, "taylor", 3, rank, False, encode=True))
    return out


def _fid_case(rank, tmp):
    from diff_pruning_b200.ldm_sampling import sample_for_fid
    from test_fid_gpu import seeded_model
    from test_vq_decoder_gpu import _tiny_ldm
    model, inc = _tiny_ldm(), seeded_model((3,))
    kw = dict(classes=[3, 11, 5], ipc=6, batch_size=2, ddim_steps=4, eta=0.5, decode_batch=2, inception=inc)     # 9 batches
    res = {}
    for shard in (True, False):
        seed = _seeds(rank if shard else 0)
        out_dir = os.path.join(tmp, "sharded" if shard else f"single{rank}")
        mu, sigma, n = sample_for_fid(model, out_dir=out_dir, generator=torch.Generator(device="cuda").manual_seed(seed), shard=shard, **kw)
        res[shard] = (mu, sigma, n)
    (mu, sigma, n), (mu1, sigma1, n1) = res[True], res[False]
    digest = hashlib.sha256(mu.tobytes() + sigma.tobytes()).hexdigest()
    rel = max(np.abs(mu - mu1).max() / np.abs(mu1).max(), np.abs(sigma - sigma1).max() / np.abs(sigma1).max())
    return {"n_files": (n, n1), "digest": digest, "rel": float(rel)}


def _worker(rank, world, backend, port, tmp, q):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    dev = rank if backend == "nccl" else 0
    torch.cuda.set_device(dev)
    kw = {"device_id": torch.device("cuda", dev)} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300), **kw)
    try:
        out = {"prune": _prune_cases(rank), "fid": _fid_case(rank, tmp)}
    except Exception:
        q.put((rank, traceback.format_exc()))
        raise
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def _rel_l2(a, b):
    return float(np.linalg.norm(a.astype(np.float64) - b) / np.linalg.norm(b.astype(np.float64)))


@pytest.mark.parametrize("backend", ["gloo", "nccl"])
def test_sharded_ldm_loops_equal_one_process(lib, backend, tmp_path):
    import torch.multiprocessing as mp
    if backend == "nccl" and torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 35500 + (os.getpid() % 2000) + (7 if backend == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, backend, port, str(tmp_path), q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = _collect(q, procs, 1200)
        for p in procs:
            p.join(120)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    errors = [v for v in results.values() if isinstance(v, str)]
    assert not errors, errors[0]
    assert len(results) == world, f"ranks {sorted(results)} reported, the others exited with {[p.exitcode for p in procs]}"
    assert all(p.exitcode == 0 for p in procs)
    r0, r1 = results[0], results[1]
    for name, ((losses, stopped_at, arena), (losses1, stopped_at1, arena1)) in r0["prune"].items():
        (o_losses, o_stopped, o_arena), _ = r1["prune"][name]
        err = _rel_l2(arena, arena1)
        print(f"\n{backend} {name}: losses {[f'{l:.6g}' for l in losses]}, stopped_at {stopped_at}, gradient rel L2 {err:.2e}")
        assert np.array_equal(np.float32(losses), np.float32(losses1)) and stopped_at == stopped_at1, (name, losses, losses1)
        assert np.array_equal(np.float32(o_losses), np.float32(losses)) and o_stopped == stopped_at, name
        assert err < 1e-6, (name, err)
        assert np.array_equal(arena, o_arena), f"{name}: the gradient differs between the ranks"
    assert len(r0["prune"]["taylor, 5 iterations"][0][0]) == 5
    f0, f1 = r0["fid"], r1["fid"]
    print(f"{backend} sample_for_fid: mu / sigma rel {f0['rel']:.2e} / {f1['rel']:.2e}")
    assert f0["n_files"] == f1["n_files"] == (18, 18)
    assert f0["digest"] == f1["digest"], "mu / sigma differ between the ranks"
    assert f0["rel"] < 1e-10 and f1["rel"] < 1e-10
    sharded, single = tmp_path / "sharded", tmp_path / "single0"
    names = sorted(os.listdir(single))
    assert sorted(os.listdir(sharded)) == names and len(names) == 18
    for f in names:
        assert (sharded / f).read_bytes() == (single / f).read_bytes(), f
