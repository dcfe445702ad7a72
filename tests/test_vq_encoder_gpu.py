"""The encode side of the LDM's VQ first stage on the device: the encoder plan against the reference Encoder / VQModelInterface.encode
(tests/golden/vq_encoder_tiny.pt) and against the float64 oracle at 256 x 256, the launch census of every distinct encoder launch, the
amax-slot audit, NaN-poisoned plans, graph against eager, micro-batch chunking, and the decode(encode(x)) round trip.

Bounds: 1e-4 max-rel is the project's fp32-grade bound for a whole network (BASELINE.json north star), which the decoder tests use too;
the census holds every launch to the chain-length error model of launch_census.py."""
import gc

import pytest
import torch

from conftest import max_rel
import vq_encoder_oracle as eo
from oracle import vq_oracle as vo
from test_vq_encoder_host import GOLD, seeded_vq

pytestmark = pytest.mark.gpu


def S():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as ge
    ge.build()
    from diff_pruning_b200 import _lib as L
    return L.load()


def _vq_f4(seed=3):
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG, VQModelInterface
    torch.manual_seed(seed)
    return VQModelInterface(**VQ_F4_CONFIG, with_encoder=True).eval()


def _images(n, hw, seed):
    return torch.rand(n, 3, hw, hw, generator=torch.Generator().manual_seed(seed)) * 2 - 1


@pytest.mark.parametrize("name", list(GOLD["configs"]))
def test_encoder_plan_matches_reference_encode(lib, name):
    c = GOLD["configs"][name]
    m = seeded_vq(name).cuda()
    got = m.encode(c["x"].cuda())
    err = max_rel(got, c["encoded"])
    print(f"{name}: max-rel {err:.2e} against the reference VQModelInterface.encode")
    assert tuple(got.shape) == tuple(c["encoded"].shape) and err < 1e-4


def test_vq_f4_256px_batch8_encode_matches_float64_oracle(lib):
    m = _vq_f4()
    x = _images(8, 256, 8)
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG
    sd64 = {k: v.detach().double().cuda() for k, v in m.state_dict().items()}
    with torch.no_grad():
        want = eo.encode(sd64, VQ_F4_CONFIG["ddconfig"], x.double().cuda())
    del sd64
    m = m.cuda()
    got = m.encode(x.cuda())
    err = max_rel(got, want)
    plan = m.__dict__["_dpb200_encode"].plan
    print(f"VQ-f4 encode 256px b8: max-rel {err:.2e} against fp64; plan bytes at micro-batch 8: {plan.bytes_allocated() / 2 ** 30:.2f} GiB")
    assert tuple(got.shape) == (8, 3, 64, 64) and err < 1e-4


def test_encode_in_chunks_and_graph_equal_separate_and_eager(lib):
    """11 images at micro-batch 8 = the first 8 and the last 3 encoded on their own (the tail chunk is zero-padded); the graph run equals
    the eager launch list."""
    m = _vq_f4().cuda()
    x = _images(11, 64, 9).cuda()
    all11 = m.encode(x)
    parts = torch.cat([m.encode(x[:8]), m.encode(x[8:])])
    assert torch.equal(all11, parts)
    m.use_graph = False
    assert torch.equal(all11, m.encode(x))


def test_encoder_plan_is_bit_identical_under_poisoned_allocations(lib):
    """Every torch.empty* filled with NaN, 1e30 or 0 before the code writes it: the same bits; and a graph captured from a plan built under
    NaN equals the eager launch list of a plan built under 0."""
    from test_pruned_widths_host import poisoned_alloc
    x = _images(3, 64, 10).cuda()
    outs = []
    for v, graph in ((float("nan"), True), (1e30, True), (0.0, True), (0.0, False)):
        m = _vq_f4().cuda()
        m.encode_batch = 4
        m.use_graph = graph
        with poisoned_alloc(v) as cnt:
            outs.append(m.encode(x))
        assert cnt.n > 0
        del m
        gc.collect()
        torch.cuda.empty_cache()
    assert bool(torch.isfinite(outs[2]).all())
    assert all(torch.equal(o, outs[2]) for o in outs)


# ---------------------------------------------------------------------------------------------------------------------- census, audit
def _encode_runs():
    """VQ-f4 at 256 x 256 (tensor-core attention over 4096 tokens) and the small config (SIMT attention), batch 2, eager."""
    out = []
    for m, x in ((_vq_f4(), _images(2, 256, 11)), (seeded_vq("tiny"), _images(2, 16, 12))):
        m = m.cuda()
        m.use_graph = False
        m.encode_batch = 2
        out.append((m, x.cuda()))
    return out


def test_vq_encoder_census(lib):
    """Every distinct launch of the two encodes, replayed on fresh seeded buffers and checked against float64 (bounds of
    launch_census.py) or bit for bit."""
    from test_eval_census_gpu import EVAL_REPLAY, _LOG
    from test_launch_census_gpu import _capture, _unique
    _LOG.clear()
    _LOG.update(geoms=set(), tc=[], simt=set())
    runs = _encode_runs()

    def run():
        for m, x in runs:
            m.encode(x)
    calls = _capture(lib, run)
    del runs
    gc.collect()
    torch.cuda.empty_cache()
    kinds = {n for n, _ in calls}
    assert {"dp_conv2d_fprop", "dp_groupnorm_fwd", "dp_gemm_nt_tc", "dp_gemm_batched", "dp_nchw_to_nhwc", "dp_nhwc_to_nchw"} <= kinds
    missing = kinds - set(EVAL_REPLAY)
    assert not missing, f"launch kinds without a replay: {sorted(missing)}"
    strided = [a[0] for n, a in calls if n == "dp_conv2d_fprop" and a[0].stride == 2]
    assert [(a.pad_t, a.pad_l, 2 * a.P == a.H) for a in strided] == [(0, 0, True)] * 3     # VQ-f4's two Downsamples, the small config's one
    rep, failures = {}, []
    g = torch.Generator().manual_seed(2027)
    uniq = _unique(calls)
    for name, args in uniq:
        try:
            EVAL_REPLAY[name](lib, g, name, args[0] if len(args) == 1 else args, rep)
        except AssertionError as e:
            failures.append(f"{name}: {e}".splitlines()[0])
        torch.cuda.synchronize()
    for f in failures:
        print("  FAIL", f)
    assert not failures
    assert set(rep) == kinds
    print(f"\nVQ encoder census: {len(calls)} launches, {len(uniq)} unique, {len(kinds)} kinds")
    for name in sorted(rep):
        print(f"  {name:26s} worst err/bound {max(rep[name]):.3f}")


def test_encoder_amax_slots_bound_their_operands(lib):
    import launch_census as lc
    import slot_audit as sa
    from test_slot_audit_gpu import ATTN, FWD, MAX_LOOSENESS
    runs = _encode_runs()
    audit = sa.SlotAudit()
    with lc.wrap_launches(lib, audit):
        for m, x in runs:
            m.encode(x)
        torch.cuda.synchronize()
    worst, where = audit.worst()
    print(f"\nVQ encoders: {audit.launches} launches name an input slot, {audit.audited} audited ({audit.simt} SIMT), "
          f"{len(audit.failures)} below the maximum; worst looseness {worst:.4g} at {where}")
    assert not audit.failures, audit.failures[:3]
    assert audit.audited > 0 and audit.audited + audit.simt == audit.launches
    assert (FWD | ATTN) <= audit.kinds
    assert worst <= MAX_LOOSENESS


# ---------------------------------------------------------------------------------------------------------------------- round trip
def test_round_trip_matches_the_oracles_round_trip(lib):
    """decode(encode(x)) for VQ-f4 at 64 x 64 (batch 4) with a codebook spread over the latents' range.  The codes the engine's
    dp_vq_quantize picks for its own latents agree with the fp64 oracle's codes for the oracle's latents, except where the oracle's two
    fp64 distances are closer than the engine's latent error can move them (|d(z, a) - d(z, b)| <= 2 |dz| |e_a - e_b|).  The images
    agree with the oracle's round trip on every image whose codes all agree, and with the oracle decoding the engine's latents on all."""
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG
    m = _vq_f4(5)
    x = _images(4, 64, 13)
    cfg = VQ_F4_CONFIG["ddconfig"]
    with torch.no_grad():
        sd64 = {k: v.detach().double().cuda() for k, v in m.state_dict().items()}
        z64 = eo.encode(sd64, cfg, x.double().cuda())
        r = float(z64.abs().max())
        g = torch.Generator().manual_seed(14)
        code = (torch.rand(8192, 3, generator=g) * 2 - 1) * r
        m.quantize.embedding.weight.copy_(code)
        sd64["quantize.embedding.weight"] = code.double().cuda()
        want = vo.decode(sd64, cfg, z64)
        _, idx64 = vo.quantize(z64, sd64["quantize.embedding.weight"])
    m = m.cuda()
    z = m.encode(x.cuda())
    run = m.decode_chunk(z, indices=True)
    idx = run.indices[:4].clone()
    got = m.decode(z)
    with torch.no_grad():
        want_own = vo.decode(sd64, cfg, z.double())
    diff = (idx != idx64).nonzero()
    n_diff = int(diff.shape[0])
    if n_diff:
        zf = z64.permute(0, 2, 3, 1)[diff[:, 0], diff[:, 1], diff[:, 2]]
        dz = (z.double().permute(0, 2, 3, 1) - z64.permute(0, 2, 3, 1))[diff[:, 0], diff[:, 1], diff[:, 2]].norm(dim=1)
        e = code.double().cuda()
        a, b = e[idx[idx != idx64]], e[idx64[idx != idx64]]
        gap = ((zf - a) ** 2).sum(1) - ((zf - b) ** 2).sum(1)
        assert bool((gap <= 2 * dz * (a - b).norm(dim=1) + 1e-300).all()), n_diff
    same = [i for i in range(4) if torch.equal(idx[i], idx64[i])]
    err_own = max_rel(got, want_own)
    err = max_rel(got[same], want[same]) if same else 0.0
    print(f"round trip: {n_diff} of {idx.numel()} codes differ from the oracle's (all near ties); images max-rel {err:.2e} on the "
          f"{len(same)} images with identical codes, {err_own:.2e} against the oracle decoding the engine's latents; latent max-rel "
          f"{max_rel(z, z64):.2e}")
    assert len(same) >= 2 and err < 1e-4 and err_own < 1e-4
