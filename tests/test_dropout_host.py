"""The finetune's dropout masks on the host: the engine's seed schedule, and the masks it gives restated bit for bit
(tests/dropout_mask.py) and tested for independence.

A mask that restates the kernel reproduces a fault in the hash instead of catching it, so these tests are statistical: for pairs of
masks the plan draws (every pair of layers within one step, one layer at consecutive steps and on two data-parallel ranks, the
channel parts of a split layer) the number of elements dropped by both, at relative shifts of -16 .. 16 elements, must be the
binomial q^2 n of independent masks within 6 sigma; and within one mask the keep rate per element position and channel, and the
joint keep rates of neighbouring elements and of the four fields of one hash word, must be those of independent draws."""
import math

import numpy as np
import pytest

import dropout_mask as dm
import diff_pruning_b200 as dp
from diff_pruning_b200.models import ResnetBlock2D
from diff_pruning_b200.engine import _dropout_seed, dropout_layer_seed

N_ELEM = 3 << 20        # elements compared per pair of masks
P = 0.1                 # the finetune's dropout (finetune_ddpm_cifar10.sh --dropout 0.1)
SIGMA = 6.0


def _n_dropout_layers(cfg) -> int:
    """Dropout GroupNorms of the finetune plan of `cfg`: one per ResnetBlock2D (its norm2 carries the block's dropout)."""
    return sum(isinstance(m, ResnetBlock2D) for m in dp.UNet2DModel(**cfg).modules())


@pytest.fixture(scope="module")
def c1_layers():
    n = _n_dropout_layers(dp.CIFAR10_DDPM_CONFIG)
    assert n == 22                      # 4 levels x 2 down, 2 mid, 4 levels x 3 up
    return n


def _drops(layer, part=0, step=1, rank=0, p=P, n=N_ELEM, mixed=True):
    seed = dm.combined_seed(dropout_layer_seed(layer, part), _dropout_seed(step, rank))
    return ~dm.keep(seed, p, n, mixed=mixed)


def _q(p=P):
    return dm.threshold(p) / 65536.0


def _assert_independent(pairs, what):
    worst = []
    for (a, b) in pairs:
        z, s, rate = dm.worst_coincidence_sigma(a[1], b[1], _q(), _q())
        worst.append((z, a[0], b[0], s, rate))
    worst.sort(reverse=True)
    z, ka, kb, s, rate = worst[0]
    assert z < SIGMA, f"{what}: masks {ka} / {kb} coincide at shift {s}: P(both dropped) {rate:.4f} vs {_q() ** 2:.4f} ({z:.1f} sigma)"


# ---------------------------------------------------------------------------------------------------------------------- schedule
def test_seed_schedule():
    """The layer / part seeds and the per-step, per-rank device seed the engine uses; every (layer, part, step, rank) of a long run gets
    its own combined seed, and the device seed fits the int64 scalar it is written to."""
    assert dropout_layer_seed(1, 0) == dm.PHI
    assert dropout_layer_seed(3, 1) == (3 * dm.PHI + 0x632BE59BD9B4E019) & dm.M64
    assert _dropout_seed(5, 0) == 5 * 0x5DEECE66D and _dropout_seed(5) == _dropout_seed(5, 0)     # no process group: rank 0
    assert _dropout_seed(2, 1) == (2 * 0x5DEECE66D + dm.PHI) & 0x7FFFFFFFFFFF
    steps, ranks, layers, parts = range(1, 2001), range(8), range(1, 60), range(3)
    dev = {_dropout_seed(t, r) for t in steps for r in ranks}
    assert len(dev) == len(steps) * len(ranks) and all(0 <= d < 2 ** 63 for d in dev)
    lay = {dropout_layer_seed(k, i) for k in layers for i in parts}
    assert len(lay) == len(layers) * len(parts)
    combined = {dm.combined_seed(a, d) for a in lay for d in list(dev)[:400]}
    assert len(combined) == len(lay) * 400


def test_restatement_reads_sixteen_bit_fields():
    """Element 4 g + e reads bits [16 e, 16 e + 16) of group g's hash, whatever the start of the restated range."""
    seed = 0x1234567890ABCDEF
    m = int(dm.fmix(np.uint64(seed)))
    for g in (0, 1, 77):
        z = int(dm.fmix(np.uint64((m + dm.PHI * (g + 1)) & dm.M64)))
        assert [int(u) for u in dm.fields(seed, 4, 4 * g)] == [(z >> (16 * e)) & 0xFFFF for e in range(4)]
    whole = dm.fields(seed, 1000)
    assert np.array_equal(dm.fields(seed, 101, 333), whole[333:434])
    assert dm.threshold(0.1) == 6554 and dm.threshold(0.5) == 32768
    assert dm.keep_scale(0.1) == np.float32(65536 / (65536 - 6554))


# ---------------------------------------------------------------------------------------------------------------------- between masks
def test_layers_within_one_step_are_independent(c1_layers):
    """Every pair of the C1 finetune plan's 22 dropout layers at one step, consecutive layers first.  Before the seed was mixed, layer
    k + 1 drew layer k's mask shifted by 4 elements (P(both dropped) 0.0999 against 0.0100)."""
    masks = [(k, _drops(k)) for k in range(1, c1_layers + 1)]
    _assert_independent([(masks[i], masks[i + 1]) for i in range(len(masks) - 1)], "consecutive layers")
    _assert_independent([(masks[i], masks[j]) for i in range(len(masks)) for j in range(i + 2, len(masks))], "layers of one step")


def test_steps_ranks_and_parts_are_independent(c1_layers):
    """One layer at steps t and t + 1, on ranks 0 and 1, and on rank 1 against the next layer on rank 0; parts 0 / 1 (and 1 / 2) of a
    layer split into channel parts."""
    for k in range(1, c1_layers + 1):
        a = ((k, 0, 7, 0), _drops(k, step=7))
        _assert_independent([(a, ((k, 0, 8, 0), _drops(k, step=8)))], "consecutive steps")
        _assert_independent([(a, ((k, 0, 7, 1), _drops(k, step=7, rank=1)))], "ranks 0 / 1")
        if k < c1_layers:
            _assert_independent([(((k, 0, 7, 1), _drops(k, step=7, rank=1)), ((k + 1, 0, 7, 0), _drops(k + 1, step=7)))],
                                "rank 1 / the next layer on rank 0")
    for k in (1, 5):
        parts = [((k, i), _drops(k, part=i)) for i in range(3)]
        _assert_independent([(parts[0], parts[1]), (parts[1], parts[2])], "channel parts")


def test_unmixed_seed_gives_shifted_masks():
    """The statistic has teeth: the hash without the seed finalizer (the definition before the fix) fails it at a 4-element shift for
    consecutive layers, and not for the same layer at consecutive steps."""
    a, b = _drops(3, mixed=False), _drops(4, mixed=False)
    z, s, rate = dm.worst_coincidence_sigma(a, b, _q(), _q())
    assert z > 100 and s == -4 and abs(rate - _q()) < 2e-3, (z, s, rate)
    z, s, rate = dm.worst_coincidence_sigma(a, _drops(3, step=2, mixed=False), _q(), _q())
    assert z < SIGMA, (z, s, rate)


# ---------------------------------------------------------------------------------------------------------------------- within a mask
def _binomial_ok(k, n, q):
    return abs(k - q * n) <= SIGMA * math.sqrt(n * q * (1 - q))


def _chi2_2x2(a, b):
    """Pearson's chi-squared of the 2 x 2 table of two boolean arrays (1 degree of freedom)."""
    n = len(a)
    t = np.array([[np.count_nonzero(a & b), np.count_nonzero(a & ~b)], [np.count_nonzero(~a & b), np.count_nonzero(~a & ~b)]], float)
    e = np.outer(t.sum(1), t.sum(0)) / n
    return float(((t - e) ** 2 / e).sum())


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_rate_per_position_and_channel(p):
    """Keep rate 1 - thr / 65536 exactly (within binomial bounds) for each element position mod 4 and each channel of a C = 64 and a
    C = 179 tensor (a pruned width: channels walk across hash words)."""
    seed = dm.combined_seed(dropout_layer_seed(2, 0), _dropout_seed(3, 0))
    kp = dm.keep(seed, p, 4 << 20)
    q = 1 - dm.threshold(p) / 65536.0
    for e in range(4):
        sub = kp[e::4]
        assert _binomial_ok(np.count_nonzero(sub), len(sub), q), (p, e)
    for C in (64, 179):
        n = len(kp) // C * C
        per_c = kp[:n].reshape(-1, C).sum(0)
        rows = n // C
        bad = [c for c in range(C) if not _binomial_ok(int(per_c[c]), rows, q)]
        assert not bad, (p, C, bad)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_neighbours_and_fields_of_one_word_are_independent(p):
    """2 x 2 chi-squared (1 dof) between element i and i + 1, i + 4, and between every two of the four fields of one hash word: below
    36, a 6-sigma bound."""
    seed = dm.combined_seed(dropout_layer_seed(9, 1), _dropout_seed(11, 3))
    kp = dm.keep(seed, p, 4 << 20)
    for s in (1, 4):
        assert _chi2_2x2(kp[:-s], kp[s:]) < SIGMA ** 2, (p, s)
    w = kp.reshape(-1, 4)
    for e in range(4):
        for f in range(e + 1, 4):
            assert _chi2_2x2(w[:, e], w[:, f]) < SIGMA ** 2, (p, e, f)
