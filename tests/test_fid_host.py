"""FID evaluation, host side: the Inception oracle against the reference's features, state-dict layout, BatchNorm folding, the
weight-file lookup, the Fréchet distance, .npz statistics and the compat command line."""
import json
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, ROOT, load_golden, max_rel
from oracle import inception_oracle as orc
import diff_pruning_b200.fid as fid

sys.path.insert(0, os.path.join(ROOT, "diff-pruning_b200", "compat"))


def _layout():
    return json.load(open(os.path.join(GOLDEN, "fid_weights.json")))


def seeded_weights():
    """The fixture weights: torchvision names as in the weight file, rebuilt from the recorded seed."""
    lay = _layout()
    sd = orc.seeded_state_dict(lay["weight_file"], lay["seed"])
    assert orc.state_dict_digest(sd) == lay["digest"]
    return sd


def test_oracle_matches_reference_features():
    sd = fid.convert_torchvision_state_dict(seeded_weights())
    gold = load_golden("fid_features.pt")
    for hw, u8 in gold["images"].items():
        x = u8.permute(0, 3, 1, 2).float() / 255.0
        with torch.no_grad():
            outs = orc.forward(sd, x, (0, 1, 2, 3))
        for b, (o, ref) in enumerate(zip(outs, gold["features"][hw])):
            assert max_rel(orc.pooled(o), ref) < 1e-5, (hw, b)


def test_state_dict_layout_both_name_sets():
    lay = _layout()
    model = fid.InceptionV3([0, 1, 2, 3], weights=False)
    assert [[k, list(v.shape)] for k, v in model.state_dict().items()] == lay["wrapper"]
    tv = seeded_weights()
    assert any(k.startswith("fc.") for k in tv)
    # the weight file (torchvision names, fc.*), with and without num_batches_tracked, and the wrapper's own names
    no_nbt = {k: v for k, v in tv.items() if not k.endswith("num_batches_tracked")}
    wrapper = fid.convert_torchvision_state_dict(tv)
    for sd in (tv, no_nbt, wrapper):
        m = fid.InceptionV3([0, 1, 2, 3], weights=sd)
        got = m.state_dict()
        for k, v in wrapper.items():
            if not k.endswith("num_batches_tracked"):
                assert torch.equal(got[k], v), k
    # fewer blocks: only their tensors, as the reference wrapper builds only blocks up to the last one needed
    m1 = fid.InceptionV3([1], weights=tv)
    assert all(k.startswith(("blocks.0.", "blocks.1.")) for k in m1.state_dict())
    with pytest.raises(KeyError):
        fid.InceptionV3([3], weights={k: v for k, v in tv.items() if not k.startswith("Mixed_7c")})


def test_bn_folding_equals_conv_bn_relu():
    sd = fid.convert_torchvision_state_dict(seeded_weights())
    model = fid.InceptionV3([3], weights=sd)
    g = torch.Generator().manual_seed(5)
    for name, kw in (("blocks.2.4.branch7x7_2", dict(padding=(0, 3))), ("blocks.3.0.branch3x3_2", dict(stride=2)),
                     ("blocks.0.0", dict(stride=2))):
        mod = model.get_submodule(name)
        w, b = fid.fold_bn(mod)
        x = torch.randn(2, w.shape[1], 17, 17, generator=g).abs()
        ref = orc.basic(sd, name, x, **kw)
        got = F.relu(F.conv2d(x, w, b, **kw))
        assert max_rel(got, ref) < 2e-6, name


def test_weight_lookup_order_and_missing_file(tmp_path, monkeypatch):
    def no_network(*a, **k):
        raise AssertionError("network access")
    monkeypatch.setattr(socket, "socket", no_network)
    monkeypatch.setattr(socket, "create_connection", no_network)
    hub = tmp_path / "hub"
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(hub))
    monkeypatch.delenv(fid.WEIGHTS_ENV, raising=False)
    with pytest.raises(FileNotFoundError) as e:
        fid.find_weights()
    assert fid.WEIGHTS_FILE in str(e.value)
    with pytest.raises(FileNotFoundError):
        fid.InceptionV3([3])
    (hub / "checkpoints").mkdir(parents=True)
    cached = hub / "checkpoints" / fid.WEIGHTS_FILE
    cached.write_bytes(b"x")
    assert fid.find_weights() == str(cached)
    env = tmp_path / "env.pth"
    env.write_bytes(b"x")
    monkeypatch.setenv(fid.WEIGHTS_ENV, str(env))
    assert fid.find_weights() == str(env)
    explicit = tmp_path / "explicit.pth"
    explicit.write_bytes(b"x")
    assert fid.find_weights(str(explicit)) == str(explicit)
    # a path that does not exist is skipped, and reported if nothing else is found
    monkeypatch.delenv(fid.WEIGHTS_ENV)
    cached.unlink()
    with pytest.raises(FileNotFoundError) as e:
        fid.find_weights(str(tmp_path / "nope.pth"))
    assert "nope.pth" in str(e.value) and fid.WEIGHTS_FILE in str(e.value)


def test_weights_load_from_file(tmp_path):
    p = tmp_path / fid.WEIGHTS_FILE
    tv = seeded_weights()
    torch.save(tv, p)
    m = fid.InceptionV3([0], weights=str(p))
    assert torch.equal(m.state_dict()["blocks.0.0.conv.weight"], tv["Conv2d_1a_3x3.conv.weight"])


def test_frechet_distance_golden():
    for case in load_golden("fid_frechet.pt"):
        args = {k: case[k] for k in ("mu1", "sigma1", "mu2", "sigma2")}
        if "error" in case:
            with pytest.raises(ValueError, match="Imaginary component"):
                fid.calculate_frechet_distance(**args)
        else:
            got = fid.calculate_frechet_distance(**args)
            assert abs(got - case["fid"]) <= 1e-12 * abs(case["fid"]), (got, case["fid"])
    with pytest.raises(ValueError):
        fid.calculate_frechet_distance(np.zeros(2), np.eye(2), np.zeros(3), np.eye(3))


def test_npz_round_trip(tmp_path):
    rng = np.random.default_rng(0)
    a = rng.standard_normal((30, 6))
    mu, sigma = a.mean(0), np.cov(a, rowvar=False)
    p = str(tmp_path / "stats.npz")
    fid.save_stats(p, mu, sigma)
    with np.load(p) as f:
        assert sorted(f.files) == ["mu", "sigma"]
    m2, s2 = fid.compute_statistics_of_path(p, None, 50, 2048, "cuda")
    assert np.array_equal(m2, mu) and np.array_equal(s2, sigma)
    assert fid.calculate_frechet_distance(m2, s2, mu, sigma) == pytest.approx(0.0, abs=1e-9)


def test_compat_cli_surface():
    import fid_score
    import inception
    assert inception.InceptionV3 is fid.InceptionV3 and inception.InceptionV3.BLOCK_INDEX_BY_DIM == {64: 0, 192: 1, 768: 2, 2048: 3}
    a = fid_score.parser.parse_args(["--save-stats", "imgs", "out.npz", "--batch-size", "256", "--dims", "768", "--device", "cuda:0"])
    assert a.save_stats and a.path == ["imgs", "out.npz"] and a.batch_size == 256 and a.dims == 768
    assert fid_score.check_args(a) == "cuda:0"
    assert fid_score.check_args(fid_score.parser.parse_args(["a", "b"])) == "cuda"
    for extra in (["--res", "64"], ["--dataset_name", "celeba"], ["--num-workers", "4"], ["--device", "cpu"]):
        with pytest.raises(NotImplementedError):
            fid_score.check_args(fid_score.parser.parse_args(["a", "b"] + extra))
    with pytest.raises(SystemExit):
        fid_score.parser.parse_args(["a", "b", "--dims", "100"])
    for name in ("get_activations", "calculate_activation_statistics", "compute_statistics_of_path", "calculate_frechet_distance",
                 "calculate_fid_given_paths", "save_fid_stats"):
        assert callable(getattr(fid_score, name))
