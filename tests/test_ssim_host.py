"""SSIM evaluation, host side: the torch oracle against the reference's utils_image.py values, the window taps, pytorch_msssim's
argument rules (checked before the library is touched), folder pairing, and the compat import."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden
from oracle import ssim_oracle as orc
import diff_pruning_b200.ssim as S
from diff_pruning_b200 import _lib as L

sys.path.insert(0, os.path.join(ROOT, "diff-pruning_b200", "compat"))


def _nchw(u8):
    return u8.permute(2, 0, 1)[None].double()


def test_fp64_oracle_matches_reference():
    """The definition (separable valid Gaussian, H then W, the map's mean) in fp64 with fp64 taps equals utils_image.py's."""
    g = orc.window(dtype=torch.float64)
    for case in load_golden("ssim_ref.pt"):
        x, y = _nchw(case["x"]), _nchw(case["y"])
        per_c = orc.ssim_per_channel(x, y, data_range=255.0, g=g)[0]
        assert float((per_c - case["ssim_c"]).abs().max()) <= 1e-10, case["name"]
        assert abs(float(per_c.mean()) - case["ssim"]) <= 1e-10, case["name"]
        # scale invariance: [0, 1] values at data_range 1 give the same numbers
        per_c1 = orc.ssim_per_channel(x / 255, y / 255, data_range=1.0, g=g)[0]
        assert float((per_c1 - case["ssim_c"]).abs().max()) <= 1e-10, case["name"]
    assert torch.equal(S.gaussian_window(dtype=torch.float64), g)


def test_window_taps_match_cv2():
    cv2 = pytest.importorskip("cv2")
    g = S.gaussian_window()
    assert g.dtype == torch.float32 and g.shape == (11,)
    ref = cv2.getGaussianKernel(11, 1.5).ravel()
    assert np.abs(g.double().numpy() - ref).max() <= 1e-7
    assert torch.equal(g, orc.window())


def test_tensor_to_tensor_division_is_correctly_rounded():
    """ToTensor's u8 / 255 in torch on the host equals the correctly rounded fp32 quotient the u8 kernel route forms."""
    u = torch.arange(256, dtype=torch.uint8)
    got = u.float().div(255).numpy()
    ref = (np.arange(256, dtype=np.float64) / 255).astype(np.float32)
    assert np.array_equal(got, ref)


@pytest.fixture
def no_library(monkeypatch):
    def refuse():
        raise AssertionError("the library was touched")
    monkeypatch.setattr(L, "load", refuse)


def test_value_errors(no_library):
    x = torch.zeros(2, 3, 16, 16)
    with pytest.raises(ValueError):
        S.ssim(x, torch.zeros(2, 3, 16, 17))                    # shapes differ
    with pytest.raises(ValueError):
        S.ssim(torch.zeros(3, 16, 16), torch.zeros(3, 16, 16))  # 3-D
    with pytest.raises(ValueError):
        S.ssim(torch.zeros(2, 3, 1, 16), torch.zeros(2, 3, 1, 16))   # the singleton squeeze leaves 3 dimensions
    with pytest.raises(ValueError):
        S.ssim(torch.zeros(2, 2, 2, 2, 16, 16), torch.zeros(2, 2, 2, 2, 16, 16))   # 6-D
    with pytest.raises(ValueError):
        S.ssim(x, x, win_size=10)
    with pytest.raises(ValueError):
        S.ssim(x, x, win=torch.ones(3, 1, 1, 10))


def test_not_implemented(no_library):
    x = torch.zeros(2, 3, 16, 16)
    for a, kw in (((x, x), {}),                                             # CPU tensors
                  ((torch.zeros(2, 3, 16, 16, 16), torch.zeros(2, 3, 16, 16, 16)), {}),   # 5-D
                  ((x, x), dict(win_size=7)),
                  ((x, x), dict(win=orc.window().view(1, 1, 1, 11).repeat(3, 1, 1, 1))),
                  ((torch.zeros(2, 3, 10, 16), torch.zeros(2, 3, 10, 16)), {})):
        with pytest.raises(NotImplementedError):
            S.ssim(*a, **kw)


@pytest.mark.gpu
def test_not_implemented_on_device(no_library):
    """dtype and size rules (checked after the CUDA one)."""
    x = torch.zeros(2, 3, 16, 16, device="cuda")
    with pytest.raises(NotImplementedError):
        S.ssim(x.double(), x.double())
    with pytest.raises(NotImplementedError):
        S.ssim(x[:, :, :10], x[:, :, :10])


def test_squeeze_keeps_trailing_singletons_out():
    # [N, C, H, W, 1] squeezes to 4-D (pytorch_msssim's rule): only the CUDA requirement is left to refuse it here
    x = torch.zeros(2, 3, 16, 16, 1)
    with pytest.raises(NotImplementedError, match="CUDA"):
        S.ssim(x, x)


def test_paths_must_pair(tmp_path, no_library):
    from PIL import Image
    im = Image.fromarray(np.zeros((16, 16, 3), np.uint8))
    for d, names in (("a", ["0.png", "1.png", "sub/2.png"]), ("b", ["0.png", "1.png", "2.png"])):
        for n in names:
            p = tmp_path / d / n
            p.parent.mkdir(parents=True, exist_ok=True)
            im.save(p)
    with pytest.raises(ValueError, match="relative paths"):
        S.ssim_of_paths(tmp_path / "a", tmp_path / "b")


def test_capi_argument_rules():
    """dp_ssim rejects bad arguments before any launch (safe without a GPU)."""
    import ctypes
    lib = L.load()

    def call(**kw):
        a = L.SsimArgs()
        a.x, a.y, a.ssim_nc, a.sse_n = 16, 32, 64, 128          # never dereferenced: every case below fails validation
        a.format, a.N, a.C, a.H, a.W, a.win_size = 0, 2, 3, 32, 32, 11
        for k, v in kw.items():
            setattr(a, k, v)
        return lib.dp_ssim(ctypes.byref(a), None)
    assert call(ssim_nc=None) == -5 and call(sse_n=None) == -5 and call(x=None) == -5
    assert call(H=10) == -1 and call(W=10) == -1 and call(N=0) == -1
    assert call(win_size=7) == -3 and call(format=3) == -3


def test_compat_import():
    import pytorch_msssim
    assert pytorch_msssim.ssim is S.ssim
