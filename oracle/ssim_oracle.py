"""pytorch_msssim._ssim / ssim restated with torch functional ops, in the input's dtype: the checker of diff_pruning_b200.ssim.  Run
in fp64 it is the exact-grade reference; run in fp32 it is what pytorch_msssim gives on the same inputs."""
import torch
import torch.nn.functional as F


def window(size=11, sigma=1.5, dtype=torch.float32):
    """The 1-D Gaussian taps of pytorch_msssim._fspecial_gauss_1d (which builds them in fp32); dtype=torch.float64 gives the exact-grade
    taps of cv2.getGaussianKernel."""
    coords = torch.arange(size, dtype=dtype)
    coords -= size // 2
    g = torch.exp(-(coords ** 2) / (2 * sigma ** 2))
    return g / g.sum()


def gaussian_filter(x, g):
    """Grouped "valid" convolution along H, then along W, with the taps g (in x's dtype)."""
    C = x.shape[1]
    k = g.to(x.device, x.dtype)
    out = F.conv2d(x, k.view(1, 1, -1, 1).repeat(C, 1, 1, 1), groups=C)
    return F.conv2d(out, k.view(1, 1, 1, -1).repeat(C, 1, 1, 1), groups=C)


def ssim_per_channel(X, Y, data_range=1.0, K=(0.01, 0.03), g=None):
    """[N, C] mean SSIM map per image and channel, computed in X's dtype."""
    g = window() if g is None else g
    C1, C2 = (K[0] * data_range) ** 2, (K[1] * data_range) ** 2
    mu1, mu2 = gaussian_filter(X, g), gaussian_filter(Y, g)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = gaussian_filter(X * X, g) - mu1_sq
    sigma2_sq = gaussian_filter(Y * Y, g) - mu2_sq
    sigma12 = gaussian_filter(X * Y, g) - mu1_mu2
    cs_map = (2 * sigma12 + C2) / (sigma1_sq + sigma2_sq + C2)
    ssim_map = ((2 * mu1_mu2 + C1) / (mu1_sq + mu2_sq + C1)) * cs_map
    return torch.flatten(ssim_map, 2).mean(-1)


def ssim(X, Y, data_range=255, size_average=True, K=(0.01, 0.03)):
    s = ssim_per_channel(X, Y, data_range, K)
    return s.mean() if size_average else s.mean(1)
