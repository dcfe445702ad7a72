"""CPU fp32 restatement of the FID Inception-v3 feature network (the reference's inception.py on torchvision's inception_v3) with torch
functional ops.  BasicConv2d stays conv -> eval BatchNorm (eps 0.001) -> ReLU, NOT folded, so the device plan's host-side folding is
checked too.  Parameters are read from a state dict with the wrapper's keys (`blocks.<block>.<layer>.<branch>.conv.weight`, ...).

Tests and the benchmark import this module; the reference checkout is never imported."""
import torch
import torch.nn.functional as F


def basic(sd, pre, x, stride=1, padding=0):
    """torchvision BasicConv2d: Conv2d(bias=False) + BatchNorm2d(eps=0.001) + ReLU."""
    x = F.conv2d(x, sd[pre + ".conv.weight"], None, stride, padding)
    x = F.batch_norm(x, sd[pre + ".bn.running_mean"], sd[pre + ".bn.running_var"], sd[pre + ".bn.weight"], sd[pre + ".bn.bias"],
                     False, 0.0, 0.001)
    return F.relu(x)


def _avg(x):   # the FID patch of blocks A / C / E_1: padded zeros are not counted (inception.py:239-242, 267-270, 300-303)
    return F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False)


def mixed_a(sd, p, x):   # FIDInceptionA.forward, inception.py:229-246
    b1 = basic(sd, p + ".branch1x1", x)
    b5 = basic(sd, p + ".branch5x5_2", basic(sd, p + ".branch5x5_1", x), padding=2)
    bd = basic(sd, p + ".branch3x3dbl_1", x)
    bd = basic(sd, p + ".branch3x3dbl_3", basic(sd, p + ".branch3x3dbl_2", bd, padding=1), padding=1)
    return torch.cat([b1, b5, bd, basic(sd, p + ".branch_pool", _avg(x))], 1)


def mixed_b(sd, p, x):   # torchvision InceptionB (Mixed_6a), unpatched
    b3 = basic(sd, p + ".branch3x3", x, stride=2)
    bd = basic(sd, p + ".branch3x3dbl_2", basic(sd, p + ".branch3x3dbl_1", x), padding=1)
    bd = basic(sd, p + ".branch3x3dbl_3", bd, stride=2)
    return torch.cat([b3, bd, F.max_pool2d(x, kernel_size=3, stride=2)], 1)


def mixed_c(sd, p, x):   # FIDInceptionC.forward, inception.py:254-274
    b1 = basic(sd, p + ".branch1x1", x)
    b7 = basic(sd, p + ".branch7x7_1", x)
    b7 = basic(sd, p + ".branch7x7_2", b7, padding=(0, 3))
    b7 = basic(sd, p + ".branch7x7_3", b7, padding=(3, 0))
    bd = basic(sd, p + ".branch7x7dbl_1", x)
    for i, pad in ((2, (3, 0)), (3, (0, 3)), (4, (3, 0)), (5, (0, 3))):
        bd = basic(sd, p + ".branch7x7dbl_%d" % i, bd, padding=pad)
    return torch.cat([b1, b7, bd, basic(sd, p + ".branch_pool", _avg(x))], 1)


def mixed_d(sd, p, x):   # torchvision InceptionD (Mixed_7a), unpatched
    b3 = basic(sd, p + ".branch3x3_2", basic(sd, p + ".branch3x3_1", x), stride=2)
    b7 = basic(sd, p + ".branch7x7x3_1", x)
    b7 = basic(sd, p + ".branch7x7x3_2", b7, padding=(0, 3))
    b7 = basic(sd, p + ".branch7x7x3_3", b7, padding=(3, 0))
    b7 = basic(sd, p + ".branch7x7x3_4", b7, stride=2)
    return torch.cat([b3, b7, F.max_pool2d(x, kernel_size=3, stride=2)], 1)


def mixed_e(sd, p, x, max_pool):   # FIDInceptionE_1 (avg pool, inception.py:282-307) / FIDInceptionE_2 (max pool, :315-341)
    b1 = basic(sd, p + ".branch1x1", x)
    b3 = basic(sd, p + ".branch3x3_1", x)
    b3 = torch.cat([basic(sd, p + ".branch3x3_2a", b3, padding=(0, 1)), basic(sd, p + ".branch3x3_2b", b3, padding=(1, 0))], 1)
    bd = basic(sd, p + ".branch3x3dbl_2", basic(sd, p + ".branch3x3dbl_1", x), padding=1)
    bd = torch.cat([basic(sd, p + ".branch3x3dbl_3a", bd, padding=(0, 1)), basic(sd, p + ".branch3x3dbl_3b", bd, padding=(1, 0))], 1)
    pool = F.max_pool2d(x, kernel_size=3, stride=1, padding=1) if max_pool else _avg(x)
    return torch.cat([b1, b3, bd, basic(sd, p + ".branch_pool", pool)], 1)


def forward(sd, x, output_blocks=(3,), resize_input=True, normalize_input=True):
    """InceptionV3.forward (inception.py:129-163): x is [N, 3, H, W] fp32 in [0, 1]; returns the outputs of `output_blocks`
    (0: first max pool, 64 ch; 1: second max pool, 192 ch; 2: Mixed_6e, 768 ch; 3: final average pool, 2048 x 1 x 1) in ascending order."""
    blocks = sorted(output_blocks)
    last = max(blocks)
    if resize_input:
        x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False)
    if normalize_input:
        x = 2 * x - 1
    out = []
    # block 0 (inception.py:85-91): Conv2d_1a_3x3, Conv2d_2a_3x3, Conv2d_2b_3x3, max pool
    x = basic(sd, "blocks.0.0", x, stride=2)
    x = basic(sd, "blocks.0.1", x)
    x = basic(sd, "blocks.0.2", x, padding=1)
    x = F.max_pool2d(x, kernel_size=3, stride=2)
    if 0 in blocks:
        out.append(x)
    if last >= 1:   # block 1 (:94-100): Conv2d_3b_1x1, Conv2d_4a_3x3, max pool
        x = F.max_pool2d(basic(sd, "blocks.1.1", basic(sd, "blocks.1.0", x)), kernel_size=3, stride=2)
        if 1 in blocks:
            out.append(x)
    if last >= 2:   # block 2 (:103-114): Mixed_5b .. Mixed_6e
        for i in range(3):
            x = mixed_a(sd, "blocks.2.%d" % i, x)
        x = mixed_b(sd, "blocks.2.3", x)
        for i in range(4, 8):
            x = mixed_c(sd, "blocks.2.%d" % i, x)
        if 2 in blocks:
            out.append(x)
    if last >= 3:   # block 3 (:117-124): Mixed_7a .. Mixed_7c, adaptive average pool to 1 x 1
        x = mixed_d(sd, "blocks.3.0", x)
        x = mixed_e(sd, "blocks.3.1", x, max_pool=False)
        x = mixed_e(sd, "blocks.3.2", x, max_pool=True)
        out.append(F.adaptive_avg_pool2d(x, (1, 1)))
    return out


def seeded_state_dict(shapes, seed=0):
    """The random stand-in for the Inception weights the fixtures are built with: `shapes` is the weight file's [(key, shape)] list in
    file order; values are drawn in that order from torch's CPU generator seeded with `seed`.  Convolutions are He-normal
    (std sqrt(2 / fan_in)); BatchNorm gets gamma, running_var ~ U[0.5, 1.5), beta, running_mean ~ 0.1 N(0, 1), so activations neither
    vanish nor blow up over the ~45 sequential layers; fc.weight ~ 0.01 N(0, 1), fc.bias = 0."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for key, shape in shapes:
        shape = tuple(shape)
        if key.endswith("num_batches_tracked"):
            sd[key] = torch.zeros(shape, dtype=torch.long)
        elif key.endswith("conv.weight"):
            fan_in = shape[1] * shape[2] * shape[3]
            sd[key] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
        elif key.endswith("bn.weight") or key.endswith("bn.running_var"):
            sd[key] = 0.5 + torch.rand(shape, generator=g)
        elif key.endswith("bn.bias") or key.endswith("bn.running_mean"):
            sd[key] = 0.1 * torch.randn(shape, generator=g)
        elif key == "fc.weight":
            sd[key] = 0.01 * torch.randn(shape, generator=g)
        elif key == "fc.bias":
            sd[key] = torch.zeros(shape)
        else:
            raise KeyError(key)
    return sd


def state_dict_digest(sd):
    """sha256 over the keys, shapes and raw bytes of a state dict, in key order."""
    import hashlib
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(str(tuple(v.shape)).encode())
        h.update(v.detach().contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


def pooled(feature_map):
    """fid_score.py:170-173: a block output that is not 1 x 1 is averaged over H x W, then flattened to [N, C]."""
    if feature_map.shape[2] != 1 or feature_map.shape[3] != 1:
        feature_map = F.adaptive_avg_pool2d(feature_map, (1, 1))
    return feature_map.flatten(1)
