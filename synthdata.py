"""Seeded synthetic inputs shared by the tests, the oracle and bench.py (``oracle/synth.py`` re-exports this module).

Workload generator, not part of the oracle and not part of the product (no reference arithmetic in here): image pairs as in
SURVEY.md section 8(d), random network weights with the reference's state_dict
key names (SURVEY.md section 8b), synthetic match sets for kernel-level RANSAC
cases.  Everything is generated on the CPU generators so both arms (GPU path
and CPU oracle) see identical bytes on any machine.
"""
import math

import numpy as np
import torch


# --------------------------------------------------------------------------
# weights
# --------------------------------------------------------------------------
def _conv(g, cout, cin, k, std=None):
    # kaiming_normal_(mode='fan_out', nonlinearity='relu'), model/model.py:78-79
    if std is None:
        std = math.sqrt(2.0 / (cout * k * k))
    return torch.randn(cout, cin, k, k, generator=g) * std


def _bn(g, sd, p, c, randomize):
    if randomize:
        sd[p + ".weight"] = torch.rand(c, generator=g) * 0.5 + 0.75
        sd[p + ".bias"] = torch.randn(c, generator=g) * 0.1
        sd[p + ".running_mean"] = torch.randn(c, generator=g) * 0.1
        sd[p + ".running_var"] = torch.rand(c, generator=g) * 0.5 + 0.75
    else:
        sd[p + ".weight"] = torch.ones(c)
        sd[p + ".bias"] = torch.zeros(c)
        sd[p + ".running_mean"] = torch.zeros(c)
        sd[p + ".running_var"] = torch.ones(c)
    sd[p + ".num_batches_tracked"] = torch.tensor(0)


def _blur_filt(c):
    a = torch.tensor([1.0, 2.0, 1.0])
    f = a[:, None] * a[None, :]
    return (f / f.sum())[None, None].repeat(c, 1, 1, 1)


def feature_extractor_state(seed=0, randomize_bn=True):
    """state_dict of model.FeatureExtractor (model/model.py:59-103; keys SURVEY 8b)."""
    g = torch.Generator().manual_seed(seed)
    sd = {"conv1.weight": _conv(g, 64, 3, 3)}
    _bn(g, sd, "bn1", 64, randomize_bn)
    sd["maxpool.1.filt"] = _blur_filt(64)
    inpl = 64
    for layer, planes, stride in (("layer1", 64, 1), ("layer2", 128, 2), ("layer3", 256, 2)):
        for b in range(2):
            p = "%s.%d" % (layer, b)
            sd[p + ".conv1.weight"] = _conv(g, planes, inpl if b == 0 else planes, 3)
            _bn(g, sd, p + ".bn1", planes, randomize_bn)
            sd[p + ".conv2.weight"] = _conv(g, planes, planes, 3)
            _bn(g, sd, p + ".bn2", planes, randomize_bn)
            if b == 0 and stride != 1:
                sd[p + ".downsample.0.filt"] = _blur_filt(inpl)
                sd[p + ".downsample.1.weight"] = _conv(g, planes, inpl, 1)
                _bn(g, sd, p + ".downsample.2", planes, randomize_bn)
        inpl = planes
    return sd


def _head_state(seed, k, cout, last_std, randomize_bn):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    chans = [k * k, 512, 256, 128]
    for i in range(3):
        sd["conv%d.weight" % (i + 1)] = _conv(g, chans[i + 1], chans[i], 3)
        _bn(g, sd, "bn%d" % (i + 1), chans[i + 1], randomize_bn)
    sd["conv4.weight"] = _conv(g, cout, 128, 3, std=last_std)
    return sd


def net_flow_coarse_state(seed=1, k=7, randomize_bn=True):
    """state_dict of model.NetFlowCoarse (model/model.py:167-203)."""
    return _head_state(seed, k, k * k, None, randomize_bn)


def net_matchability_state(seed=2, k=7, randomize_bn=True, conv4_std=0.02):
    """state_dict of model.NetMatchability (model/model.py:254-285).  The
    reference initialises conv4 with std 1e-4 (matchability == 0.5 everywhere);
    the synthetic default is larger so the map is not degenerate (SURVEY A.6)."""
    return _head_state(seed, k, 1, conv4_std, randomize_bn)


RESNET50_LAYERS = (("layer1", 64, 3, 1), ("layer2", 128, 4, 2), ("layer3", 256, 6, 2))


def resnet50_conv4_state(seed=0, randomize_bn=True):
    """state_dict of torchvision resnet50 truncated at layer3 (key names of
    ``torchvision.models.resnet50().state_dict()``)."""
    g = torch.Generator().manual_seed(seed + 1000)
    sd = {"conv1.weight": _conv(g, 64, 3, 7)}
    _bn(g, sd, "bn1", 64, randomize_bn)
    inpl = 64
    for layer, planes, blocks, stride in RESNET50_LAYERS:
        for b in range(blocks):
            p = "%s.%d" % (layer, b)
            sd[p + ".conv1.weight"] = _conv(g, planes, inpl, 1)
            _bn(g, sd, p + ".bn1", planes, randomize_bn)
            sd[p + ".conv2.weight"] = _conv(g, planes, planes, 3)
            _bn(g, sd, p + ".bn2", planes, randomize_bn)
            sd[p + ".conv3.weight"] = _conv(g, planes * 4, planes, 1)
            _bn(g, sd, p + ".bn3", planes * 4, randomize_bn)
            if b == 0:
                sd[p + ".downsample.0.weight"] = _conv(g, planes * 4, inpl, 1)
                _bn(g, sd, p + ".downsample.1", planes * 4, randomize_bn)
            inpl = planes * 4
    return sd


def tiny_resnet_like_state(seed=0, widths=(16, 8, 16, 32), randomize_bn=True):
    """A structurally identical but narrow ResNet-50[:layer3] (same key names,
    same block counts) so CPU tests of the whole trunk run in milliseconds."""
    g = torch.Generator().manual_seed(seed + 2000)
    stem, p1, p2, p3 = widths
    sd = {"conv1.weight": _conv(g, stem, 3, 7)}
    _bn(g, sd, "bn1", stem, randomize_bn)
    inpl = stem
    for (layer, _, blocks, stride), planes in zip(RESNET50_LAYERS, (p1, p2, p3)):
        for b in range(blocks):
            p = "%s.%d" % (layer, b)
            sd[p + ".conv1.weight"] = _conv(g, planes, inpl, 1)
            _bn(g, sd, p + ".bn1", planes, randomize_bn)
            sd[p + ".conv2.weight"] = _conv(g, planes, planes, 3)
            _bn(g, sd, p + ".bn2", planes, randomize_bn)
            sd[p + ".conv3.weight"] = _conv(g, planes * 4, planes, 1)
            _bn(g, sd, p + ".bn3", planes * 4, randomize_bn)
            if b == 0:
                sd[p + ".downsample.0.weight"] = _conv(g, planes * 4, inpl, 1)
                _bn(g, sd, p + ".downsample.1", planes * 4, randomize_bn)
            inpl = planes * 4
    return sd


SEGNET_LAYERS = (("layer1", 64, 3), ("layer2", 128, 4), ("layer3", 256, 6), ("layer4", 512, 3))


def _bn_small(g, sd, p, c, gamma):
    """An eval-mode BN drawn from the generator with its weights scaled by ``gamma``: a residual branch that adds a fraction of
    its input's scale, so activations stay O(1..100) through 16 blocks (fp16 range) without calibrating on data."""
    _bn(g, sd, p, c, True)
    sd[p + ".weight"] = sd[p + ".weight"] * gamma


def _syncbn_extras(g, sd, p, c):
    # SynchronizedBatchNorm2d checkpoints carry these too; the network never reads them
    sd[p + "._tmp_running_mean"] = torch.randn(c, generator=g)
    sd[p + "._tmp_running_var"] = torch.rand(c, generator=g)
    sd[p + "._running_iter"] = torch.ones(1)


def segnet_encoder_state(seed=0):
    """state_dict of segNet's ResnetDilated(resnet50) (segNet/segModel.py:59-216; key names of the ADE20K encoder checkpoint)."""
    g = torch.Generator().manual_seed(seed + 3000)
    sd = {}
    for i, (cin, cout) in enumerate(((3, 64), (64, 64), (64, 128)), 1):
        sd["conv%d.weight" % i] = _conv(g, cout, cin, 3)
        _bn(g, sd, "bn%d" % i, cout, True)
    _syncbn_extras(g, sd, "bn1", 64)
    inpl = 128
    for layer, planes, blocks in SEGNET_LAYERS:
        for b in range(blocks):
            p = "%s.%d" % (layer, b)
            sd[p + ".conv1.weight"] = _conv(g, planes, inpl, 1)
            _bn(g, sd, p + ".bn1", planes, True)
            sd[p + ".conv2.weight"] = _conv(g, planes, planes, 3)
            _bn(g, sd, p + ".bn2", planes, True)
            sd[p + ".conv3.weight"] = _conv(g, planes * 4, planes, 1)
            _bn_small(g, sd, p + ".bn3", planes * 4, 0.25)
            if b == 0:
                sd[p + ".downsample.0.weight"] = _conv(g, planes * 4, inpl, 1, std=math.sqrt(1.0 / inpl))
                _bn(g, sd, p + ".downsample.1", planes * 4, True)
            inpl = planes * 4
    return sd


def segnet_decoder_state(seed=0, class_bias=(3.5, 3.0)):
    """state_dict of segNet's PPMDeepsup(150 classes, fc_dim 2048) (segNet/segModel.py:218-243; key names of the ADE20K decoder
    checkpoint, deep-supervision weights included).  ``class_bias`` = the bias of classes 1 (building) and 2 (sky): they dominate
    the other classes, and which of the two wins varies over the image."""
    g = torch.Generator().manual_seed(seed + 4000)
    sd = {}
    for j in range(4):
        sd["ppm.%d.1.weight" % j] = _conv(g, 512, 2048, 1, std=math.sqrt(1.0 / 2048))
        _bn(g, sd, "ppm.%d.2" % j, 512, True)
    sd["cbr_deepsup.0.weight"] = _conv(g, 512, 1024, 3)
    _bn(g, sd, "cbr_deepsup.1", 512, True)
    sd["conv_last.0.weight"] = _conv(g, 512, 4096, 3, std=math.sqrt(1.0 / (9 * 4096)))
    _bn(g, sd, "conv_last.1", 512, True)
    _syncbn_extras(g, sd, "conv_last.1", 512)
    sd["conv_last.4.weight"] = _conv(g, 150, 512, 1, std=math.sqrt(1.0 / 512))
    bias = torch.randn(150, generator=g) * 0.1
    bias[1], bias[2] = class_bias
    sd["conv_last.4.bias"] = bias
    sd["conv_last_deepsup.weight"] = _conv(g, 150, 512, 1)
    sd["conv_last_deepsup.bias"] = torch.zeros(150)
    return sd


def segnet_image(seed, h, w):
    """A seeded uint8 [h, w, 3] test image for segNet (a smooth texture: region structure, not noise)."""
    rs = np.random.RandomState(5000 + seed)
    return np.clip(_texture(rs, h, w) + rs.normal(0, 4, (h, w, 3)), 0, 255).astype(np.uint8)


# --------------------------------------------------------------------------
# image pairs (SURVEY.md section 8d)
# --------------------------------------------------------------------------
def _texture(rs, h, w):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.zeros((h, w, 3), dtype=np.float32)
    for c in range(3):
        acc = np.zeros((h, w), dtype=np.float32)
        for _ in range(8):
            fx, fy = rs.uniform(-0.08, 0.08, 2)
            ph = rs.uniform(0, 2 * np.pi)
            amp = rs.uniform(10, 40)
            acc += amp * np.sin(2 * np.pi * (fx * xx + fy * yy) + ph).astype(np.float32)
        img[..., c] = 128 + acc
    return img


def _bilinear_zero(img, gx, gy):
    """Sample (h,w,3) float image at pixel coords (gx, gy), zeros outside."""
    h, w = img.shape[:2]
    x0 = np.floor(gx).astype(np.int64)
    y0 = np.floor(gy).astype(np.int64)
    out = np.zeros(gx.shape + (3,), dtype=np.float32)
    for dy in (0, 1):
        for dx in (0, 1):
            xi, yi = x0 + dx, y0 + dy
            wgt = (1 - np.abs(gx - xi)) * (1 - np.abs(gy - yi))
            ok = (xi >= 0) & (xi < w) & (yi >= 0) & (yi < h)
            v = img[np.clip(yi, 0, h - 1), np.clip(xi, 0, w - 1)]
            out += (wgt * ok)[..., None].astype(np.float32) * v
    return out


def random_homography(rs):
    H = np.eye(3)
    H[:2, :] += rs.uniform(-0.08, 0.08, (2, 3))
    H[2, :2] += rs.uniform(-0.02, 0.02, 2)
    return H


def make_pair(i, h=480, w=640):
    """Pair ``i`` (seed 1000 + i): (source uint8 (h,w,3), target uint8 (h,w,3), H_t2s 3x3).

    target(x) = source(H x) in normalised [-1,1] coordinates + noise."""
    rs = np.random.RandomState(1000 + i)
    src = _texture(rs, h, w)
    src_n = np.clip(src + rs.normal(0, 8, src.shape), 0, 255)
    H = random_homography(rs)
    ys, xs = np.meshgrid(np.linspace(-1, 1, h), np.linspace(-1, 1, w), indexing="ij")
    den = H[2, 0] * xs + H[2, 1] * ys + H[2, 2]
    sx = (H[0, 0] * xs + H[0, 1] * ys + H[0, 2]) / den
    sy = (H[1, 0] * xs + H[1, 1] * ys + H[1, 2]) / den
    gx = (sx + 1) / 2 * (w - 1)
    gy = (sy + 1) / 2 * (h - 1)
    tgt = _bilinear_zero(src_n.astype(np.float32), gx.astype(np.float32), gy.astype(np.float32))
    tgt = np.clip(tgt + rs.normal(0, 4, tgt.shape), 0, 255)
    return src_n.astype(np.uint8), tgt.astype(np.uint8), H


def make_rotated_pair(i, h=480, w=640, k=1):
    """``make_pair(i, h, w)`` with the target rotated by 90 k degrees counter-clockwise (``np.rot90``, which is what
    ``PIL.Image.rotate(90 k, expand=True)`` does): the rotation evalYFCC's target search must undo is 360 - 90 k.
    Returns (source (h,w,3), rotated target ((h,w) or (w,h),3), H_t2s of the unrotated target)."""
    src, tgt, H = make_pair(i, h, w)
    return src, np.ascontiguousarray(np.rot90(tgt, k % 4)), H


# --------------------------------------------------------------------------
# match sets for kernel-level RANSAC cases (SURVEY.md section 8d)
# --------------------------------------------------------------------------
def make_matches(seed, M=636, inlier_frac=0.6, noise=0.005, grid=None):
    """(match1 (M,3), match2 (M,3)) fp32 with ``match1 ~ H match2`` for the
    inliers (the reference's convention: source = H * target, utils/outil.py:98)."""
    rs = np.random.RandomState(seed)
    H = random_homography(rs)
    if grid is None:
        m2 = rs.uniform(-1, 1, (M, 2))
    else:                                    # cell centres of an (h, w) grid, like getWHTensor
        gh, gw = grid
        r = rs.randint(0, gh, M)
        c = rs.randint(0, gw, M)
        m2 = np.stack([((c + 0.5) / gw - 0.5) * 2, ((r + 0.5) / gh - 0.5) * 2], axis=1)
    p = np.concatenate([m2, np.ones((M, 1))], axis=1) @ H.T
    m1 = p[:, :2] / p[:, 2:]
    m1 += rs.normal(0, noise, m1.shape)
    nout = int(round(M * (1 - inlier_frac)))
    out = rs.permutation(M)[:nout]
    m1[out] = rs.uniform(-1, 1, (nout, 2))
    one = np.ones((M, 1))
    return (np.concatenate([m1, one], 1).astype(np.float32),
            np.concatenate([m2, one], 1).astype(np.float32), H)


def draw_samples(seed, M, nbIter):
    """(nbIter,4) int64 sample indices on the CPU generator (tests feed the same
    array to the CUDA kernel and to the oracle)."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(M, (nbIter, 4), generator=g).numpy()
