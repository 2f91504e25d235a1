"""Torch-CPU oracle of segNet's getSky (segNet/segEval.py:23-43, segModel.py:59-264, segData.py:46-82), in fp32 or fp64.

Restated from the contract, not copied: the same resizes, dilated ResNet-50 encoder, PPM decoder and five-pass vote, written
with torch.nn.functional on explicit state_dict tensors.  Each distinct resized size is computed once; the vote then adds the
passes in the reference's order, repeats included (a repeated pass is the same deterministic computation).
"""
import numpy as np
import PIL.Image as Image
import torch
import torch.nn.functional as F

SIZES = (300, 375, 450, 525, 600)
MAX_SIZE = 500
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
LAYERS = (("layer1", 3, 1, 1), ("layer2", 4, 2, 1), ("layer3", 6, 1, 2), ("layer4", 3, 1, 4))   # blocks, stride, dilation
BINS = (1, 2, 3, 6)


def pass_sizes(H, W):
    out = []
    for s in SIZES:
        r = min(s / float(min(H, W)), MAX_SIZE / float(max(H, W)))
        h, w = int(H * r), int(W * r)
        out.append((-(-h // 8) * 8, -(-w // 8) * 8))
    return out


def _prep(img, h, w, dtype):
    a = np.float32(np.array(img.resize((w, h), Image.BILINEAR))) / 255.
    t = torch.from_numpy(a.transpose(2, 0, 1).copy())
    t = (t - torch.tensor(MEAN).view(3, 1, 1)) / torch.tensor(STD).view(3, 1, 1)
    return t.unsqueeze(0).to(dtype)


class _Net:
    def __init__(self, enc, dec, dtype, stats):
        self.enc = {k: v.to(dtype) for k, v in enc.items() if torch.is_tensor(v) and v.is_floating_point()}
        self.dec = {k: v.to(dtype) for k, v in dec.items() if torch.is_tensor(v) and v.is_floating_point()}
        self.stats = stats

    def _rec(self, name, x):
        if self.stats is not None:
            self.stats[name] = max(self.stats.get(name, 0.0), float(x.abs().max()))
        return x

    @staticmethod
    def _bn(sd, p, x):
        return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False, 0.0, 1e-5)

    def cbr(self, sd, conv, bn, x, stride=1, pad=0, dil=1, relu=True, name=None):
        y = self._bn(sd, bn, F.conv2d(x, sd[conv + ".weight"], None, stride, pad, dil))
        y = F.relu(y) if relu else y
        return self._rec(name or conv, y)

    def encoder(self, x):
        e = self.enc
        x = self.cbr(e, "conv1", "bn1", x, 2, 1)
        x = self.cbr(e, "conv2", "bn2", x, 1, 1)
        x = self.cbr(e, "conv3", "bn3", x, 1, 1)
        x = F.max_pool2d(x, 3, 2, 1)
        for layer, blocks, stride, dil in LAYERS:
            for b in range(blocks):
                p = "%s.%d" % (layer, b)
                s, d = (stride, max(dil // 2, 1)) if b == 0 else (1, dil)
                y = self.cbr(e, p + ".conv1", p + ".bn1", x)
                y = self.cbr(e, p + ".conv2", p + ".bn2", y, s, d, d)
                y = self.cbr(e, p + ".conv3", p + ".bn3", y, relu=False)
                r = self.cbr(e, p + ".downsample.0", p + ".downsample.1", x, s, relu=False) if b == 0 else x
                x = self._rec(p, F.relu(y + r))
        return x

    def decoder_logits(self, c5):
        d = self.dec
        h, w = c5.shape[2:]
        parts = [c5]
        for j, b in enumerate(BINS):
            y = self.cbr(d, "ppm.%d.1" % j, "ppm.%d.2" % j, F.adaptive_avg_pool2d(c5, b))
            parts.append(F.interpolate(y, (h, w), mode="bilinear", align_corners=False))
        x = self.cbr(d, "conv_last.0", "conv_last.1", torch.cat(parts, 1), 1, 1)
        return self._rec("logits", F.conv2d(x, d["conv_last.4.weight"], d["conv_last.4.bias"]))


def get_sky(enc, dec, img, segId=1, segFg=True, dtype=torch.float32, stats=None):
    """(mask float32 [H][W], pred int64 [H][W], scores [150][H][W] numpy in ``dtype``, pass sizes).  ``stats`` (dict): filled with
    each layer's max |activation|."""
    img = img.convert("RGB")
    W, H = img.size
    net = _Net(enc, dec, dtype, stats)
    sizes = pass_sizes(H, W)
    probs = {}
    with torch.no_grad():
        for hw in dict.fromkeys(sizes):
            logits = net.decoder_logits(net.encoder(_prep(img, hw[0], hw[1], dtype)))
            probs[hw] = torch.softmax(F.interpolate(logits, (H, W), mode="bilinear", align_corners=False), dim=1)
        scores = torch.zeros(1, probs[sizes[0]].shape[1], H, W, dtype=dtype)
        for hw in sizes:
            scores = scores + probs[hw] / 5
        pred = torch.max(scores, dim=1)[1][0]                           # first maximum on ties
    hit = (pred == segId).numpy().astype(np.float32)
    return (1 - hit if segFg else hit), pred.numpy(), scores[0].numpy(), sizes


def margins(scores, segId):
    """Per pixel: top-1 - top-2 score and top-1 - score[segId] (the tie proofs of a mask pixel)."""
    s = np.sort(scores, axis=0)
    return s[-1] - s[-2], s[-1] - scores[segId]
