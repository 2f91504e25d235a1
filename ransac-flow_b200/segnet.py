"""Mirror of the reference's segNet (segNet/segEval.py:6-43 ``SegNet``): the ADE20K scene-parsing network the evaluation drivers'
``--segNet`` option uses to keep the sky out of the matches (``CoarseAlign.skyFromSeg``).

The network is ``ResnetDilated(resnet50, dilate_scale=8)`` + ``PPMDeepsup`` (segNet/segModel.py:59-264) in inference:

  * encoder: one ``LayerProgram`` (deep stem, max-pool, layer1..4 with dilated 3x3 convolutions in layer3 / layer4) run as ONE
    ``rf_run_layers`` call over a ragged batch of every DISTINCT resized size of the image (the reference's five scales often repeat
    one size: 480 x 640 gives 304 x 400 once and 376 x 504 four times);
  * decoder: ``rf_adaptive_avgpool_split`` (the four PPM poolings), four 1x1 convolutions, ``rf_ppm_concat_split`` (conv5 + the
    upsampled branches), conv_last as a two-layer program whose 150-class 1x1 writes fp32 logits;
  * vote: ``rf_seg_vote`` adds each of the reference's five passes (repeats included, in order) as ``scores += softmax / 5`` per
    output pixel and writes the mask; the reference's five [150][H][W] score tensors never exist.

Everything runs on the split engine (engine 4: fp16 hi / lo operands, fp32-grade), whatever ``model.set_engine`` selects: the
dilated convolutions exist on that engine only.  Split tensors carry activations up to |x| <= 65504.
"""
import ctypes as C
import os

import numpy as np
import PIL.Image as Image
import torch

from . import ops
from ._lib import check, lib, ptr, stream
from .model import FoldedConv
from .ops import Ragged
from .program import LayerProgram

IMG_SIZES = (300, 375, 450, 525, 600)      # segEval.py:19 TestDataset(imgSizes, imgMaxSize=500, padding_constant=8)
IMG_MAX_SIZE = 500
PADDING = 8
NUM_CLASS = 150
POOL_SCALES = (1, 2, 3, 6)                 # segModel.py:220
PPM_CHANNELS = 512
# (layer, planes, blocks, stride, dilation of blocks 1..; block 0 has half of it) - ResnetDilated(dilate_scale=8), segModel.py:161-199
ENCODER_LAYERS = (("layer1", 64, 3, 1, 1), ("layer2", 128, 4, 2, 1), ("layer3", 256, 6, 1, 2), ("layer4", 512, 3, 1, 4))
ENCODER_PTH = "../../model/pretrained/ade20k_resnet50dilated_encoder.pth"       # relative to the driver's directory
DECODER_PTH = "../../model/pretrained/ade20k_resnet50dilated_decoder.pth"


class SegNetWeightsNotFound(FileNotFoundError, NotImplementedError):
    """No segNet checkpoint: a FileNotFoundError like the reference's ``torch.load``, and a NotImplementedError like the
    ``segNet=True`` refusal of earlier versions of this package."""


def _bn_keys(p):
    return [p + s for s in (".weight", ".bias", ".running_mean", ".running_var")]


def encoder_keys():
    """Every encoder checkpoint key the inference path reads."""
    keys = []
    for i in (1, 2, 3):
        keys += ["conv%d.weight" % i] + _bn_keys("bn%d" % i)
    for layer, _, blocks, _, _ in ENCODER_LAYERS:
        for b in range(blocks):
            p = "%s.%d" % (layer, b)
            for i in (1, 2, 3):
                keys += ["%s.conv%d.weight" % (p, i)] + _bn_keys("%s.bn%d" % (p, i))
            if b == 0:
                keys += [p + ".downsample.0.weight"] + _bn_keys(p + ".downsample.1")
    return keys


def decoder_keys():
    """Every decoder checkpoint key the inference path reads (not the deep-supervision branch)."""
    keys = []
    for j in range(len(POOL_SCALES)):
        keys += ["ppm.%d.1.weight" % j] + _bn_keys("ppm.%d.2" % j)
    return keys + ["conv_last.0.weight"] + _bn_keys("conv_last.1") + ["conv_last.4.weight", "conv_last.4.bias"]


def _select(sd, keys, what):
    """The keys the network reads, as fp32 host tensors; every other entry (deep supervision, SyncBN's ``_tmp_running_*`` /
    ``_running_iter``, ``num_batches_tracked``) is ignored.  A missing key is an error that names it."""
    missing = [k for k in keys if k not in sd]
    if missing:
        raise KeyError("segNet %s checkpoint lacks %d key(s) the network reads: %s" % (what, len(missing), ", ".join(missing[:8])))
    return {k: sd[k].detach().to(device="cpu", dtype=torch.float32) for k in keys}


def segnet_weights(state_dicts=None):
    """(encoderPth, decoderPth, state_dicts) for CoarseAlign(segNet=True): ``state_dicts`` = (encoder, decoder) if given, else
    ``$RF_SEGNET_ENCODER`` / ``$RF_SEGNET_DECODER``, else the reference's relative paths.  Raises SegNetWeightsNotFound."""
    if state_dicts is not None:
        return None, None, tuple(state_dicts)
    enc = os.environ.get("RF_SEGNET_ENCODER") or ENCODER_PTH
    dec = os.environ.get("RF_SEGNET_DECODER") or DECODER_PTH
    for p in (enc, dec):
        if not os.path.isfile(p):
            raise SegNetWeightsNotFound("segNet weights not found: %s (set $RF_SEGNET_ENCODER / $RF_SEGNET_DECODER, pass "
                                        "segnet_state_dicts=, or put the ADE20K checkpoints where the reference expects them)" % p)
    return enc, dec, None


def scale_sizes(H, W):
    """(h, w) of each of the reference's five passes (segData.py:60-68)."""
    out = []
    for s in IMG_SIZES:
        scale = min(s / float(min(H, W)), IMG_MAX_SIZE / float(max(H, W)))
        th, tw = int(H * scale), int(W * scale)
        out.append((((th - 1) // PADDING + 1) * PADDING, ((tw - 1) // PADDING + 1) * PADDING))
    return out


class _BN:
    def __init__(self, sd, p):
        self.weight, self.bias = sd[p + ".weight"], sd[p + ".bias"]
        self.running_mean, self.running_var = sd[p + ".running_mean"], sd[p + ".running_var"]
        self.eps = 1e-5                        # SynchronizedBatchNorm2d in eval = BatchNorm2d(eps=1e-5)


class SegNet:
    """segEval.SegNet(encoderPth, decoderPth, segId, segFg) on the library's kernels, always on the split engine (engine 4).
    ``state_dicts`` = (encoder, decoder) replaces the two checkpoint files."""

    def __init__(self, encoderPth, decoderPth, segId=1, segFg=True, state_dicts=None, device="cuda"):
        if state_dicts is None:
            state_dicts = (torch.load(encoderPth, map_location="cpu"), torch.load(decoderPth, map_location="cpu"))
        self.device = torch.device(device)
        self.segId, self.segFg = int(segId), bool(segFg)
        enc = _select(state_dicts[0], encoder_keys(), "encoder")
        dec = _select(state_dicts[1], decoder_keys(), "decoder")
        self.encoder = self._build_encoder(enc)
        dev = self.device
        self.ppm_convs = [FoldedConv(dec["ppm.%d.1.weight" % j], _BN(dec, "ppm.%d.2" % j), 1, pad=0, device=dev) for j in range(len(POOL_SCALES))]
        self.head = LayerProgram(2048 + len(POOL_SCALES) * PPM_CHANNELS, device=dev)
        x = self.head.conv(0, FoldedConv(dec["conv_last.0.weight"], _BN(dec, "conv_last.1"), 1, pad=1, device=dev), relu=True)
        last = FoldedConv(dec["conv_last.4.weight"], None, 1, pad=0, device=dev)
        last.bias = dec["conv_last.4.bias"].contiguous().to(dev)
        self.head.conv(x, last, relu=False, out_f32=True)              # Dropout2d is the identity in eval
        self._bins = _int_array(POOL_SCALES)

    def _build_encoder(self, sd):
        dev = self.device
        P = LayerProgram(3, device=dev)
        x = P.stem3(0, sd["conv1.weight"], _BN(sd, "bn1"))                        # 3x3 / 2, 3 -> 64, one fused kernel
        x = P.conv(x, FoldedConv(sd["conv2.weight"], _BN(sd, "bn2"), 1, pad=1, device=dev), relu=True)
        x = P.conv(x, FoldedConv(sd["conv3.weight"], _BN(sd, "bn3"), 1, pad=1, device=dev), relu=True)
        x = P.maxpool(x, 3, 2, 1)
        for layer, _, blocks, stride, dil in ENCODER_LAYERS:
            for b in range(blocks):
                p = "%s.%d" % (layer, b)
                s = stride if b == 0 else 1
                d = max(dil // 2, 1) if b == 0 else dil
                out = P.conv(x, FoldedConv(sd[p + ".conv1.weight"], _BN(sd, p + ".bn1"), 1, pad=0, device=dev), relu=True)
                out = P.conv(out, FoldedConv(sd[p + ".conv2.weight"], _BN(sd, p + ".bn2"), s, pad=d, device=dev), relu=True, dil=d)
                c3 = FoldedConv(sd[p + ".conv3.weight"], _BN(sd, p + ".bn3"), 1, pad=0, device=dev)
                if b == 0:              # conv3 + the 1x1 down-sampling branch (stride s; 1 in the dilated layers) + add + ReLU: one GEMM
                    ds = FoldedConv(sd[p + ".downsample.0.weight"], _BN(sd, p + ".downsample.1"), s, pad=0, device=dev)
                    x = P.conv_dual(out, x, FoldedConv.concat_k(c3, ds), s, relu=True)
                else:
                    x = P.conv(out, c3, relu=True, res=x)
        return P

    # -- stages (tools/segnet_profile.py times them one by one) -------------------------------------------------------------------
    @staticmethod
    def load(img):
        """segData.py:55: a path or a PIL image -> RGB PIL image."""
        return (Image.open(img) if isinstance(img, (str, os.PathLike)) else img).convert("RGB")

    def plan(self, H, W):
        """(distinct sizes in first-use order, the pass -> distinct-size index list)."""
        sizes = scale_sizes(H, W)
        distinct = list(dict.fromkeys(sizes))
        return distinct, [distinct.index(s) for s in sizes]

    def resize(self, u8, distinct):
        """PIL BILINEAR resizes of the uint8 [H, W, 3] CUDA image + ToTensor + Normalize (segData.py:33-38, 71-74) as one ragged
        fp32 batch."""
        imgs = [ops.resize_bilinear_u8(u8, w, h) for (h, w) in distinct]
        flat = torch.cat([t.reshape(-1, 3) for t in imgs], dim=0) if len(imgs) > 1 else imgs[0].reshape(-1, 3)
        return Ragged(ops.preproc_u8(flat, normalize=True), distinct)

    def encode(self, x):
        """ResnetDilated: ragged fp32 images -> conv5, split [2][sum HW / 64][2048] (a view of the program's buffer)."""
        out, ohw = self.encoder.run(x, ops.ENGINE_SPLIT)
        return Ragged(out, ohw)

    def ppm(self, conv5):
        """PPMDeepsup's pyramid pooling (segModel.py:249-256): split [2][sum HW][2048 + 4 * 512]."""
        n, dev = conv5.n, conv5.data.device
        pooled = [torch.empty((2, n * b * b, conv5.C), device=dev, dtype=torch.float16) for b in POOL_SCALES]
        check(lib.rf_adaptive_avgpool_split(ptr(conv5.data), n, conv5._c, conv5.C, self._bins, len(POOL_SCALES),
                                            _ptr_array(pooled), stream()))
        branches = [ops.conv2d(Ragged(t, [(b, b)] * n), fc.w, fc.bias, PPM_CHANNELS, 1, 1, 0, True, None, ops.ENGINE_SPLIT, fc.w_split).data
                    for t, b, fc in zip(pooled, POOL_SCALES, self.ppm_convs)]
        cat = torch.empty((2, conv5.data.shape[1], self.head.chan[0]), device=dev, dtype=torch.float16)
        check(lib.rf_ppm_concat_split(ptr(conv5.data), n, conv5._c, conv5.C, _ptr_array(branches), self._bins, len(POOL_SCALES),
                                      PPM_CHANNELS, ptr(cat), stream()))
        return Ragged(cat, conv5.hw)

    def conv_last(self, cat):
        """conv_last (segModel.py:235-242, 258): fp32 logits [sum HW][150] (a view of the program's buffer)."""
        out, ohw = self.head.run(cat, ops.ENGINE_SPLIT)
        return Ragged(out, ohw)

    def vote(self, logits, order, H, W, want_class=False, want_scores=False):
        """segEval.py:28-43: (mask float32 [H][W], class map int32 or None, scores [H][W][150] or None) on the device."""
        dev = logits.data.device
        mask = torch.empty((H, W), device=dev, dtype=torch.float32)
        cls = torch.empty((H, W), device=dev, dtype=torch.int32) if want_class else None
        scores = torch.empty((H, W, NUM_CLASS), device=dev, dtype=torch.float32) if want_scores else None
        check(lib.rf_seg_vote(ptr(logits.data), logits.n, logits._c, NUM_CLASS, _int_array(order), len(order), H, W, self.segId,
                              int(self.segFg), ptr(mask), ptr(cls), ptr(scores), stream()))
        return mask, cls, scores

    def run(self, img, want_class=False, want_scores=False):
        """The whole of getSky on the device: (mask, class map, scores) as in ``vote``."""
        img = self.load(img)
        W, H = img.size
        u8 = torch.from_numpy(np.array(img, dtype=np.uint8)).to(self.device)
        distinct, order = self.plan(H, W)
        with torch.no_grad():
            logits = self.conv_last(self.ppm(self.encode(self.resize(u8, distinct))))
            return self.vote(logits, order, H, W, want_class, want_scores)

    def getSky(self, imgPath):
        """segEval.py:23-43: float32 [H][W] numpy mask, (pred == segId) or 1 - that when segFg."""
        return self.run(imgPath)[0].cpu().numpy()


def _int_array(vals):
    return (C.c_int * len(vals))(*[int(v) for v in vals])


def _ptr_array(tensors):
    return (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
