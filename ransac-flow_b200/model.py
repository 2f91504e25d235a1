"""Drop-in for the reference's ``model`` module (model/model.py): same class names,
constructor arguments, ``state_dict`` keys and call signatures; ``forward`` runs the
library's CUDA kernels (inference only - the training path is out of scope).

The ``nn.Conv2d`` / ``nn.BatchNorm2d`` children are parameter containers only, so
``load_state_dict(torch.load(resumePth)[key])`` works unchanged
(quick_start/align2images.py:47-50).  BatchNorm (eval, eps 1e-5) is folded into the
preceding bias-free convolution when the weights are first used.
"""
import torch
import torch.nn as nn

from . import ops
from .ops import Ragged
from .program import LayerProgram

_engine = ops.ENGINE_FP32


def set_engine(engine):
    """'fp32' (exact FMA, SIMT), 'f16x3' (wgmma tensor cores with fp16 hi / lo split operands and activations: fp32-GRADE,
    22 significand bits, three MMAs per MAC - the engine that reproduces the reference's fp32 match set), 'tf32' (wgmma,
    fp32 activations, 10-bit operands), 'f16' (wgmma with fp16 activations: the fast, reduced-precision mode; the 49- /
    1-channel head outputs stay TF32 / fp32) or 'f16-trunk' (fp16 trunk only, fine-flow networks on 'tf32')."""
    global _engine, _fine_f16
    _fine_f16 = engine != "f16-trunk"
    _engine = ({"fp32": ops.ENGINE_FP32, "tf32": ops.ENGINE_TF32, "f16": ops.ENGINE_F16, "f16-trunk": ops.ENGINE_F16,
                "f16x3": ops.ENGINE_SPLIT}[engine] if isinstance(engine, str) else int(engine))


def get_engine():
    return _engine


_fine_f16 = True


def fine_engine():
    """Engine of FeatureExtractor / NetFlowCoarse / NetMatchability ('f16-trunk' keeps them on 'tf32')."""
    return _engine if (_engine != ops.ENGINE_F16 or _fine_f16) else ops.ENGINE_TF32


def conv3x3(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False)


def conv1x1(in_planes, out_planes, stride=1):
    return nn.Conv2d(in_planes, out_planes, kernel_size=1, stride=stride, bias=False)


def _init_like_reference(module):
    # model/model.py:75-84
    for m in module.modules():
        if isinstance(m, nn.Conv2d):
            nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
        elif isinstance(m, nn.BatchNorm2d):
            nn.init.constant_(m.weight, 1)
            nn.init.constant_(m.bias, 0)


class FoldedConv:
    """conv weight (+ following eval-mode BatchNorm) packed for the kernels."""

    def __init__(self, weight, bn=None, stride=1, pad=None, eps=None, cin_pad=None, device=None):
        # folding and packing run on the HOST (a few hundred KB per layer, once per model): no swarm of tiny elementwise
        # launches in front of the first pair, one H2D copy per packed tensor
        dev = weight.device if device is None else torch.device(device)
        w = weight.detach().float().cpu()
        if cin_pad is not None and cin_pad > w.shape[1]:          # zero input channels (49 -> 64 for the heads)
            w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, cin_pad - w.shape[1]))
        cout, cin, k, _ = w.shape
        if bn is not None:
            e = bn.eps if eps is None else eps
            scale = bn.weight.detach().float().cpu() / torch.sqrt(bn.running_var.detach().float().cpu() + e)
            self.bias = (bn.bias.detach().float().cpu() - bn.running_mean.detach().float().cpu() * scale).contiguous().to(dev)
            w = w * scale.view(-1, 1, 1, 1)
        else:
            self.bias = None
        self.w = w.permute(2, 3, 1, 0).reshape(k * k * cin, cout).contiguous().to(dev)      # [R*S*Cin][Cout]
        # tensor-core copy: [Cout][R*S*Cin], rounded to nearest-even TF32 once (the MMA would truncate)
        wt = w.permute(0, 2, 3, 1).reshape(cout, k * k * cin).contiguous()
        bits = wt.view(torch.int32)
        bits = (bits + 0xFFF + ((bits >> 13) & 1)) & ~0x1FFF
        self.w_tc = bits.view(torch.float32).contiguous().to(dev)
        self._wt = wt                                                                        # host copy: source of the fp16 / split packings
        self._dev = dev
        self._w_f16 = None
        self.cout, self.cin, self.k, self.stride = cout, cin, k, stride
        self.pad = (k // 2) if pad is None else pad

    @classmethod
    def concat_k(cls, fa, fb):
        """Two folded 1x1 convolutions with the same output channels as ONE whose K axis is [fa's inputs | fb's inputs] and whose
        bias is the sum: y = fa(x1) + fb(x2) (LayerProgram.conv_dual; fb's stride is applied by the kernel to its input)."""
        assert fa.k == 1 and fb.k == 1 and fa.cout == fb.cout and fa.pad == 0 and fb.pad == 0
        f = cls.__new__(cls)
        f._wt = torch.cat([fa._wt, fb._wt], dim=1).contiguous()
        f._dev, f._w_f16 = fa._dev, None
        f.w = torch.cat([fa.w, fb.w], dim=0).contiguous()
        f.w_tc = torch.cat([fa.w_tc, fb.w_tc], dim=1).contiguous()
        ba = fa.bias if fa.bias is not None else torch.zeros(fa.cout, device=fa._dev)
        f.bias = (ba + fb.bias) if fb.bias is not None else ba
        f.cout, f.cin, f.cin2, f.k, f.stride, f.pad = fa.cout, fa.cin, fb.cin, 1, 1, 0
        return f

    @property
    def w_split(self):
        """[2][Cout][R*S*Cin] fp16: hi = fp16(w), lo = fp16((w - hi) * 2^11) - the engine-4 operand; built on first use."""
        if getattr(self, "_w_split", None) is None:
            hi = self._wt.to(torch.float16)
            lo = ((self._wt - hi.float()) * 2048.0).to(torch.float16)
            self._w_split = torch.stack([hi, lo]).contiguous().to(self._dev)
        return self._w_split

    @property
    def w_f16(self):
        """[Cout][R*S*Cin] fp16 (round to nearest), the engine-2 operand; built on first use."""
        if self._w_f16 is None:
            self._w_f16 = self._wt.to(torch.float16).contiguous().to(self._dev)
        return self._w_f16

    def __call__(self, x, relu, residual=None, engine=None):
        eng = min(fine_engine(), ops.ENGINE_TF32) if engine is None else engine     # fp32 activations here; the library keeps unsupported shapes on the FMA engine
        if int(eng) == ops.ENGINE_SPLIT:
            return ops.conv2d(x, self.w, self.bias, self.cout, self.k, self.stride, self.pad, relu, residual, eng, self.w_split)
        return ops.conv2d(x, self.w, self.bias, self.cout, self.k, self.stride, self.pad, relu, residual, eng, self.w_tc)


class _Engine(nn.Module):
    """Caches folded weights; rebuilt whenever parameters change or move."""

    def _folded(self, f16=False):
        """The layer program for fp32 activations (False / 0), the fp16 engine (True / 2) or the split engine (4)."""
        f16 = 2 if f16 is True else (int(f16) if int(f16) in (ops.ENGINE_F16, ops.ENGINE_SPLIT) else 0)
        ver = tuple((p._version, p.data_ptr()) for p in list(self.parameters()) + list(self.buffers()))
        if getattr(self, "_fold_ver", None) != ver:
            self._fold = {}
            self._fold_ver = ver
        if f16 not in self._fold:
            with torch.no_grad():
                self._fold[f16] = self._fold_build(f16)
        return self._fold[f16]

    def _check(self, *xs):
        if self.training:
            raise RuntimeError("ransac_flow_b200.model is inference-only: call .eval() first (training is out of scope)")
        for x in xs:
            ops.need_cuda(x)


class Downsample(nn.Module):
    """model/downsample.py:12-46 as a parameter container (buffer ``filt``)."""

    def __init__(self, pad_type="reflect", filt_size=3, stride=2, channels=None, pad_off=0):
        super().__init__()
        assert filt_size == 3 and pad_type in ("refl", "reflect") and pad_off == 0, "only the configuration the hot path uses"
        self.stride, self.channels = stride, channels
        a = torch.tensor([1.0, 2.0, 1.0])
        filt = a[:, None] * a[None, :]
        self.register_buffer("filt", (filt / filt.sum())[None, None].repeat(channels, 1, 1, 1))


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = conv3x3(inplanes, planes, stride)
        self.bn1 = nn.BatchNorm2d(planes, eps=1e-05)
        self.conv2 = conv3x3(planes, planes)
        self.bn2 = nn.BatchNorm2d(planes, eps=1e-05)
        self.downsample = downsample
        self.stride = stride


class FeatureExtractor(_Engine):
    """model/model.py:59-125.  (N,3,H,W) -> (N,256,H/8,W/8)."""

    def __init__(self):
        super().__init__()
        self.inplanes = 64
        self.conv1 = nn.Conv2d(3, 64, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(64, eps=1e-05)
        self.maxpool = nn.Sequential(nn.MaxPool2d(kernel_size=2, stride=1), Downsample(filt_size=3, stride=2, channels=64))
        self.layer1 = self._make_layer(BasicBlock, 64, 2)
        self.layer2 = self._make_layer(BasicBlock, 128, 2, stride=2)
        self.layer3 = self._make_layer(BasicBlock, 256, 2, stride=2)
        _init_like_reference(self)

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = [Downsample(filt_size=3, stride=stride, channels=self.inplanes)] if stride != 1 else []
            downsample += [conv1x1(self.inplanes, planes * block.expansion, 1), nn.BatchNorm2d(planes * block.expansion)]
            downsample = nn.Sequential(*downsample)
        layers = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes, 1, None))
        return nn.Sequential(*layers)

    def _fold_build(self, f16=False):
        """The whole network as one layer program (model/model.py:106-114 do_forward)."""
        P = LayerProgram(3)
        if f16:
            x = P.stem7_fused(0, self.conv1.weight, self.bn1)                        # conv1 + bn1 + relu, patches gathered on chip
        else:
            x = P.stem(0, self.conv1.weight, self.bn1, 1, 1)                         # conv1 + bn1 + relu as im2col + 1x1
        x = P.poolblur(x)                                                            # MaxPool2d(2, 1) + anti-aliased stride 2, fused
        for layer in (self.layer1, self.layer2, self.layer3):
            for b in layer:
                out = P.conv(x, FoldedConv(b.conv1.weight, b.bn1, b.stride), relu=True)
                r = x
                if b.downsample is not None:
                    mods = list(b.downsample)
                    if isinstance(mods[0], Downsample):
                        r = P.blur(r, mods[0].stride)
                    r = P.conv(r, FoldedConv(mods[-2].weight, mods[-1], 1, pad=0), relu=False)
                x = P.conv(out, FoldedConv(b.conv2.weight, b.bn2, 1), relu=True, res=r)   # conv2 + bn2 + residual + relu
        return P

    def forward_ragged(self, x):
        """Ragged [P, 3] -> Ragged [P/64, 256].  The returned buffer is owned by the program and valid until
        the next forward with the same image sizes; callers normalise / copy it right away."""
        eng = fine_engine()
        out, ohw = self._folded(eng).run(x, eng)
        return Ragged(out, ohw)                 # fp16 rows / split planes under the tensor-core engines (ops.l2norm returns fp32 either way)

    def forward(self, x):
        self._check(x)
        with torch.no_grad():
            r = self.forward_ragged(Ragged.from_nchw(x))
            if r.split:
                r = Ragged(ops.from_split(r.data), r.hw)
            return r.to_nchw().float().clone(memory_format=torch.channels_last)


class CorrNeigh(nn.Module):
    """model/model.py:129-160."""

    def __init__(self, kernelSize):
        super().__init__()
        assert kernelSize % 2 == 1
        self.kernelSize = kernelSize
        self.paddingSize = kernelSize // 2

    def forward(self, x, y):
        ops.need_cuda(x, y)
        with torch.no_grad():
            return ops.corr_neigh(Ragged.from_nchw(x), Ragged.from_nchw(y), self.kernelSize).to_nchw()


class _Head(_Engine):
    def __init__(self, kernelSize, cout):
        super().__init__()
        assert kernelSize % 2 == 1
        self.conv1 = conv3x3(kernelSize * kernelSize, 512)
        self.bn1 = nn.BatchNorm2d(512, eps=1e-05)
        self.conv2 = conv3x3(512, 256)
        self.bn2 = nn.BatchNorm2d(256, eps=1e-05)
        self.conv3 = conv3x3(256, 128)
        self.bn3 = nn.BatchNorm2d(128, eps=1e-05)
        self.conv4 = conv3x3(128, cout)
        self.kernelSize = kernelSize
        self.paddingSize = kernelSize // 2
        _init_like_reference(self)

    CORR_LD = 64      # the k*k = 49-channel correlation volume is carried with 64 channels (15 zeros)

    def _fold_build(self, f16=False):
        # under the fp16 engine conv1..conv3 read fp16; conv3 writes fp32 and the 49- / 1-channel conv4 stays on TF32.  Under the
        # split engine all four layers are split-operand convolutions and conv4 writes plain fp32 rows
        P = LayerProgram(self.CORR_LD)
        split = f16 == 4
        x = P.conv(0, FoldedConv(self.conv1.weight, self.bn1, cin_pad=self.CORR_LD), relu=True)
        x = P.conv(x, FoldedConv(self.conv2.weight, self.bn2), relu=True)
        x = P.conv(x, FoldedConv(self.conv3.weight, self.bn3), relu=True, out_f32=not split)
        P.conv(x, FoldedConv(self.conv4.weight, None), relu=False, tf32=not split, out_f32=split)
        return P

    def _padded(self, corr, dtype, split=False):
        """Accept the reference's 49-channel volume or the library's 64-channel one (fp32, fp16 for the fp16 engine, split
        planes for the split engine)."""
        if corr.C == self.CORR_LD and corr.data.dtype == dtype and corr.split == split:
            return corr
        if split:
            src = ops.from_split(corr.data) if corr.split else corr.data.float()
            d = torch.zeros((src.shape[0], self.CORR_LD), device=src.device, dtype=torch.float32)
            d[:, :min(src.shape[1], self.kernelSize ** 2)] = src[:, :self.kernelSize ** 2]
            return Ragged(ops.to_split(d), corr.hw)
        d = torch.zeros((corr.data.shape[0], self.CORR_LD), device=corr.data.device, dtype=dtype)
        d[:, :min(corr.C, self.kernelSize ** 2)] = corr.data[:, :self.kernelSize ** 2].to(dtype)
        return Ragged(d, corr.hw)

    def trunk(self, corr):
        eng = fine_engine()
        f16, split = eng == ops.ENGINE_F16, eng == ops.ENGINE_SPLIT
        corr = self._padded(corr, torch.float16 if (f16 or split) else torch.float32, split)
        out, ohw = self._folded(eng).run(corr, eng)
        return Ragged(out, ohw)


class NetFlowCoarse(_Head):
    """model/model.py:167-249."""

    def __init__(self, kernelSize):
        super().__init__(kernelSize, kernelSize * kernelSize)
        r = self.paddingSize
        self.gridY = torch.arange(-r, r + 1).view(1, 1, -1, 1).expand(1, 1, kernelSize, kernelSize).contiguous().view(1, -1, 1, 1).float()
        self.gridX = torch.arange(-r, r + 1).view(1, 1, 1, -1).expand(1, 1, kernelSize, kernelSize).contiguous().view(1, -1, 1, 1).float()

    def cuda(self, device=None):
        super().cuda(device)
        self.gridX, self.gridY = self.gridX.cuda(), self.gridY.cuda()
        return self     # the reference returns None here (model/model.py:205-207); callers ignore the value

    def forward_ragged(self, corr):
        return ops.softmax_flow(self.trunk(corr), self.kernelSize)

    def forward(self, coef, up8X=True):
        self._check(coef)
        with torch.no_grad():
            flow = self.forward_ragged(Ragged.from_nchw(coef))
            if up8X:                                   # F.upsample_bilinear == align_corners=True; not used at inference
                flow = torch.nn.functional.interpolate(flow, scale_factor=8, mode="bilinear", align_corners=True)
            return flow


class NetMatchability(_Head):
    """model/model.py:254-322."""

    def __init__(self, kernelSize):
        super().__init__(kernelSize, 1)
        nn.init.normal_(self.conv4.weight, mean=0.0, std=0.0001)

    def forward_ragged(self, corr):
        x = self.trunk(corr)                                # [P, 1]
        h, w = corr.hw[0]
        return ops.sigmoid(x.data).view(corr.n, 1, h, w)

    def forward(self, feat, up8X=True):
        self._check(feat)
        with torch.no_grad():
            m = self.forward_ragged(Ragged.from_nchw(feat))
            if up8X:
                m = torch.nn.functional.interpolate(m, scale_factor=8, mode="bilinear", align_corners=True)
            return m


def predFlowCoarse(corrKernel21, NetFlowCoarse, grid, up8X=True):
    """model/model.py:331-340."""
    flowCoarse = NetFlowCoarse(corrKernel21, up8X)
    b, _, w, h = flowCoarse.size()
    flowGrad = flowCoarse.narrow(2, 1, w - 1).narrow(3, 1, h - 1) - flowCoarse.narrow(2, 0, w - 1).narrow(3, 0, h - 1)
    flowGrad = torch.norm(flowGrad, dim=1, keepdim=True)
    flowCoarse = flowCoarse.permute(0, 2, 3, 1)
    flowCoarse = torch.clamp(flowCoarse + grid, min=-1, max=1)
    return flowGrad, flowCoarse


def predFlowCoarseNoGrad(corrKernel21, NetFlowCoarse, grid, up8X=True):
    """model/model.py:342-350."""
    flowCoarse = NetFlowCoarse(corrKernel21, up8X).permute(0, 2, 3, 1)
    return torch.clamp(flowCoarse + grid, min=-1, max=1)


def predMatchability(corrKernel21, NetMatchability, up8X=True):
    """model/model.py:353-357."""
    return NetMatchability(corrKernel21, up8X)
