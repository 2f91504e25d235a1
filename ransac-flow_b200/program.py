"""Layer programs: a network (list of conv / pool / blur layers with folded weights) compiled for one
image-set signature and executed by ONE call into the library (``rf_run_layers``).

The topology is written in Python next to the mirror of the reference module it belongs to
(model.py, coarseAlignFeatMatch.py); this class only assigns buffer slots, sizes and caches the
activation buffers (stable device pointers => the library's TMA-descriptor cache always hits).
"""
import ctypes as C

import torch

from ._lib import check, lib, need_cuda, stream

RF_OP_CONV, RF_OP_MAXPOOL, RF_OP_BLUR, RF_OP_IM2COL, RF_OP_POOLBLUR, RF_OP_STEM7, RF_OP_CONV_DUAL, RF_OP_STEM3 = 0, 1, 2, 3, 4, 5, 6, 7
RF_MAX_SLOTS = 32
RF_LAYER_OUT_F32, RF_LAYER_TF32, RF_LAYER_STEM_POOL = 1, 2, 4


class rf_layer_t(C.Structure):
    _fields_ = [("op", C.c_int), ("src", C.c_int), ("dst", C.c_int), ("res", C.c_int),
                ("Cin", C.c_int), ("Cout", C.c_int), ("k", C.c_int), ("stride", C.c_int), ("pad", C.c_int), ("relu", C.c_int),
                ("w", C.c_void_p), ("w_tc", C.c_void_p), ("bias", C.c_void_p), ("w_f16", C.c_void_p), ("flags", C.c_int),
                ("src2", C.c_int), ("Cin2", C.c_int), ("stride2", C.c_int), ("dil", C.c_int)]


lib.rf_run_layers.restype = C.c_int
lib.rf_run_layers.argtypes = [C.POINTER(rf_layer_t), C.c_int, C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_int), C.c_int, C.c_void_p]


class LayerProgram:
    """Symbolic tensors are integers; tensor 0 is the input."""

    def __init__(self, cin, device=None):
        self.device = device     # where folded weights built by stem() / stem7_fused() go (default: the weight's own device)
        self.ops = []            # (op, src, res, cin, cout, k, stride, pad, relu, folded)
        self.chan = [cin]
        self._keep = []          # folded weights (keeps the device tensors alive)
        self.flags = {}          # op index -> RF_LAYER_* (fp16 engine only)
        self.dual = {}           # op index -> (second input tensor, its channels, its stride)   (RF_OP_CONV_DUAL, split engine only)
        self.dil = {}            # op index -> dilation of a 3x3 / stride-1 conv (split engine only)
        self._compiled = {}

    # -- topology --------------------------------------------------------------------------------
    def conv(self, src, fc, relu, res=None, out_f32=False, tf32=False, dil=1):
        """``out_f32`` / ``tf32`` only matter under the fp16 engine: the layer that hands fp32 to a TF32 layer, and that
        TF32 layer (fp32 in and out; e.g. the 49- / 1-channel head outputs, which stay fp32).  ``dil`` > 1: a dilated 3x3 /
        stride-1 convolution (split engine only)."""
        assert self.chan[src] == fc.cin, (self.chan[src], fc.cin)
        if dil > 1:
            assert fc.k == 3 and fc.stride == 1 and not (out_f32 or tf32), "dilation: 3x3 / stride 1 layers with split outputs"
            self.split_only = True
        self.dil[len(self.ops)] = int(dil)
        self.flags[len(self.ops)] = (RF_LAYER_OUT_F32 if out_f32 else 0) | (RF_LAYER_TF32 if tf32 else 0)
        self.ops.append((RF_OP_CONV, src, -1 if res is None else res, fc.cin, fc.cout, fc.k, fc.stride, fc.pad, int(relu), fc))
        self._keep.append(fc)
        self.chan.append(fc.cout)
        return len(self.chan) - 1

    def conv_dual(self, src, src2, fc, stride2, relu):
        """Split engine only: 1x1 conv over [src | src2 sampled with stride2] (``fc`` = FoldedConv.concat_k(conv3, downsample)):
        a bottleneck's conv3 + its down-sampling branch + the add + ReLU in one GEMM."""
        assert fc.k == 1 and self.chan[src] == fc.cin and self.chan[src2] == fc.cin2, (self.chan[src], self.chan[src2], fc.cin, fc.cin2)
        self.dual[len(self.ops)] = (src2, fc.cin2, stride2)
        self.ops.append((RF_OP_CONV_DUAL, src, -1, fc.cin, fc.cout, 1, 1, 0, int(relu), fc))
        self._keep.append(fc)
        self.chan.append(fc.cout)
        self.split_only = True
        return len(self.chan) - 1

    def maxpool(self, src, k, stride, pad):
        c = self.chan[src]
        self.ops.append((RF_OP_MAXPOOL, src, -1, c, c, k, stride, pad, 0, None))
        self.chan.append(c)
        return len(self.chan) - 1

    def poolblur(self, src):
        """MaxPool2d(2, stride 1) + anti-aliased stride-2 blur in one pass (same output size rule as k=4, s=2, p=1)."""
        c = self.chan[src]
        self.ops.append((RF_OP_POOLBLUR, src, -1, c, c, 4, 2, 1, 0, None))
        self.chan.append(c)
        return len(self.chan) - 1

    def im2col(self, src, k, stride, pad, kpad):
        """k x k patches of a few-channel image as rows of ``kpad`` floats (the stem becomes a 1x1 conv)."""
        c = self.chan[src]
        assert kpad >= k * k * c
        self.ops.append((RF_OP_IM2COL, src, -1, c, kpad, k, stride, pad, 0, None))
        self.chan.append(kpad)
        return len(self.chan) - 1

    def stem(self, src, weight, bn, stride, pad, kalign=32):
        """conv(k x k, few input channels) + BN + ReLU as im2col + 1x1 conv (tensor-core friendly).  ``kalign`` = channels
        per 128-byte K block of the engine that will run the program (32 fp32, 64 fp16)."""
        from .model import FoldedConv
        cout, cin, k, _ = weight.shape
        kpad = (k * k * cin + kalign - 1) // kalign * kalign
        dev = self.device or weight.device
        w = weight.detach().float().cpu().permute(0, 2, 3, 1).reshape(cout, k * k * cin)    # (r, s, c) order
        w = torch.nn.functional.pad(w, (0, kpad - k * k * cin)).reshape(cout, kpad, 1, 1)
        x = self.im2col(src, k, stride, pad, kpad)
        return self.conv(x, FoldedConv(w, bn, 1, pad=0, device=dev), relu=True)

    def stem7_fused(self, src, weight, bn):
        """fp16 engine only: the ResNet-50 stem (7x7 / 2 / pad 3, 3 -> 64, BN, ReLU) in one kernel that builds the patches
        in shared memory (no im2col matrix in HBM).  Same packed weights as ``stem(kalign=64)``."""
        from .model import FoldedConv
        cout, cin, k, _ = weight.shape
        assert (cout, cin, k) == (64, 3, 7) and self.chan[src] == 3
        dev = self.device or weight.device
        w = weight.detach().float().cpu().permute(0, 2, 3, 1).reshape(cout, k * k * cin)
        w = torch.nn.functional.pad(w, (0, 192 - k * k * cin)).reshape(cout, 192, 1, 1)
        fc = FoldedConv(w, bn, 1, pad=0, device=dev)
        self.ops.append((RF_OP_STEM7, src, -1, 3, 64, 7, 2, 3, 1, fc))
        self._keep.append(fc)
        self.chan.append(64)
        self.f16_only = True
        return len(self.chan) - 1

    def stem3(self, src, weight, bn):
        """Split engine only: segNet's deep-stem conv1 (3x3 / 2 / pad 1, 3 -> 64, BN, ReLU) in one exact-fp32 kernel that reads the
        fp32 image and writes split rows (no patch matrix)."""
        from .model import FoldedConv
        assert tuple(weight.shape) == (64, 3, 3, 3) and self.chan[src] == 3
        fc = FoldedConv(weight, bn, 2, pad=1, device=self.device or weight.device)
        self.ops.append((RF_OP_STEM3, src, -1, 3, 64, 3, 2, 1, 1, fc))
        self._keep.append(fc)
        self.chan.append(64)
        self.split_only = True
        return len(self.chan) - 1

    def blur(self, src, stride):
        c = self.chan[src]
        self.ops.append((RF_OP_BLUR, src, -1, c, c, 3, stride, 1, 0, None))
        self.chan.append(c)
        return len(self.chan) - 1

    # -- compilation for one image-set signature --------------------------------------------------
    def _compile(self, hw, device, f16=False, split=False):
        n_t = len(self.chan)
        last_use = [0] * n_t
        for i, o in enumerate(self.ops):
            last_use[o[1]] = i
            if o[2] >= 0:
                last_use[o[2]] = i
            if i in self.dual:
                last_use[self.dual[i][0]] = i
        last_use[n_t - 1] = len(self.ops)                       # the output outlives the program
        # pixel counts per tensor
        hws = [list(hw)]
        for i, o in enumerate(self.ops):
            k, s, p, d = o[5], o[6], o[7], self.dil.get(i, 1)
            hws.append([((h + 2 * p - d * (k - 1) - 1) // s + 1, (w + 2 * p - d * (k - 1) - 1) // s + 1) for h, w in hws[o[1]]])
        # element size per tensor: fp32 everywhere, except under the fp16 engine (fp32 only for the image an im2col
        # reads and around RF_LAYER_OUT_F32 / RF_LAYER_TF32 convs)
        esize = [4] * n_t          # engine 4: split tensors are 2 fp16 planes = 4 bytes per element, like the fp32 image / OUT_F32 outputs
        if f16:
            esize[0] = 4 if self.ops[0][0] in (RF_OP_IM2COL, RF_OP_STEM7) else 2
            for i, o in enumerate(self.ops):
                fl = self.flags.get(i, 0)
                esize[i + 1] = 4 if fl else 2
                if fl & RF_LAYER_TF32:
                    assert esize[o[1]] == 4, "a TF32 layer under the fp16 engine needs an fp32 input (out_f32 on its producer)"
                elif o[0] not in (RF_OP_IM2COL, RF_OP_STEM7):
                    assert esize[o[1]] == 2 and (o[2] < 0 or esize[o[2]] == 2), "fp16 layer fed by an fp32 tensor"
        elems = [sum(h * w for h, w in hws[t]) * self.chan[t] * esize[t] for t in range(n_t)]        # BYTES per tensor
        # the stem and a 3x3 / stride 2 / pad 1 max-pool that is its only reader run as one kernel (engines 2 / 4): the stem's
        # full-resolution output is never written, so it sizes no buffer (its layer keeps a nominal slot for the wiring)
        stem_pool = set()
        for i, o in enumerate(self.ops[:-1]):
            q = self.ops[i + 1]
            if (f16 or split) and o[0] == RF_OP_STEM7 and q[0] == RF_OP_MAXPOOL and q[1] == i + 1 and tuple(q[5:8]) == (3, 2, 1) \
                    and last_use[i + 1] == i + 1:
                stem_pool.add(i)
                elems[i + 1] = 0
        # slot assignment: slot 0 = external input; others from a free list
        slot_of, free, slot_elems = {0: 0}, [], [0]
        layers = (rf_layer_t * len(self.ops))()
        for i, o in enumerate(self.ops):
            t_out = i + 1
            # choose a free slot (prefer the smallest that fits, else the largest one and grow it)
            if free:
                fit = [s for s in free if slot_elems[s] >= elems[t_out]]
                s = min(fit, key=lambda q: slot_elems[q]) if fit else max(free, key=lambda q: slot_elems[q])
                free.remove(s)
                slot_elems[s] = max(slot_elems[s], elems[t_out])
            else:
                s = len(slot_elems)
                slot_elems.append(elems[t_out])
            slot_of[t_out] = s
            L = layers[i]
            L.op, L.src, L.dst, L.res = o[0], slot_of[o[1]], s, (slot_of[o[2]] if o[2] >= 0 else -1)
            L.Cin, L.Cout, L.k, L.stride, L.pad, L.relu = o[3], o[4], o[5], o[6], o[7], o[8]
            fc = o[9]
            if fc is not None:
                L.w, L.w_tc = fc.w.data_ptr(), fc.w_tc.data_ptr()
                L.w_f16 = fc.w_f16.data_ptr() if f16 else (fc.w_split.data_ptr() if split else None)
                L.flags = (self.flags.get(i, 0) | (RF_LAYER_STEM_POOL if i in stem_pool else 0)) if (f16 or split) else 0
                L.bias = fc.bias.data_ptr() if fc.bias is not None else None
            L.src2 = -1
            L.dil = self.dil.get(i, 1)
            if i in self.dual:
                L.src2, L.Cin2, L.stride2 = slot_of[self.dual[i][0]], self.dual[i][1], self.dual[i][2]
            for t in {o[1], o[2], self.dual[i][0] if i in self.dual else -1}:
                if t > 0 and last_use[t] == i:
                    free.append(slot_of[t])
        assert len(slot_elems) <= RF_MAX_SLOTS
        bufs = [None] + [torch.empty(max(16, e), device=device, dtype=torch.uint8) for e in slot_elems[1:]]       # bytes
        out_slot = slot_of[n_t - 1]
        chw = (C.c_int * (2 * len(hw)))(*[v for p in hw for v in p])
        out_split = split and not (self.flags.get(len(self.ops) - 1, 0) & RF_LAYER_OUT_F32)
        in_split = split and self.ops[0][0] not in (RF_OP_IM2COL, RF_OP_STEM7, RF_OP_STEM3)
        return dict(layers=layers, bufs=bufs, out_slot=out_slot, out_hw=hws[-1], out_elems=elems[-1], chw=chw, nslots=len(slot_elems),
                    out_dtype=torch.float16 if (esize[-1] == 2 or out_split) else torch.float32, out_split=out_split,
                    in_dtype=torch.float16 if (esize[0] == 2 or in_split) else torch.float32)

    def run(self, x, engine):
        """x: ops.Ragged input -> (output buffer view [P_out, C_out] valid until the next run, out_hw)."""
        need_cuda(x.data)
        f16, split = int(engine) == 2, int(engine) == 4
        assert f16 or split or not getattr(self, "f16_only", False), "this program uses tensor-core-engine-only layers"
        assert split or not getattr(self, "split_only", False), "this program uses split-engine-only layers (conv_dual, dilation)"
        key = (tuple(x.hw), str(x.data.device), int(engine) if (f16 or split) else 0)
        if key not in self._compiled:
            # compiled entries own the activation buffers; captured CUDA graphs hold raw pointers into them, so entries are
            # never evicted behind a live graph's back: the cache only grows (one entry per image-set signature; callers with
            # many sizes bound it with `release()` once no graph / result refers to the buffers any more)
            self._compiled[key] = self._compile(x.hw, x.data.device, f16, split)
        c = self._compiled[key]
        self.__dict__.setdefault("_touched", set()).add(key)       # pipeline.GraphedAligner ties graphs to the entries they use
        assert x.data.dtype == c["in_dtype"], (x.data.dtype, c["in_dtype"])
        slots = (C.c_void_p * c["nslots"])()
        slots[0] = x.data.data_ptr()
        for i in range(1, c["nslots"]):
            slots[i] = c["bufs"][i].data_ptr()
        check(lib.rf_run_layers(c["layers"], len(self.ops), slots, len(x.hw), c["chw"], int(engine), stream()))
        out = c["bufs"][c["out_slot"]][:c["out_elems"]].view(c["out_dtype"])
        out = out.view(2, -1, self.chan[-1]) if c["out_split"] else out.view(-1, self.chan[-1])
        return out, c["out_hw"]

    def release(self, keep=()):
        """Drop the compiled entries (activation buffers) of every image-set signature except those in ``keep``.  Only safe
        when no captured CUDA graph and no live result view refers to them (pipeline.GraphedAligner.release does both)."""
        for k in [k for k in self._compiled if k not in keep]:
            del self._compiled[k]
