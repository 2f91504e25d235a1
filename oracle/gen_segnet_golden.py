"""Generate tests/golden/segnet.npz by running the UNMODIFIED reference segNet (segNet/segEval.py ``SegNet.getSky``) on the CPU:

    python -m oracle.gen_segnet_golden           # needs the reference checkout ($RF_REFERENCE), writes tests/golden/segnet.npz

Weights come from synthdata (saved to temporary .pth files, loaded by the reference's own ModelBuilder).  Harness-side shims
only: ``cpu_as_cuda`` (gen_golden.py) and a recorder on ``torch.max`` that keeps the vote's score tensor, from which the tie
proofs (per-pixel top-1 - top-2 and top-1 - segId margins) are computed.  Two seeded images: 96 x 128 (two distinct pass sizes,
304 x 400 and 376 x 504) and 20 x 400 (one size, 32 x 504, whose conv5 has 4 rows: fewer than the 6 PPM bins).
"""
import os
import sys
import tempfile

import numpy as np
import PIL.Image as Image
import torch

from . import synth
from .gen_golden import REF, cpu_as_cuda, save
from .seg_oracle import margins, pass_sizes

IMAGES = ((0, 96, 128), (1, 20, 400))
VARIANTS = ((2, False), (1, True))          # (segId, segFg): evalHpatch / evalCorr / evalKITTI, evalYFCC


def gen_segnet():
    torch.set_num_threads(os.cpu_count() or 1)
    seg_dir = os.path.join(REF, "segNet")
    sys.path.insert(0, seg_dir)
    import segEval                           # noqa: E402  (the reference module, as is)
    real_max = torch.max
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        enc_p, dec_p = os.path.join(tmp, "enc.pth"), os.path.join(tmp, "dec.pth")
        torch.save(synth.segnet_encoder_state(0), enc_p)
        torch.save(synth.segnet_decoder_state(0), dec_p)
        for (seed, h, w) in IMAGES:
            img_p = os.path.join(tmp, "img%d.png" % seed)
            Image.fromarray(synth.segnet_image(seed, h, w)).save(img_p)
            out["sizes_%d" % seed] = np.array(pass_sizes(h, w), dtype=np.int32)
            for segId, segFg in VARIANTS:
                seen = []

                def rec_max(x, *a, **k):
                    if k.get("dim") == 1 and x.dim() == 4:
                        seen.append(x.detach().clone())
                    return real_max(x, *a, **k)
                with cpu_as_cuda():
                    net = segEval.SegNet(enc_p, dec_p, segId, segFg)
                    torch.max = rec_max
                    try:
                        mask = net.getSky(img_p)
                    finally:
                        torch.max = real_max
                scores = seen[-1][0].double().numpy()
                top12, top1_seg = margins(scores, segId)
                tag = "%d_%d_%d" % (seed, segId, int(segFg))
                out["mask_" + tag] = mask.astype(np.float32)
                out["class_" + tag] = scores.argmax(0).astype(np.int16)
                out["margin12_" + tag] = top12.astype(np.float32)
                out["margin_seg_" + tag] = top1_seg.astype(np.float32)
    sys.path.remove(seg_dir)
    save("segnet", **out)


if __name__ == "__main__":
    gen_segnet()
