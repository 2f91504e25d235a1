"""Write tests/golden/yfcc_pose.npz from the reference's own evalYFCC functions (evaluation/evalYFCC/getResults.py:
matches_from_flow, norm_kp, opencv_decompose, evaluate_R_t, extracted with oracle.gen_golden.extract_function, run with OpenCV).

    RF_REFERENCE=<reference checkout> python tests/gen_pose_golden.py

Scenes are seeded (tests/pose_oracle.py: scene); each stores its inputs, cv2's E / RANSAC mask, recoverPose's count, R, t and
mask, and the pose error against the scene's ground truth.  Four flow / mask inputs at angles 0 / 90 / 180 / 270 with odd sizes
store the driver's matches.  Masks are stored bit-packed (np.packbits)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import cv2  # noqa: E402

import pose_oracle as PO  # noqa: E402
from oracle.gen_golden import REF, extract_function  # noqa: E402

SCRIPT = os.path.join(REF, "evaluation", "evalYFCC", "getResults.py")
THRESHOLD = 0.0005
# (N, outlier ratio, seed, planar)
SCENES = [(4, 0.0, 1, False), (5, 0.0, 2, False), (5, 0.0, 3, False), (6, 0.0, 4, False), (6, 0.2, 5, False), (7, 0.0, 6, False),
          (7, 0.3, 7, False), (50, 0.0, 8, False), (50, 0.3, 9, False), (50, 0.6, 10, False), (200, 0.8, 11, False),
          (2000, 0.0, 12, False), (2000, 0.1, 13, False), (2000, 0.3, 14, False), (2000, 0.5, 15, False), (2000, 0.7, 16, False),
          (2000, 0.8, 17, False), (2000, 0.3, 18, True), (500, 0.5, 19, True), (100000, 0.1, 20, False), (100000, 0.3, 21, False)]
# (angle, hB, wB, hA, wA)
FLOWS = [(0, 37, 53, 41, 47), (90, 37, 53, 41, 47), (180, 29, 45, 33, 39), (270, 29, 45, 33, 39)]


def main():
    ns = {"np": np, "cv2": cv2}
    matches_from_flow = extract_function(SCRIPT, "matches_from_flow", ns)
    norm_kp = extract_function(SCRIPT, "norm_kp", ns)
    opencv_decompose = extract_function(SCRIPT, "opencv_decompose", ns)
    evaluate_R_t = extract_function(SCRIPT, "evaluate_R_t", ns)
    out = {"threshold": np.float64(THRESHOLD), "scenes": np.array(SCENES, dtype=np.float64), "flows": np.array(FLOWS)}
    for s, (N, outlier, seed, planar) in enumerate(SCENES):
        p1, p2, R, t = PO.scene(int(N), outlier, seed, planar=planar)
        out["s%d_checksum" % s] = np.array([p1.sum(), p2.sum()])       # the scene is regenerated from its seed by the tests
        out["s%d_R_gt" % s], out["s%d_t_gt" % s] = R, t
        if N >= 5:
            E, m = cv2.findEssentialMat(p1, p2, method=cv2.RANSAC, threshold=THRESHOLD)
            out["s%d_E" % s] = np.zeros((0, 3)) if E is None else E
            out["s%d_mask" % s] = np.packbits(np.zeros(0, np.uint8) if m is None else m.ravel())
        res, mask_final = opencv_decompose(p1, p2, True, THRESHOLD)
        out["s%d_has_pose" % s] = np.bool_(res is not None)
        if res is not None:
            out["s%d_R" % s], out["s%d_t" % s] = res
            out["s%d_pose_mask" % s] = np.packbits(mask_final.ravel().astype(bool))
            out["s%d_pose_count" % s] = np.int64(mask_final.astype(bool).sum())
            out["s%d_err" % s] = np.float64(max(evaluate_R_t(R, t, res[0], res[1])))
        print("scene", s, N, outlier, "pose" if res is not None else "none")
    rs = np.random.RandomState(5)
    for f, (angle, hB, wB, hA, wA) in enumerate(FLOWS):
        H, W = (hB, wB) if (angle // 90) % 2 == 0 else (wB, hB)
        flow = rs.uniform(-1, 1, (H, W, 2)).astype(np.float32)
        mb = rs.rand(H, W) < 0.6
        K_A = np.array([[300.0 + f, 0, 3.5], [0, 310.0, -2.25], [0, 0, 1]])
        K_B = np.array([[280.0, 0, -1.75], [0, 290.0 + f, 4.0], [0, 0, 1]])
        orgA, orgB = (wA * 3 + 1, hA * 3 - 1), (wB * 2 + 1, hB * 2 + 3)
        pts1, pts2 = matches_from_flow(flow.copy(), mb, (wA, hA), (wB, hB), angle)
        out["f%d_flow" % f], out["f%d_mask" % f] = flow, mb
        out["f%d_KA" % f], out["f%d_KB" % f] = K_A, K_B
        out["f%d_orgA" % f], out["f%d_orgB" % f] = np.array(orgA), np.array(orgB)
        out["f%d_pts1" % f] = norm_kp(orgA, (wA, hA), K_A, pts1)
        out["f%d_pts2" % f] = norm_kp(orgB, (wB, hB), K_B, pts2)
    path = os.path.join(ROOT, "tests", "golden", "yfcc_pose.npz")
    np.savez_compressed(path, **out)
    print("wrote", path)


if __name__ == "__main__":
    main()
