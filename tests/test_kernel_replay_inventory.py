"""Every ``ops`` function that reaches the library's kernels is assigned a check.

``INVENTORY`` maps each such function to "replayed here" (tests/test_gpu_kernel_replay.py records its calls while the
pipeline runs and checks each call's output against a reference computed from the operands that call read) or to the test
file that covers it instead, with the reason.  The set of functions is found from the source: those whose body calls
``lib.rf_``, plus ``resample_coeffs``, which reaches the library through ``getattr(lib, fn)``.  A new kernel entry therefore
fails this test until someone decides how it is checked.  Runs without a GPU.
"""
import inspect

REPLAYED = "replayed here"
INVENTORY = {
    "_resize_u8": REPLAYED,
    "bytescale_mask_u8": REPLAYED,
    "preproc_u8": REPLAYED,
    "l2norm": REPLAYED,
    "l2norm_planes": REPLAYED,
    "corr_mutual_nn": REPLAYED,
    "corr_mutual_nn_presplit": REPLAYED,
    "build_matches": REPLAYED,
    "ransac_homography": REPLAYED,
    "warp_grid": REPLAYED,
    "grid_sample": REPLAYED,
    "upsample_bilinear": REPLAYED,
    "compose_fine": REPLAYED,
    "corr_neigh": REPLAYED,
    "corr_neigh_pair": REPLAYED,
    "corr_neigh_pair_split": REPLAYED,
    "softmax_flow": REPLAYED,
    "sigmoid": REPLAYED,
    "remove_small_cc": REPLAYED,
    "kitti_region_step": REPLAYED,
    "fill_nearest_matched": REPLAYED,
    # host tables: checked against Pillow on the host, and through every recorded _resize_u8 call that reads them
    "resample_coeffs": "test_resample_host.py",
    # the layer ops outside the layer programs' own runner: every layer of every program is replayed against fp64
    "conv2d": "test_gpu_program_replay.py, test_gpu_layer_ops.py",
    "conv1x1_dual_split": "test_gpu_program_replay.py, test_gpu_wgmma_edges.py",
    "maxpool2d": "test_gpu_program_replay.py, test_gpu_layer_ops.py",
    "blur_downsample": "test_gpu_program_replay.py, test_gpu_layer_ops.py",
    # reached only by the host-steered outil.RANSAC (align_pair / getCoarse without the device path), not by the pair paths
    "homography_dlt": "test_gpu_geometry.py, test_gpu_ransac_exact.py (not reached by the device pair paths)",
    "prediction": "test_gpu_ransac.py (not reached by the device pair paths)",
    # evalYFCC's relative pose
    "yfcc_matches": "test_gpu_pose_stages.py",
    "essential_ransac": "test_gpu_pose_stages.py",
    "recover_pose": "test_gpu_pose_stages.py",
    "essential_samples": "test_gpu_pose_stages.py",
    "essential_five_point": "test_gpu_pose_stages.py",
    "essential_score": "test_gpu_pose_stages.py",
    "fundamental_8point": "test_gpu_pose_stages.py",
    "fundamental_moments": "test_gpu_pose_stages.py",
}


def kernel_entries(ops):
    """Names of the functions defined in ``ops`` whose source calls the library."""
    found = set()
    for name, fn in vars(ops).items():
        if inspect.isfunction(fn) and fn.__module__ == ops.__name__:
            src = inspect.getsource(fn)
            if "lib.rf_" in src or "getattr(lib," in src:
                found.add(name)
    return found


def test_inventory_names_every_kernel_entry(rf):
    found = kernel_entries(rf.ops)
    assert "resample_coeffs" in found and "_resize_u8" in found
    missing, stale = found - set(INVENTORY), set(INVENTORY) - found
    assert not missing, "ops functions that launch kernels without a check assigned: %s" % sorted(missing)
    assert not stale, "inventory entries that are no longer kernel entries of ops: %s" % sorted(stale)


def test_inventory_files_exist():
    import os
    from conftest import ROOT
    for name, where in INVENTORY.items():
        if where != REPLAYED:
            for f in where.split(" (")[0].split(", "):
                assert os.path.exists(os.path.join(ROOT, "tests", f)), (name, f)
