"""Every function or method of the package that reaches the library's kernels is assigned a check.

``INVENTORY`` maps each such callable, keyed ``module.qualname`` (``ops.l2norm``, ``program.LayerProgram.run``), to
"replayed here" (tests/test_gpu_kernel_replay.py records its calls while the pipeline runs and checks each call's output
against a reference computed from the operands that call read) or to the test files (``file.py``) or tests
(``file.py::test_name``) that cover it instead, with the reason.  The set of callables is found from the source of every
module of the package: the module-level functions and the methods of module-level classes whose body calls ``lib.rf_`` or
reaches the library through ``getattr(lib, ...)``.  ``HOST_ONLY`` lists the helpers that do so without launching anything.
A new kernel entry in any module therefore fails this test until someone decides how it is checked.  Runs without a GPU.
"""
import glob
import importlib
import inspect
import os
import re
import types

REPLAYED = "replayed here"
INVENTORY = {
    "ops._resize_u8": REPLAYED,
    "ops.bytescale_mask_u8": REPLAYED,
    "ops.preproc_u8": REPLAYED,
    "ops.l2norm": REPLAYED,
    "ops.l2norm_planes": REPLAYED,
    "ops.corr_mutual_nn": REPLAYED,
    "ops.corr_mutual_nn_presplit": REPLAYED,
    "ops.build_matches": REPLAYED,
    "ops.ransac_homography": REPLAYED,
    "ops.warp_grid": REPLAYED,
    "ops.grid_sample": REPLAYED,
    "ops.upsample_bilinear": REPLAYED,
    "ops.compose_fine": REPLAYED,
    "ops.corr_neigh": REPLAYED,
    "ops.corr_neigh_pair": REPLAYED,
    "ops.corr_neigh_pair_split": REPLAYED,
    "ops.softmax_flow": REPLAYED,
    "ops.sigmoid": REPLAYED,
    "ops.remove_small_cc": REPLAYED,
    "ops.kitti_region_step": REPLAYED,
    "ops.fill_nearest_matched": REPLAYED,
    "validation.affine_sample_u8": REPLAYED,
    "validation.val_keypoints": REPLAYED,
    "corr_results.corr_keypoints": REPLAYED,
    "train_pairs.warp_sample_u8": REPLAYED,
    # host tables: checked against Pillow on the host, and through every recorded _resize_u8 call that reads them
    "ops.resample_coeffs": "test_resample_host.py",
    # the layer ops outside the layer programs' own runner: every layer of every program is replayed against fp64
    "ops.conv2d": "test_gpu_program_replay.py, test_gpu_layer_ops.py",
    "ops.conv1x1_dual_split": "test_gpu_program_replay.py, test_gpu_wgmma_edges.py",
    "ops.maxpool2d": "test_gpu_program_replay.py, test_gpu_layer_ops.py",
    "ops.blur_downsample": "test_gpu_program_replay.py, test_gpu_layer_ops.py",
    "program.LayerProgram.run": "test_gpu_program_replay.py",
    # segNet's decoder pooling, PPM concatenation and vote, replayed on the network's own conv5
    "segnet.SegNet.ppm": "test_gpu_program_replay.py, test_gpu_segnet.py",
    "segnet.SegNet.vote": "test_gpu_program_replay.py, test_gpu_segnet.py",
    # reached only by the host-steered outil.RANSAC (align_pair / getCoarse without the device path), not by the pair paths
    "ops.homography_dlt": "test_gpu_geometry.py, test_gpu_ransac_exact.py (not reached by the device pair paths)",
    "ops.prediction": "test_gpu_ransac.py (not reached by the device pair paths)",
    # evalYFCC's relative pose
    "ops.yfcc_matches": "test_gpu_pose_stages.py",
    "ops.essential_ransac": "test_gpu_pose_stages.py",
    "ops.recover_pose": "test_gpu_pose_stages.py",
    "ops.essential_samples": "test_gpu_pose_stages.py",
    "ops.essential_five_point": "test_gpu_pose_stages.py",
    "ops.essential_score": "test_gpu_pose_stages.py",
    "ops.fundamental_8point": "test_gpu_pose_stages.py",
    "ops.fundamental_moments": "test_gpu_pose_stages.py",
    # evalYFCC's graphed pair: the drawn RANSAC, the rotation choice and the slot copy
    "yfcc_graph.ransac_homography_drawn": "test_gpu_yfcc_graph.py::test_slot_chain_reads_the_eager_tables",
    "yfcc_graph.rotation_select": "test_gpu_yfcc_graph.py::test_rotation_select_is_the_numpy_restatement",
    "yfcc_graph.select_copy": "test_gpu_yfcc_graph.py::test_select_copy",
}

# callables that call the library but launch nothing
HOST_ONLY = {
    "_lib._load": "binds the entry points' ctypes signatures",
    "_lib.check": "reads the library's last error string",
    "_lib.launch_count": "reads the library's launch counter",
    "build.lib_digest": "reads the source digest of a built library",
}

_CALLS_LIB = re.compile(r"\blib\.rf_\w|\bgetattr\(\s*lib\s*,")


def _callables(mod):
    """(qualname, function) of the module-level functions and of the methods of module-level classes written in ``mod``'s
    own file (not those a decorator or a named tuple generates)."""
    out = []
    for name, obj in vars(mod).items():
        if inspect.isclass(obj) and obj.__module__ == mod.__name__:
            for k, v in vars(obj).items():
                fn = v.__func__ if isinstance(v, (staticmethod, classmethod)) else v.fget if isinstance(v, property) else v
                if inspect.isfunction(fn):
                    out.append(("%s.%s" % (name, k), fn))
        elif inspect.isfunction(obj) and obj.__module__ == mod.__name__:
            out.append((name, obj))
    return [(q, fn) for q, fn in out if fn.__code__.co_filename == mod.__file__]


def kernel_entries(mod, prefix=None):
    """``prefix.qualname`` of every callable of ``mod`` whose source calls the library (prefix: the module's last name)."""
    prefix = mod.__name__.rsplit(".", 1)[-1] if prefix is None else prefix
    return {"%s.%s" % (prefix, q) for q, fn in _callables(mod) if _CALLS_LIB.search(inspect.getsource(fn))}


def package_modules(rf):
    """(short name, module) of every Python module of the package, the package itself as ``__init__``."""
    root = os.path.dirname(rf.__file__)
    mods = []
    for path in sorted(glob.glob(os.path.join(root, "*.py"))):
        name = os.path.basename(path)[:-3]
        mods.append((name, rf if name == "__init__" else importlib.import_module("%s.%s" % (rf.__name__, name))))
    return mods


def package_entries(rf):
    found = set()
    for name, mod in package_modules(rf):
        found |= kernel_entries(mod, name)
    return found


def test_inventory_names_every_kernel_entry(rf):
    names = {n for n, _ in package_modules(rf)}
    assert {"ops", "validation", "corr_results", "train_pairs", "segnet", "yfcc_graph", "program", "pipeline"} <= names, names
    found = package_entries(rf)
    assert {"ops.resample_coeffs", "ops._resize_u8", "program.LayerProgram.run", "validation.val_keypoints"} <= found
    assert not set(INVENTORY) & set(HOST_ONLY)
    listed = set(INVENTORY) | set(HOST_ONLY)
    missing, stale = found - listed, listed - found
    assert not missing, "callables that launch kernels without a check assigned: %s" % sorted(missing)
    assert not stale, "inventory entries that are no longer kernel entries of the package: %s" % sorted(stale)


def test_scanner_finds_functions_and_methods(tmp_path):
    """A synthetic module with one function and one method that call the library (and helpers that do not)."""
    src = (
        "lib = None\n"
        "def launch(x):\n"
        "    return lib.rf_something(x)\n"
        "def host(x):\n"
        "    '''mentions lib but calls nothing'''\n"
        "    return x\n"
        "class Runner:\n"
        "    def run(self, x):\n"
        "        return lib.rf_something(x, 1)\n"
        "    @staticmethod\n"
        "    def table(fn):\n"
        "        return getattr(lib, fn)()\n"
        "    def idle(self):\n"
        "        return None\n"
    )
    path = tmp_path / "synthetic_kernels.py"
    path.write_text(src)
    mod = types.ModuleType("synthetic_kernels")
    mod.__file__ = str(path)
    exec(compile(src, str(path), "exec"), mod.__dict__)
    assert kernel_entries(mod) == {"synthetic_kernels.launch", "synthetic_kernels.Runner.run", "synthetic_kernels.Runner.table"}


def test_inventory_files_exist():
    from conftest import ROOT
    for name, where in INVENTORY.items():
        if where == REPLAYED:
            continue
        for f in where.split(" (")[0].split(", "):
            f, _, test = f.partition("::")
            path = os.path.join(ROOT, "tests", f)
            assert os.path.exists(path), (name, f)
            if test:
                assert re.search(r"^def %s\(" % re.escape(test), open(path).read(), re.M), (name, f, test)
