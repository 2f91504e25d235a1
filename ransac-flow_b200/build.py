"""Build libransacflow_b200.so in-tree with nvcc for sm_90a (H100).

    python ransac-flow_b200/build.py [--force]

The .so and the object files under build/ are build products (git-ignored).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libransacflow_b200.so")
SOURCES = ["api.cu", "ransac.cu", "gemm_simt.cu", "gemm_tc.cu", "elementwise.cu", "runner.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _digest():
    h = hashlib.sha256()
    for root, _, files in sorted(os.walk(CSRC)):
        for f in sorted(files):
            h.update(f.encode())
            h.update(open(os.path.join(root, f), "rb").read())
    h.update(open(os.path.join(os.path.dirname(HERE), "include", "ransacflow_b200.h"), "rb").read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def lib_digest(path=LIB):
    """The digest embedded in a built library (rf_source_digest), or None."""
    if not os.path.exists(path):
        return None
    import ctypes
    try:
        lib = ctypes.CDLL(path)
        fn = lib.rf_source_digest
        fn.restype = ctypes.c_char_p
        return fn().decode()
    except (OSError, AttributeError):
        return None


def is_current():
    return lib_digest() == _digest()


def build(force=False, verbose=True):
    if not force and is_current():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    digest = _digest()
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    procs = []
    for s in SOURCES:
        o = os.path.join(objdir, s.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + (['-DRF_SOURCE_DIGEST="%s"' % digest] if s == "api.cu" else []) + ["-c", os.path.join(CSRC, s), "-o", o]
        procs.append((s, o, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    objs = []
    for s, o, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (s, out))
        if verbose and out.strip():
            print(out)
        objs.append(o)
    cmd = [nvcc, "-shared", "-Wno-deprecated-gpu-targets", "-o", LIB] + objs + ["-lcudart"]
    subprocess.check_call(cmd)
    if verbose:
        print("built", LIB)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
