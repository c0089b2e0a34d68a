"""Builds libdemon_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

The library and its objects (demon_b200/lib/) are build products and stay out of git.
"""
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_DIR = os.path.join(_HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libdemon_b200.so")
SOURCES = ["geometry_ops.cu", "metrics.cu", "evaluation.cu", "training_ops.cu", "conv_simt.cu", "conv_tc_halo.cu", "images.cu", "vis.cu", "fusion.cu", "dataset_tools.cu",
           "correlation.cu", "flow_ops.cu", "losses.cu", "datareader.cu", "net.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _deps():
    out = []
    for root in (CSRC, os.path.join(_HERE, "..", "include")):
        for f in os.listdir(root):
            if f.endswith((".cu", ".cuh", ".h")):
                out.append(os.path.join(root, f))
    return out


def needs_build():
    if not os.path.isfile(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(d) > t for d in _deps())


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    os.makedirs(LIB_DIR, exist_ok=True)
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIB_DIR, src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write("[nvcc %s]\n%s\n" % (src, out))
        failed = failed or p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    # the driver API (cuTensorMapEncodeTiled) is resolved at run time through cudaGetDriverEntryPoint
    tmp = LIB_PATH + ".tmp"   # link beside the target and rename: a snapshot never sees a half-written library
    subprocess.check_call([nvcc, "-shared", "-o", tmp] + objs + GENCODE)
    os.replace(tmp, LIB_PATH)
    return LIB_PATH


def build_variant(name, extra_flags):
    """Diagnostic builds (extra nvcc flags, e.g. -lineinfo -G) next to the product library:
    lib/variants/<name>/libdemon_b200.so, selected at run time with DEMON_B200_LIB."""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    out_dir = os.path.join(LIB_DIR, "variants", name)
    os.makedirs(out_dir, exist_ok=True)
    procs, objs = [], []
    for src in SOURCES:
        obj = os.path.join(out_dir, src.replace(".cu", ".o"))
        objs.append(obj)
        procs.append(subprocess.Popen([nvcc] + NVCC_FLAGS + list(extra_flags) + ["-c", os.path.join(CSRC, src), "-o", obj]))
    if any(p.wait() != 0 for p in procs):
        raise RuntimeError("nvcc failed")
    path = os.path.join(out_dir, "libdemon_b200.so")
    subprocess.check_call([nvcc, "-shared", "-o", path] + objs + GENCODE)
    return path


if __name__ == "__main__":
    if "--variant" in sys.argv:
        i = sys.argv.index("--variant")
        print(build_variant(sys.argv[i + 1], sys.argv[i + 2:]))
    else:
        print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
