"""ORACLE (test infrastructure) -- the reference's OWN kernels of FlowWarp, FlowWarpGrad, FlowOutOfFrame and Resample
(lmbspecialops/src/{flowwarp,flow_out_of_frame,resample}.cc and {flowwarp,resample}_cuda.cu, compiled unmodified for
sm_90a by oracle/flow_ops.mk into oracle/_ref/libref_flow_ops.so, a git-ignored build product).

Two families:
  * the CPU kernels (FlowWarp, FlowWarpGrad, FlowOutOfFrame; `*_cpu` below) run on host buffers and need no device;
  * the GPU kernels (FlowWarp, FlowWarpGrad, Resample; `*_gpu`) run on the current CUDA device.
Where the library is absent (no reference tree when it was built), every call returns the stored RESULT DIGESTS of the same
call (shape, dtype, SHA-256 with NaNs canonicalised, oracle/recorded.py:digest) from tests/golden/flow_ops_digests.json, keyed by
a hash of the kernel, its attributes and its inputs; record them from the compiled kernels with DEMON_REF_RECORD=<json path>.

Never call the reference's NEAREST resample where its source pixel leaves the image (`nearest_in_range` False): it then
reads another row or past its buffer, so `resample_gpu` refuses it.  FlowWarp with the 'not_a_number' fill writes NaN bits
that the digest canonicalises; tests check those bits on our side.

Only tests/ and tools/ may import this module.
"""
import ctypes
import hashlib
import os

import numpy as np

from .recorded import REF_SRC, Recorded, Store, build_artefact, entry, record

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_ref", "libref_flow_ops.so")
_STORE = Store("flow_ops_digests.json")
_SOURCES = ["flowwarp.cc", "flow_out_of_frame.cc", "resample.cc", "flowwarp_cuda.cu", "resample_cuda.cu"]
_DEPS = ["flow_ops_harness.cu", "flow_ops.mk", "flow_ops_stub.h", "ref_stub_gpu/cuda_helper_shim.h", "ref_stub/tf_stub.h",
         "ref_stub/tensorflow/core/framework/common_shape_fns.h"]
RESAMPLE_TYPES = ("NEAREST", "CUBIC", "LINEAR")


def build(force=False):
    """Compile _ref/libref_flow_ops.so if the reference tree is present; returns the path or None."""
    return build_artefact(_LIB_PATH, [os.path.join(REF_SRC, s) for s in _SOURCES], _DEPS,
                          ["-f", "flow_ops.mk", "flow_ops"], force)


_lib = None


def have_library():
    return build() is not None


def available():
    """The reference kernels can be run here, or their recorded results are stored."""
    return have_library() or bool(_STORE.entries())


def lib():
    global _lib
    if _lib is None:
        path = build()
        if path is None:
            raise RuntimeError("oracle/_ref/libref_flow_ops.so is not built and DEMON_REF_SRC names no reference sources")
        L = ctypes.CDLL(path)
        P, I, I64, S = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_char_p
        L.ref_flow_run.argtypes = [S, S, I, I, I, S, I, P, P, I64, I, P, P, P, S, I]
        L.ref_flow_run.restype = I
        _lib = L
    return _lib


def _key(kernel, attrs, arrays):
    h = hashlib.sha256(("%s|%s" % (kernel, attrs)).encode())
    for a in arrays:
        h.update(("%s|%s" % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def run(kernel, arrays, attrs, out_shapes):
    """Run reference kernel `kernel` ("<op>/<CPU|GPU>/<float|double|>") on 4D numpy `arrays`; attrs = (fill_parameter, width,
    height, antialias, type).  Returns a list of numpy outputs, or of Recorded digests where the library is absent."""
    dt = np.float64 if kernel.endswith("/double") else np.float32
    arrays = [np.ascontiguousarray(a, dtype=dt) for a in arrays]
    key = _key(kernel, attrs, arrays)
    if not have_library():
        return [Recorded(d) for d in _STORE.lookup(key, "reference result for this %s call" % kernel)]
    gpu = "/GPU/" in kernel
    min_elems = max(a.size for a in arrays)   # FlowWarpGrad_CPU clears n*c*h*w elements of its [n,2,h,w] output
    outs = [np.zeros(tuple(max(0, s) for s in shp), dtype=dt) for shp in out_shapes]
    if gpu:
        import torch
        dev_in = [torch.from_numpy(a).cuda() for a in arrays]
        dev_out = [torch.from_numpy(o).cuda() for o in outs]
        in_ptrs = [t.data_ptr() for t in dev_in]
        out_ptrs = [t.data_ptr() for t in dev_out]
        torch.cuda.synchronize()
    else:
        in_ptrs = [a.ctypes.data for a in arrays]
        out_ptrs = [o.ctypes.data for o in outs]
    shapes = (ctypes.c_int64 * (4 * len(arrays)))(*[int(d) for a in arrays for d in a.shape])
    caps = (ctypes.c_int64 * len(outs))(*[o.size for o in outs])
    oshape = (ctypes.c_int64 * 4)()
    err = ctypes.create_string_buffer(1024)
    fill, width, height, antialias, rtype = attrs
    rc = lib().ref_flow_run(kernel.encode(), fill.encode(), int(width), int(height), int(antialias), rtype.encode(), len(arrays),
                            (ctypes.c_void_p * len(arrays))(*in_ptrs), shapes, min_elems, len(outs),
                            (ctypes.c_void_p * len(outs))(*out_ptrs), caps, oshape, err, 1024)
    if rc != 0:
        raise RuntimeError("reference kernel %s: %s" % (kernel, err.value.decode()))
    if tuple(oshape) != tuple(out_shapes[0]):
        raise RuntimeError("reference kernel %s made shape %s, expected %s" % (kernel, tuple(oshape), tuple(out_shapes[0])))
    res = [t.cpu().numpy() for t in dev_out] if gpu else outs
    record(key, [entry(r) for r in res])
    return res


_NO_RESAMPLE = (0, 0, 0, "LINEAR")


def flow_warp_gpu(image, flow, fill_parameter="zero"):
    """FlowWarpOp_GPU::Compute (flowwarp_cuda.cu:226-342) -> warped."""
    return run("FlowWarp/GPU/float", [image, flow], (fill_parameter,) + _NO_RESAMPLE, [np.shape(image)])[0]


def flow_warp_cpu(image, flow, fill_parameter="zero"):
    """FlowWarpOp::Compute (flowwarp.cc:95-178) -> warped."""
    return run("FlowWarp/CPU/float", [image, flow], (fill_parameter,) + _NO_RESAMPLE, [np.shape(image)])[0]


def flow_warp_grad_gpu(image, flow, gradient):
    """FlowWarpGradOp_GPU::Compute (flowwarp_cuda.cu:365-449) -> (image_grad with atomics, flow_grad)."""
    return tuple(run("FlowWarpGrad/GPU/float", [image, flow, gradient], ("zero",) + _NO_RESAMPLE, [np.shape(image), np.shape(flow)]))


def flow_warp_grad_cpu(image, flow, gradient):
    """FlowWarpGradOp::Compute (flowwarp.cc:217-324) -> image_grad (its flow_grad is not used: for c < 2 it leaves the
    second component of out-of-frame pixels unwritten)."""
    return run("FlowWarpGrad/CPU/float", [image, flow, gradient], ("zero",) + _NO_RESAMPLE, [np.shape(image), np.shape(flow)])[0]


def flow_out_of_frame_cpu(flow, occ):
    """FlowOutOfFrameOp::Compute (flow_out_of_frame.cc:38-91) -> [n,1,h,w]."""
    n, _, h, w = np.shape(flow)
    occ4 = np.asarray(occ, dtype=np.float32).reshape(n, 1, h, w)
    return run("FlowOutOfFrame/CPU/", [flow, occ4], ("zero",) + _NO_RESAMPLE, [(n, 1, h, w)])[0]


def nearest_in_range(in_h, in_w, out_h, out_w):
    """Whether every source pixel of the reference's NEAREST kernel lies in the image (float32 arithmetic as it has it)."""
    from .flow_ops import resample_positions
    xr, yr = resample_positions(in_h, in_w, out_h, out_w)
    return xr.min() >= 0 and xr.max() < in_w and yr.min() >= 0 and yr.max() < in_h


def resample_gpu(input, width, height, antialias=True, type="LINEAR"):
    """ResampleOp_GPU::Compute (resample_cuda.cu:155-239) -> output, float32 or float64 as the input."""
    a = np.asarray(input)
    n, c, ih, iw = a.shape
    if type == "NEAREST" and not nearest_in_range(ih, iw, height, width):
        raise ValueError("the reference's NEAREST kernel reads outside its input here; use oracle/flow_ops.py")
    kern = "Resample/GPU/" + ("double" if a.dtype == np.float64 else "float")
    return run(kern, [a], ("zero", int(width), int(height), int(bool(antialias)), type), [(n, c, int(height), int(width))])[0]
