"""ORACLE (test infrastructure) -- the reference's OWN CUDA kernels of Correlation, CorrelationGrad, Correlation1D and
Correlation1DGrad (lmbspecialops/src/correlation{,_1d}.cc and correlation{,_1d}_cuda.cu, compiled unmodified for sm_90a by
oracle/correlation.mk into oracle/_ref/libref_correlation.so, a git-ignored build product) run on the current CUDA device.

Where the library is absent (no reference tree when it was built), every call returns the stored RESULT DIGESTS of the same
call (shape, dtype, SHA-256 with NaNs canonicalised, oracle/recorded.py:digest) from tests/golden/correlation_digests.json, keyed
by a hash of the op, its attributes and its inputs; record them from the compiled kernels with DEMON_REF_RECORD=<json path>.

Never call the reference with single_dir = -1: its kernels then read before the start of their padded buffer (the first
output column's displaced window starts at x = max_displacement - (R+1) stride2 < 0), so `run` refuses it.

Only tests/ and tools/ may import this module.
"""
import ctypes
import hashlib
import os

import numpy as np

from .recorded import REF_SRC, Recorded, Store, build_artefact, entry, record

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_ref", "libref_correlation.so")
_STORE = Store("correlation_digests.json")
_SOURCES = ["correlation.cc", "correlation_1d.cc", "correlation_cuda.cu", "correlation_1d_cuda.cu"]
_DEPS = ["correlation_harness.cu", "correlation.mk", "ref_stub_gpu/tf_gpu_stub.h", "ref_stub_gpu/cuda_helper_shim.h",
         "ref_stub/tf_stub.h"]


def build(force=False):
    """Compile _ref/libref_correlation.so if the reference tree is present; returns the path or None."""
    return build_artefact(_LIB_PATH, [os.path.join(REF_SRC, s) for s in _SOURCES], _DEPS,
                          ["-f", "correlation.mk", "correlation"], force)


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
            raise RuntimeError("oracle/_ref/libref_correlation.so is not built and DEMON_REF_SRC names no reference sources")
        L = ctypes.CDLL(path)
        P, I, I64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
        L.ref_correlation_run.argtypes = [ctypes.c_char_p, ctypes.c_char_p] + [I] * 11 + [P, P, P, P, P, I64, P, I64, P,
                                                                                         ctypes.c_char_p, I]
        L.ref_correlation_run.restype = I
        _lib = L
    return _lib


def _attrs(corr_type, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs, single_dir):
    return (str(corr_type), int(kernel_size), int(max_displacement), int(stride1), int(stride2), int(pad_size), int(bool(do_abs)),
            int(single_dir))


def _key(op, attrs, arrays):
    h = hashlib.sha256(("%s|%s" % (op, attrs)).encode())
    for a in arrays:
        h.update(("%s|%s" % (a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def run(op, arrays, attrs, out_shapes):
    """Run reference op `op` on float32 numpy `arrays` (input1, input2[, gradient]); returns a list of numpy outputs, or of
    Recorded digests where the library is absent."""
    arrays = [np.ascontiguousarray(a, dtype=np.float32) for a in arrays]
    if attrs[-1] == -1:
        raise ValueError("the reference's kernels read out of bounds with single_dir = -1; use oracle/correlation.py")
    key = _key(op, attrs, arrays)
    if not have_library():
        return [Recorded(d) for d in _STORE.lookup(key, "reference result for this %s call" % op)]
    import torch
    dev = [torch.from_numpy(a).cuda() for a in arrays]
    outs = [torch.empty(tuple(max(0, s) for s in shp), dtype=torch.float32, device="cuda") for shp in out_shapes]
    gshape = (ctypes.c_int64 * 4)(*(arrays[2].shape if len(arrays) > 2 else (0, 0, 0, 0)))
    oshape = (ctypes.c_int64 * 4)()
    err = ctypes.create_string_buffer(1024)
    n, c, h, w = arrays[0].shape
    o1 = outs[1] if len(outs) > 1 else None
    torch.cuda.synchronize()
    rc = lib().ref_correlation_run(op.encode(), attrs[0].encode(), *attrs[1:], n, c, h, w, dev[0].data_ptr(), dev[1].data_ptr(),
                                   dev[2].data_ptr() if len(dev) > 2 else None, gshape, outs[0].data_ptr(), outs[0].numel(),
                                   o1.data_ptr() if o1 is not None else None, o1.numel() if o1 is not None else 0, oshape, err, 1024)
    if rc != 0:
        raise RuntimeError("reference kernel %s: %s" % (op, err.value.decode()))
    if tuple(oshape) != tuple(out_shapes[0]):
        raise RuntimeError("reference kernel %s made shape %s, expected %s" % (op, tuple(oshape), tuple(out_shapes[0])))
    res = [o.cpu().numpy() for o in outs]
    record(key, [entry(r) for r in res])
    return res


def correlation(input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False, corr_type="mult"):
    """CorrelationOp_GPU::Compute (correlation_cuda.cu:488-555) -> output (or its Recorded digest)."""
    from demon_b200.lmbspecialops import correlation_top_shape
    shp = correlation_top_shape(np.shape(input1), max_displacement, kernel_size, stride1, stride2, pad_size)
    return run("Correlation", [input1, input2], _attrs(corr_type, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs, 0),
               [shp])[0]


def correlation_grad(gradient, input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False,
                     corr_type="mult"):
    """CorrelationGradOp_GPU::Compute (correlation_cuda.cu:698-764) -> (input1_grad, input2_grad)."""
    return tuple(run("CorrelationGrad", [input1, input2, gradient],
                     _attrs(corr_type, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs, 0),
                     [np.shape(input1), np.shape(input2)]))


def correlation_1d(input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False, corr_type="mult",
                   single_dir=0):
    """Correlation1DOp_GPU::Compute (correlation_1d_cuda.cu:466-544) -> output (or its Recorded digest)."""
    from demon_b200.lmbspecialops import correlation_top_shape
    shp = correlation_top_shape(np.shape(input1), max_displacement, kernel_size, stride1, stride2, pad_size, True, single_dir)
    return run("Correlation1D", [input1, input2],
               _attrs(corr_type, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs, single_dir), [shp])[0]


def correlation_1d_grad(gradient, input1, input2, max_displacement, kernel_size, stride1=1, stride2=1, pad_size=0, do_abs=False,
                        corr_type="mult", single_dir=0):
    """Correlation1DGradOp_GPU::Compute (correlation_1d_cuda.cu:689-767) -> (input1_grad, input2_grad)."""
    return tuple(run("Correlation1DGrad", [input1, input2, gradient],
                     _attrs(corr_type, kernel_size, max_displacement, stride1, stride2, pad_size, do_abs, single_dir),
                     [np.shape(input1), np.shape(input2)]))
