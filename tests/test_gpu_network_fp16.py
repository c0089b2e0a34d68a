"""GPU: the v1 and v2 networks at precision 'fp16'.

* Layer trace (tests/test_gpu_layer_trace.py, tests/test_gpu_layer_trace_v2.py): every layer's input tap bit for bit the
  oracle's, every tensor-core layer's output under the FP16 per-element bound of tests/test_gpu_conv_fp16.py, the SIMT and
  dense layers under gamma_n S as at every precision; bootstrap, iterative and refine.
* End to end on the sculpture pair with synthetic weights: the v1 and v2 pipelines against the fp32 CPU oracle inside the
  bar the single-pass TF32 mode is held to (3e-2): inverse-depth L1-rel of predict_depth0, EPE of predict_flow2."""
import os

import numpy as np
import pytest
import torch

import test_gpu_layer_trace as trace1
import test_gpu_layer_trace_v2 as trace2
from demon_b200.networks_original import DemonPipeline, Session
from demon_b200.v2 import weights as W2
from demon_b200.v2.networks import DemonPipelineV2, Session as SessionV2
from oracle.network_v2 import OracleNetsV2
from test_conv_variants import tc_error_bound
from test_gpu_conv_fp16 import fp16_error_bound
from test_plans_fp16 import FP16

pytestmark = pytest.mark.gpu

TF32_BAR = 3e-2   # tests/test_gpu_blocks_v2.py's and tests/test_gpu_network_v2.py's bar for single-pass TF32


def l1_rel(a, r):
    return float(np.abs(a - r).sum() / np.abs(r).sum())


def epe(a, r):
    return float(np.sqrt(((a - r) ** 2).sum(axis=1)).mean())


@pytest.fixture
def fp16_trace(monkeypatch):
    """The trace modules' checks with 'fp16' as one of their precisions and the FP16 bound for it."""
    def bound(precision, Cin, kh, kw, deconv, ksplit):
        return fp16_error_bound(Cin, kh, kw, deconv, ksplit) if precision == FP16 else tc_error_bound(precision, Cin, kh, kw, deconv, ksplit)
    monkeypatch.setitem(trace1.PRECISIONS, "fp16", FP16)
    for m in (trace1, trace2):
        monkeypatch.setattr(m, "tc_error_bound", bound)


def test_trace_v1_fp16(fp16_trace, synthetic_weights):
    s = Session(precision="fp16")
    s.load_weights(synthetic_weights)
    g = torch.Generator().manual_seed(1234)
    ip = (torch.rand(2, 6, 192, 256, generator=g) - 0.5).numpy()
    from oracle import ops as oops
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    trace1.run_all_stages(s, "fp16", synthetic_weights, ip, i22)
    ratio, share, name = trace1.WORST["fp16"]
    print("\nv1 layer trace, fp16: largest |err| / S = %.3g (%.3g of the bound) at %s" % (ratio, share, name))


def test_trace_v2_fp16(fp16_trace):
    weights = W2.synthetic_weights(0)
    s = SessionV2(precision="fp16")
    s.load_weights(weights)
    g = torch.Generator().manual_seed(4321)
    ip = (torch.rand(2, 6, 192, 256, generator=g) - 0.5).numpy()
    from oracle import ops as oops
    i22 = oops.median3x3_downsample(oops.median3x3_downsample(np.ascontiguousarray(ip[:, 3:6])))
    r0, _ = trace2.run_stage(s, "fp16", weights, "bootstrap", 2, (ip, i22))
    r1, _ = trace2.run_stage(s, "fp16", weights, "iterative", 2, trace2.iterative_inputs(ip, i22, r0))
    trace2.run_stage(s, "fp16", weights, "refine", 2, (np.ascontiguousarray(ip[:, 0:3]), r1["predict_depth2"].cpu().numpy()))
    ratio, share, name = trace2.WORST["fp16"]
    print("\nv2 layer trace, fp16: largest |err| / S = %.3g (%.3g of the bound) at %s" % (ratio, share, name))


def run_pipeline(pipe, sculpture):
    out = pipe.forward(torch.from_numpy(sculpture["image_pair"]).cuda(), torch.from_numpy(sculpture["image2_2"]).cuda())
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}


def test_v1_pipeline_fp16_on_sculpture(synthetic_weights, sculpture, golden_dir):
    s = Session(precision="fp16")
    s.load_weights(synthetic_weights)
    out = run_pipeline(DemonPipeline(s, batch_size=1, iterations=3), sculpture)
    g = np.load(os.path.join(golden_dir, "oracle_pipeline.npz"))   # the fp32 CPU oracle's outputs
    d0, f2 = l1_rel(out["predict_depth0"], g["predict_depth0_f32"]), epe(out["predict_flow2"], g["predict_flow2_f32"])
    print("\nv1 fp16 on the sculpture pair: predict_depth0 L1-rel %.3e, predict_flow2 EPE %.3e" % (d0, f2))
    assert d0 < TF32_BAR and f2 < TF32_BAR


def test_v2_pipeline_fp16_on_sculpture(sculpture):
    weights = W2.synthetic_weights(0)
    s = SessionV2(precision="fp16")
    s.load_weights(weights)
    out = run_pipeline(DemonPipelineV2(s, batch_size=1, iterations=3), sculpture)
    ref = OracleNetsV2(weights).pipeline(sculpture["image_pair"], sculpture["image2_2"], iterations=3)
    n = lambda t: t.numpy() if hasattr(t, "numpy") else t
    d0, f2 = l1_rel(out["predict_depth0"], n(ref["predict_depth0"])), epe(out["predict_flow2"], n(ref["predict_flow2"]))
    print("\nv2 fp16 on the sculpture pair: predict_depth0 L1-rel %.3e, predict_flow2 EPE %.3e" % (d0, f2))
    assert d0 < TF32_BAR and f2 < TF32_BAR
