"""Latency / throughput of the BASELINE.json configurations other than the bench workload:
configs[1] full pipeline at batch 1 (latency), configs[4] RefinementNet at 1024x768 batch 8, plus batch 8 and 16."""
import torch

from benchkit import span_ms
from demon_b200 import weights as W
from demon_b200.networks_original import Session, DemonPipeline, RefinementNet


def main():
    sess = Session("3xtf32")
    sess.load_weights(W.synthetic_weights(0))
    for B in (1, 8, 16):
        pipe = DemonPipeline(sess, B, 3)
        x = torch.rand(B, 6, 192, 256, device="cuda") - 0.5
        outs = pipe.forward(x, None)
        ms = span_ms(lambda: pipe.forward(x, None, outs), 30, warmup=5)
        print("full pipeline batch %2d: %.3f ms per call (CUDA graph replay, device resident) = %.0f pairs/s" % (B, ms, B / ms * 1e3))
    net = RefinementNet(sess, "channels_first", 8, image_size=(768, 1024))
    img = torch.rand(8, 3, 768, 1024, device="cuda") - 0.5
    d2 = torch.rand(8, 1, 192, 256, device="cuda") + 0.3
    ms = span_ms(lambda: net.eval(img, d2), 10)
    macs = W.macs_per_pair()["refine_fn"](768, 1024) * 8
    print("RefinementNet 1024x768 batch 8: %.3f ms per call = %.1f algorithmic TFLOP/s (98.675 GFLOP per image)" % (ms, 2 * macs / (ms / 1e3) / 1e12))


if __name__ == "__main__":
    main()
