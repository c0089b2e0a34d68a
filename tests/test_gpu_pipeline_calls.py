"""GPU: every kind of fused-pipeline call on one DemonPipeline, interleaved, through eager runs, graph capture and replay.

The device-side calls below all write into the pipeline's own output buffers and read inputs staged in the same buffers
every time, so only the remaining fields of a call (its input kind, sizes, modes, snapshot mode and input pointers) tell
one CUDA graph from another.  Every result must equal the eager result of the same kind on the same inputs, bit for bit,
whatever ran before it, and the launch counts must stay those of the eager call."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from demon_b200 import _lib

B, ITERATIONS, H, W = 2, 3, 480, 640
SNAPSHOT_KINDS = ("snapshots_refined", "snapshots")


def make_inputs(seed):
    rng = np.random.default_rng(seed)
    f = rng.uniform(380, 700, (B, 2))
    K = np.stack([f, f * rng.uniform(0.95, 1.05, (B, 2)), rng.uniform(250, 390, (B, 2)), rng.uniform(180, 300, (B, 2))], -1)
    return {"image_pair": rng.uniform(-0.5, 0.5, (B, 6, 192, 256)).astype(np.float32),
            "image2_2": rng.uniform(-0.5, 0.5, (B, 3, 48, 64)).astype(np.float32),
            "u8": rng.integers(0, 256, (B, 2, 192, 256, 3), dtype=np.uint8),
            "u8_image2_2": rng.integers(0, 256, (B, 48, 64, 3), dtype=np.uint8),
            "photos": rng.integers(0, 256, (B, 2, H, W, 3), dtype=np.uint8),
            "K": K}


def test_interleaved_call_kinds_equal_their_eager_results(synthetic_weights):
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    from demon_b200.networks_original import DemonPipeline, Session
    session = Session(precision="3xtf32")
    session.load_weights(synthetic_weights)
    pipe = DemonPipeline(session, batch_size=B, iterations=ITERATIONS)
    sets = [make_inputs(11), make_inputs(12)]
    x = {k: torch.from_numpy(v).cuda() for k, v in sets[0].items()}                     # the same tensors every call
    hx = {k: torch.from_numpy(sets[0][k]).pin_memory() for k in ("image_pair", "image2_2")}

    def load(inputs):
        for k in x:
            x[k].copy_(torch.from_numpy(inputs[k]))
        for k in hx:
            hx[k].copy_(torch.from_numpy(inputs[k]))

    def host(_):
        o = {"predict_depth0": torch.empty(B, 1, 192, 256).pin_memory(), "predict_rotation": torch.empty(B, 3).pin_memory(),
             "predict_translation": torch.empty(B, 3).pin_memory()}
        pipe.forward_host(hx["image_pair"], hx["image2_2"], o["predict_depth0"], o["predict_rotation"], o["predict_translation"])
        return o

    kinds = {
        "forward": lambda o: pipe.forward(x["image_pair"], x["image2_2"], outputs=o),
        "forward_median": lambda o: pipe.forward(x["image_pair"], None, outputs=o),
        "snapshots_refined": lambda o: pipe.forward_snapshots(x["image_pair"], x["image2_2"], refine=True, outputs=o),
        "snapshots": lambda o: pipe.forward_snapshots(x["image_pair"], x["image2_2"], refine=False, outputs=o),
        "u8": lambda o: pipe.forward_u8(x["u8"], x["u8_image2_2"], outputs=o),
        "images_resize": lambda o: pipe.forward_images(x["photos"], image2_2="resize", outputs=o),
        "images_median": lambda o: pipe.forward_images(x["photos"], image2_2="median", outputs=o),
        "views": lambda o: pipe.forward_views(x["photos"], x["K"], outputs=o),
        "host": host,
    }

    def launches(kind):
        return pipe.snapshot_launches() if kind in SNAPSHOT_KINDS else pipe.launches()

    def fresh(kind):
        if kind == "host":
            return None   # its device outputs are the net's own buffers
        own = pipe.own_snapshot_outputs(kind == "snapshots_refined") if kind in SNAPSHOT_KINDS else pipe.own_outputs()
        return {k: torch.empty_like(v) for k, v in own.items()}

    # eager references on fresh output tensors, kept alive so that no later tensor reuses their addresses (the host
    # entry's second reference call already captures: its call is the same for both input sets)
    refs, counts, keep = {}, {}, []
    for s, inputs in enumerate(sets):
        load(inputs)
        for kind, call in kinds.items():
            keep.append(fresh(kind))
            refs[s, kind] = {k: v.clone() for k, v in call(keep[-1]).items()}
            assert counts.setdefault(kind, launches(kind)) == launches(kind), kind
        for k, v in refs[s, "host"].items():   # the same bits as forward() on the same inputs
            assert torch.equal(v, refs[s, "forward"][k].cpu()), k

    order = ("forward", "snapshots_refined", "u8", "images_median", "forward_median", "views", "snapshots", "host", "images_resize")
    for rnd in range(3):   # the pipeline's own outputs: eager, capture, replay (the host entry: replays)
        s = rnd % 2
        load(sets[s])
        for kind in order:
            got = {k: v.clone() for k, v in kinds[kind](None).items()}
            assert launches(kind) == counts[kind], (kind, rnd)
            assert set(got) == set(refs[s, kind]), (kind, rnd)
            for k, v in refs[s, kind].items():
                assert torch.equal(got[k], v), (kind, k, rnd)
    _lib.check_errors()
