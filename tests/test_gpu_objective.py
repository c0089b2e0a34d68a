"""GPU: demon_b200.v2.objective for every evolution of training/v2/training.py against the float64 oracle
(tests/objective_oracle.py) on a training batch of datareader.build_batch, at 3xTF32 and fp32: each selected loss, the
regularisation and the total within 1e-4 relative."""
import numpy as np
import pytest
import torch

from demon_b200.v2 import objective as dobj
from demon_b200.v2 import weights as W2

import objective_oracle as oobj
from test_gpu_blocks_v2 import training_batch

pytestmark = pytest.mark.gpu

TOL = 1e-4


@pytest.fixture(scope="module")
def weights():
    return W2.synthetic_weights(0)


@pytest.fixture(scope="module")
def sessions(weights):
    from demon_b200.v2.networks import Session
    out = {}
    for prec in ("fp32", "3xtf32"):
        out[prec] = Session(precision=prec)
        out[prec].load_weights(weights)
    return out


@pytest.fixture(scope="module")
def batch():
    return training_batch(4, 9)


@pytest.fixture(scope="module")
def earlier():
    """Predictions of an earlier iteration for the batch's last two samples (4_iterative, 5_refine): 2 new + 2 earlier."""
    rng = np.random.RandomState(1)
    n = np.zeros((2, 3, 48, 64), np.float32)
    n[:, 2] = -1
    return {"predict_depth2": rng.uniform(0.4, 0.6, (2, 1, 48, 64)).astype(np.float32), "predict_normal2": n,
            "predict_rotation": np.array([[0.01, -0.02, 0.01], [0.0, 0.01, -0.01]], np.float32),
            "predict_translation": np.array([[0.9, 0.1, -0.05], [0.95, 0.0, 0.1]], np.float32)}


@pytest.fixture(scope="module")
def oracle(weights, batch, earlier):
    host = {k: v.cpu().numpy() for k, v in batch.items()}
    out = {e: oobj.objective(weights, host, e) for e in dobj.EVOLUTIONS}
    for e in ("4_iterative", "5_refine"):
        out[e + "+earlier"] = oobj.objective(weights, host, e, earlier)
    return out


def compare(got, ref):
    assert list(got) == list(ref)
    for k, r in ref.items():
        v = got[k]
        assert isinstance(v, torch.Tensor) and v.is_cuda and v.dim() == 0 and v.dtype == torch.float32, k
        v = float(v)
        assert abs(v - r) <= TOL * abs(r) if r != 0 else v == 0, (k, v, r)


@pytest.mark.parametrize("prec", ("fp32", "3xtf32"))
@pytest.mark.parametrize("evolution", dobj.EVOLUTIONS)
def test_objective_against_fp64_oracle(sessions, batch, oracle, evolution, prec):
    compare(dobj.objective(sessions[prec], batch, evolution), oracle[evolution])


@pytest.mark.parametrize("evolution", ("4_iterative", "5_refine"))
def test_objective_with_earlier_iterations(sessions, batch, earlier, oracle, evolution):
    """netFlow1 and netDM1 on the two new samples; netFlow2 on all four, the last two from the earlier predictions."""
    prev = {k: torch.from_numpy(v).cuda() for k, v in earlier.items()}
    got = dobj.objective(sessions["3xtf32"], batch, evolution, prev)
    compare(got, oracle[evolution + "+earlier"])
    assert float(got["total"]) != float(dobj.objective(sessions["3xtf32"], batch, evolution)["total"])


def test_objective_refuses_earlier_iterations_before_4_iterative(sessions, batch, earlier):
    with pytest.raises(ValueError, match="prev_predictions"):
        dobj.objective(sessions["fp32"], batch, "3_dm2", earlier)
