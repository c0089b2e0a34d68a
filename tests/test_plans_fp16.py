"""CPU, no device: the FP16 precision's plans (DEMON_PREC_FP16, conv_tc_halo_kernel MODE 1).

FP16 packs the weights at 64 bytes per 32-channel row instead of 128 (TF32) or 256 (3xTF32 hi and lo), so its class blocks
and weight ring slots are smaller and more layers may keep their weights resident.  It must not lose a layer: every conv
of the v1 and v2 nets that has a tensor-core plan at 3xTF32 has one at FP16 and conversely, each inside the shared-memory
budget and described as mode 1.  And the variant table of tests/test_conv_variants.py reaches every FP16 instantiation
that tests/test_gpu_conv_fp16.py runs."""
import re

import pytest

from test_conv_variants import VARIANTS, X3TF32, describe, features, required_targets
from test_gpu_conv_fold import FOLD_ROWS, fold_of
from test_v2_plan import describe_plan

FP16 = 3
SMEM_BUDGET = 224 * 1024 + 1024   # the plan's operand stages plus the 1 KB alignment slack (conv_tc_halo.cu: kSmemBudget)
CONFIGS = {"b64": (64, (192, 256)), "b1": (1, (192, 256)), "refine1024": (8, (768, 1024))}
# Rows (the VARIANTS format) for what the variant tables no longer reach at FP16, whose weights are four times smaller:
# the one halo split-K row of VARIANTS and the ring-weight rows of FOLD_ROWS keep their weights resident there
FP16_ROWS = [
    (1, 16, 8, 512, 48, 3, 3, 1, 1, 0, 64, 4),     # halo split-K, weight ring
    (1, 48, 64, 256, 24, 3, 3, 1, 1, 0, 0, 4),     # FOLD 3, 24 weight blocks through the ring
]


def tc_plans(variant, batch, refine_hw, precision):
    """{layer: plan text} of the layers that get a tensor-core plan."""
    out = {}
    for name, (g, tap0, text) in describe_plan(variant, batch, refine_hw, precision).items():
        plan = text.split(" : ", 1)[1] if text.startswith("tap0") else text
        if plan.startswith("halo "):
            out[name] = plan
    return out


def field(plan, key):
    return int(re.search(r" %s (\d+)" % key, plan).group(1))


def class_block(plan):
    """Bytes of one class block: every step's weight bytes divided by the classes it multiplies."""
    sizes = {int(w) // bin(int(c, 16)).count("1") for c, w in re.findall(r"\[c([0-9a-f]+) w\d+\+(\d+)\]", plan)}
    assert len(sizes) == 1, plan
    return sizes.pop()


@pytest.mark.parametrize("variant", (1, 2), ids=["v1", "v2"])
@pytest.mark.parametrize("config", sorted(CONFIGS))
def test_fp16_plans_the_same_layers_as_3xtf32(variant, config):
    batch, refine_hw = CONFIGS[config]
    x3 = tc_plans(variant, batch, refine_hw, X3TF32)
    f16 = tc_plans(variant, batch, refine_hw, FP16)
    assert x3, "no tensor-core layer at 3xTF32"
    assert sorted(f16) == sorted(x3), set(f16) ^ set(x3)
    for name, plan in f16.items():
        assert field(plan, "mode") == 1, (name, plan)
        assert field(plan, "smem") <= SMEM_BUDGET, (name, plan)
        # the fold mode takes the same heads at every precision (its tile is fixed by the layer's shape)
        assert fold_of(plan) == fold_of(x3[name]), (name, plan, x3[name])
        # an FP16 class block is a quarter of 3xTF32's [W_hi ; W_lo] for the same N tile (fold mode: N = taps x Cout)
        if field(plan, "n_tile") == field(x3[name], "n_tile"):
            assert class_block(plan) * 4 == class_block(x3[name]), (name, plan, x3[name])
    wres = lambda plans: sum(field(p, "wres") for p in plans.values())
    print("\n%s %s: %d tensor-core layers, weights resident in %d at FP16, %d at 3xTF32" % (
        ("v1", "v2")[variant - 1], config, len(f16), wres(f16), wres(x3)))
    assert wres(f16) >= wres(x3)


def test_variant_rows_reach_every_fp16_instantiation():
    """The FP16 counterparts of test_conv_variants.py's targets (every instantiation, resident and ring weights, split-K,
    the A and weight rings) and both fold instantiations, reached by the rows tests/test_gpu_conv_fp16.py runs (VARIANTS,
    FP16_ROWS and test_gpu_conv_fold.py's FOLD_ROWS)."""
    reached = set()
    for row in VARIANTS + FP16_ROWS:
        d = describe(row, FP16)
        assert d is not None and d["mode"] == 1, row
        reached |= features(row, d)
    # a transposed convolution's step of all four classes always fits at FP16 (4 x 64 x 64 bytes per slot at N 64), so
    # steps are never capped at 2 classes
    want = {t for t in required_targets() if "mode 0" not in t and "mode 2" not in t and "at most 2 classes" not in t[-1]}
    want |= {tuple("mode 1" if e == "mode 2" else e for e in t) for t in required_targets() if "mode 2" in t}
    # FP16 weight slots are a quarter of 3xTF32's, so the halo mode's A ring gets more stages: every ring size still
    # reached is wrapped, and 4 stages always are
    got_rings = {t for t in reached if "A ring" in t[-1]}
    want = {t for t in want if "A ring" not in t[-1]} | got_rings
    assert ("halo", "mode 1", "a CTA wraps the A ring of 4 stages") in got_rings
    missing = sorted(want - reached)
    assert not missing, "FP16 targets no VARIANTS row reaches: %s" % missing
    folds = {}
    for row in FOLD_ROWS + FP16_ROWS:
        d = describe(row, FP16)
        if fold_of(d["text"]):
            assert d["mode"] == 1 and d["kind"] == "halo" and d["ksplit"] == 1, d["text"]
            folds.setdefault(fold_of(d["text"]), set()).add(d["wres"])
    assert folds == {9: {1}, 3: {0, 1}}, folds
