"""The loss gradient kernels of csrc/losses.cu bit for bit against their kernel-order restatement (oracle/loss_grads.py,
itself held to oracle/losses.py's independent float64 gradients by tests/test_loss_grads.py), and the forward's on-the-fly
SIG tiles pixel by pixel through the eps-0 mean.

Shapes: training.py's (batch 32: flow and confidence [32,2,48,64], level 5 [32,2,6,8], depth2 / normal2 [32,1|3,48,64],
depth0 / normal0 [32,1|3,192,256], pose [32,3]) -- the only ones where sig_u_kernel's and pointwise_grad_kernel's
grid-stride loops and the forward's 264-slot cap run more than once -- plus every plane width in {1, 16, 17, 63, 64, 65,
129} against every height in {1, 15, 16, 17, 33} (the 64x16 tiles' seams and ragged edges) and plane counts that put
several tiles on one CTA.  Inputs hold NaN, +-inf and 0 in prediction and target, and values where pr - gt cancels.
"""
import ctypes
import gc
import math
import time

import numpy as np
import pytest
import torch

from demon_b200 import _lib
from demon_b200 import lmbspecialops as sops
from demon_b200.v2 import losses as L
from oracle import loss_grads as LG
from oracle import losses as OL

pytestmark = pytest.mark.gpu

DT = {torch.float32: np.float32, torch.float64: np.float64}
UPSTREAM = {"loss_flow5": 0.75, "loss_flow2": -1.25, "loss_conf5": 0.5, "loss_conf2": 1.5, "loss_flow2_sig": -0.75, "loss_conf2_sig": 1.25,
            "loss_depth2": 0.75, "loss_depth2_sig": -1.25, "loss_normal2": 0.5, "loss_rotation": 1.5, "loss_translation": -0.75,
            "loss_translation_no_factor": 0.25, "loss_depth0": 0.75, "loss_depth0_sig": -1.25, "loss_normal0": 1.5}
FLOW_ARGS = dict(flow_weight=1.7, conf_weight=0.3, flow_sig_weight=2.5, conf_sig_weight=0.8)
DN_ARGS = dict(depth_weight=300.0, depth_sig_weight=1500.0, normal_weight=50.0, rotation_weight=160.0, translation_weight=15.0,
               translation_factor=1.3)
REFINE_ARGS = dict(depth_weight=300.0, depth_sig_weight=1500.0, normal_weight=100.0)
WIDTHS = (1, 16, 17, 63, 64, 65, 129)
HEIGHTS = (1, 15, 16, 17, 33)


def flow_combos():
    """(pr_conf2, pr_conf5, flow_sig_weight set, conf_sig_weight set, conf_diff_scale, level5_factor): every option set of
    tests/golden/make_losses_golden.py, training.py's level5_factor=0 and conf_diff_scale=10 among them."""
    import itertools
    out = [c + (1, 0.5) for c in itertools.product((True, False), repeat=4)]
    return out + [(True, True, True, True, 10, 0.0), (True, False, True, True, 2.5, 0.25)]


@pytest.fixture(scope="module", autouse=True)
def wall_time_and_peak_memory():
    """Reports this module's wall time and peak device memory, then leaves the device idle for later modules."""
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    yield
    torch.cuda.synchronize()
    print("\ntest_gpu_loss_grads: %.1f s, peak device memory %.1f MiB" % (time.time() - t0, torch.cuda.max_memory_allocated() / 2 ** 20))
    gc.collect()
    torch.cuda.empty_cache()


def _np(t):
    return t.detach().cpu().numpy()


def assert_bits(got, want, what):
    g = _np(got) if isinstance(got, torch.Tensor) else np.asarray(got)
    assert g.dtype == want.dtype and g.shape == want.shape, (what, g.dtype, want.dtype, g.shape, want.shape)
    iv = np.int32 if g.dtype == np.float32 else np.int64
    bad = g.view(iv) != want.view(iv)
    if bad.any():
        i = tuple(int(v[0]) for v in np.nonzero(bad))
        raise AssertionError("%s: %d of %d elements differ, first at %s: %r, want %r" % (what, int(bad.sum()), bad.size, i, g[i], want[i]))


# ---- inputs ---------------------------------------------------------------------------------------------------------------
def _poison(rng, a, frac=0.03):
    """NaN, +inf, -inf and 0 at frac of the elements."""
    m = rng.rand(*a.shape)
    a = a.copy()
    a[m < frac / 4] = np.nan
    a[(m >= frac / 4) & (m < frac / 2)] = np.inf
    a[(m >= frac / 2) & (m < 3 * frac / 4)] = -np.inf
    a[(m >= 3 * frac / 4) & (m < frac)] = 0.0
    return a


def _cancel(rng, pr, gt, dtype, frac=0.02):
    """Targets of +-1e4 and predictions a few ulp from them at frac of the elements: pr - gt cancels."""
    m = rng.rand(*pr.shape) < frac
    big = np.where(rng.rand(*pr.shape) < 0.5, 1e4, -1e4).astype(dtype)
    pr, gt = pr.copy(), gt.copy()
    gt[m] = big[m]
    pr[m] = (big + rng.randint(-3, 4, pr.shape) * np.spacing(big))[m]
    return pr, gt


def _cuda(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a)).to("cuda", dtype)


def _sig(x, eps):
    """The 10-channel SIG stack from the mirror op, one call per delta."""
    return torch.cat([sops.scale_invariant_gradient(x, [d], [1], eps) for d in LG.SIG_DELTAS], 1)


def flow_inputs(n, h, w, h5, w5, dtype, seed):
    rng = np.random.RandomState(seed)
    nd = DT[dtype]
    g2, g5 = rng.normal(0, 0.1, (n, 2, h, w)).astype(nd), rng.normal(0, 0.1, (n, 2, h5, w5)).astype(nd)
    p2, g2 = _cancel(rng, _poison(rng, g2 + rng.normal(0, 0.02, g2.shape).astype(nd)), _poison(rng, g2, 0.01), nd)
    p5 = _poison(rng, g5 + rng.normal(0, 0.02, g5.shape).astype(nd))
    gsig = _poison(rng, _np(_sig(_cuda(g2, dtype), 0.001)), 0.01)
    c2, c5 = rng.uniform(0.05, 1.0, p2.shape).astype(nd), rng.uniform(0.05, 1.0, p5.shape).astype(nd)
    c2 = _poison(rng, c2, 0.01)
    return {k: _cuda(v, dtype) for k, v in dict(gt_flow2=g2, gt_flow5=g5, gt_flow2_sig=gsig, pr_flow2=p2, pr_flow5=p5, pr_conf2=c2,
                                                   pr_conf5=c5).items()}


def depth_inputs(n, h, w, dtype, seed):
    """depth [n,1,h,w], its target and SIG target stack, normals [n,3,h,w], poses [n,3]."""
    rng = np.random.RandomState(seed)
    nd = DT[dtype]
    gd = rng.uniform(0.2, 2.0, (n, 1, h, w)).astype(nd)
    pd, gd = _cancel(rng, _poison(rng, np.abs(gd + rng.normal(0, 0.1, gd.shape)).astype(nd)), _poison(rng, gd, 0.01), nd)
    gsig = _poison(rng, _np(_sig(_cuda(gd, dtype), 0.001)), 0.01)
    gn = rng.uniform(-1, 1, (n, 3, h, w)).astype(nd)
    pn = _poison(rng, gn + rng.normal(0, 0.1, gn.shape).astype(nd))
    gr, gt = rng.uniform(-0.1, 0.1, (n, 3)).astype(nd), rng.uniform(-0.5, 0.5, (n, 3)).astype(nd)
    pr, pt = gr + rng.normal(0, 0.05, (n, 3)).astype(nd), gt + rng.normal(0, 0.05, (n, 3)).astype(nd)
    pr[0, 0] = gr[0, 0]   # x = 0: the L1 gradient's 0 / sqrt(eps)
    return {k: _cuda(v, dtype) for k, v in dict(gt_depth=gd, gt_sig=gsig, gt_normal=gn, gt_rotation=gr, gt_translation=gt, pr_depth=pd,
                                                   pr_normal=pn, pr_rotation=pr, pr_translation=pt).items()}


def upstream_tensors(dtype):
    """UPSTREAM as device scalars, made before any graph capture (a host-to-device copy cannot be captured)."""
    return {k: torch.tensor(v, dtype=dtype, device="cuda") for k, v in UPSTREAM.items()}


def _backward(result, ups=None):
    outs, grads = [], []
    for k, v in result.items():
        if v.requires_grad:
            outs.append(v)
            grads.append(ups[k] if ups is not None else torch.tensor(UPSTREAM[k], dtype=v.dtype, device="cuda"))
    torch.autograd.backward(outs, grads)


def run_flow(inp, combo):
    c2, c5, fs, cs, scale, l5 = combo
    pr = {k: inp[k].clone().requires_grad_(True) for k in ("pr_flow2", "pr_flow5", "pr_conf2", "pr_conf5")}
    r = L.flow_loss_block(inp["gt_flow2"], inp["gt_flow5"], inp["gt_flow2_sig"], pr["pr_flow2"], pr["pr_flow5"], pr["pr_conf2"] if c2 else None,
                          pr["pr_conf5"] if c5 else None, FLOW_ARGS["flow_weight"], FLOW_ARGS["conf_weight"],
                          FLOW_ARGS["flow_sig_weight"] if fs else None, FLOW_ARGS["conf_sig_weight"] if cs else None, conf_diff_scale=scale,
                          level5_factor=l5)
    _backward(r)
    return {k: v.grad for k, v in pr.items() if v.grad is not None}


def want_flow(inp, combo):
    c2, c5, fs, cs, scale, l5 = combo
    n = {k: _np(v) for k, v in inp.items()}
    conf2 = _np(L.compute_confidence_map(inp["pr_flow2"], inp["gt_flow2"], scale))   # the device's own target (exp in double)
    conf5 = _np(L.compute_confidence_map(inp["pr_flow5"], inp["gt_flow5"], scale))
    return LG.flow_block_grads(n["gt_flow2"], n["gt_flow5"], n["gt_flow2_sig"], n["pr_flow2"], n["pr_flow5"], n["pr_conf2"] if c2 else None,
                               n["pr_conf5"] if c5 else None, FLOW_ARGS["flow_weight"], FLOW_ARGS["conf_weight"],
                               FLOW_ARGS["flow_sig_weight"] if fs else None, FLOW_ARGS["conf_sig_weight"] if cs else None, UPSTREAM,
                               conf_diff_scale=scale, level5_factor=l5, conf2=conf2, conf5=conf5)


def run_depth_blocks(inp):
    """(depthnormal gradients, refine gradients) of the same depth inputs."""
    pr = {k: inp[k].clone().requires_grad_(True) for k in ("pr_depth", "pr_normal", "pr_rotation", "pr_translation")}
    r = L.depthnormal_loss_block(inp["gt_depth"], inp["gt_sig"], inp["gt_normal"], inp["gt_rotation"], inp["gt_translation"], pr["pr_depth"],
                                 pr["pr_normal"], pr["pr_rotation"], pr["pr_translation"], **DN_ARGS)
    _backward(r)
    dn = {"pr_depth2": pr["pr_depth"].grad, "pr_normal2": pr["pr_normal"].grad, "pr_rotation": pr["pr_rotation"].grad,
          "pr_translation": pr["pr_translation"].grad}
    d, nn = inp["pr_depth"].clone().requires_grad_(True), inp["pr_normal"].clone().requires_grad_(True)
    r = L.depth_refine_loss_block(inp["gt_depth"], inp["gt_sig"], inp["gt_normal"], d, nn, **REFINE_ARGS)
    _backward(r)
    return dn, {"pr_depth0": d.grad, "pr_normal0": nn.grad}


def want_depth_blocks(inp):
    n = {k: _np(v) for k, v in inp.items()}
    dn = LG.depthnormal_block_grads(n["gt_depth"], n["gt_sig"], n["gt_normal"], n["gt_rotation"], n["gt_translation"], n["pr_depth"],
                                    n["pr_normal"], n["pr_rotation"], n["pr_translation"], upstream=UPSTREAM, **DN_ARGS)
    rf = LG.depth_refine_block_grads(n["gt_depth"], n["gt_sig"], n["gt_normal"], n["pr_depth"], n["pr_normal"], upstream=UPSTREAM,
                                     **REFINE_ARGS)
    return dn, rf


def assert_grads(got, want, what):
    assert sorted(got) == sorted(k for k, v in want.items() if v is not None), what
    for k in got:
        assert_bits(got[k], want[k], "%s %s" % (what, k))


# ---- bit-for-bit gradients of every block --------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=[torch.float32, torch.float64], ids=["f32", "f64"])
def training_flow(request):
    return request.param, flow_inputs(32, 48, 64, 6, 8, request.param, 21)


@pytest.mark.parametrize("j", range(len(flow_combos())))
def test_flow_block_gradients_bit_for_bit_at_training_shapes(training_flow, j):
    dtype, inp = training_flow
    combo = flow_combos()[j]
    assert_grads(run_flow(inp, combo), want_flow(inp, combo), "flow combo %d %s" % (j, dtype))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_depth_block_gradients_bit_for_bit_at_training_shapes(dtype):
    """depthnormal at depth2's [32,1,48,64] / [32,3,48,64] with poses [32,3]; refine at depth0's [32,1,192,256] /
    [32,3,192,256]: 1536 SIG tiles against sig_u_kernel's 1056 CTAs, 6144 blocks' worth of pixels against
    pointwise_grad_kernel's 1056."""
    inp = depth_inputs(32, 48, 64, dtype, 22)
    dn, _ = run_depth_blocks(inp)
    want_dn, _ = want_depth_blocks(inp)
    assert_grads(dn, want_dn, "depthnormal")
    inp = depth_inputs(32, 192, 256, dtype, 23)
    _, rf = run_depth_blocks(inp)
    _, want_rf = want_depth_blocks(inp)
    assert_grads(rf, want_rf, "refine")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("h", HEIGHTS)
@pytest.mark.parametrize("w", WIDTHS)
def test_block_gradients_bit_for_bit_at_tile_seams_and_ragged_edges(w, h, dtype):
    inp = flow_inputs(2, h, w, (h + 1) // 2, (w + 1) // 2, dtype, 100 * w + h)
    for j in (0, 16):   # every option; training.py's level5_factor=0, conf_diff_scale=10
        assert_grads(run_flow(inp, flow_combos()[j]), want_flow(inp, flow_combos()[j]), "flow %dx%d combo %d" % (h, w, j))
    inp = depth_inputs(3, h, w, dtype, 100 * w + h + 1)
    dn, rf = run_depth_blocks(inp)
    want_dn, want_rf = want_depth_blocks(inp)
    assert_grads(dn, want_dn, "depthnormal %dx%d" % (h, w))
    assert_grads(rf, want_rf, "refine %dx%d" % (h, w))


def test_refine_gradients_bit_for_bit_with_more_than_two_tiles_per_cta():
    """240 planes of 33x129: 2160 tiles, more than two per sig_u_kernel CTA, and 4000 blocks' worth of pixels."""
    inp = depth_inputs(240, 33, 129, torch.float32, 24)
    _, rf = run_depth_blocks(inp)
    _, want_rf = want_depth_blocks(inp)
    assert_grads(rf, want_rf, "refine 240x33x129")


# ---- the C ABI: term tables built directly --------------------------------------------------------------------------------
def term(kind, pr, gt, n, c, h, w, eps=LG.EPS, s_eps=0.0, gt_plane=False, gt_s_eps=0.0, weight=1.0, weight_dev=None, out=None, out0=None,
         grad_out=None, grad=None, accumulate=False):
    t = L._Term()
    t.kind, t.c, t.h, t.w, t.n, t.gt_plane, t.accumulate = kind, c, h, w, n, int(gt_plane), int(accumulate)
    t.pr, t.gt = pr.data_ptr(), (gt.data_ptr() if gt is not None else None)
    t.eps, t.sig_eps, t.gt_sig_eps, t.weight = eps, s_eps, gt_s_eps, weight
    for name, v in (("weight_dev", weight_dev), ("out", out), ("out0", out0), ("grad_out", grad_out), ("grad", grad)):
        setattr(t, name, v.data_ptr() if v is not None else None)
    return t


def table(*terms):
    arr = (L._Term * len(terms))(*terms)
    return ctypes.cast(arr, ctypes.c_void_p), len(terms), arr


def ws_bytes(tab, dtype, backward):
    p, num, _ = tab
    return _lib.load().demon_loss_workspace_bytes(p, num, 4 if dtype == torch.float32 else 8, int(backward))


def call(entry, tab, dtype, ws, nbytes):
    p, num, _ = tab
    sfx = "_f32" if dtype == torch.float32 else "_f64"
    return getattr(_lib.load(), entry + sfx)(p, num, ws.data_ptr() if ws is not None else None, nbytes, sops._stream())


GUARD = 4096   # sentinel elements on each side of every buffer


class Guarded:
    """A buffer of `shape` inside a sentinel-filled block, pre-filled with `fill`."""

    def __init__(self, shape, dtype, fill=float("nan")):
        self.n = int(np.prod(shape))
        self.block = torch.full((self.n + 2 * GUARD,), 1.2345e-7, dtype=dtype, device="cuda")
        self.block[GUARD:GUARD + self.n] = fill
        self.t = self.block[GUARD:GUARD + self.n].view(shape)

    def guards_intact(self):
        s = torch.cat([self.block[:GUARD], self.block[GUARD + self.n:]])
        return bool((s == torch.tensor(1.2345e-7, dtype=s.dtype)).all())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_cabi_backward_writes_every_element_and_nothing_else(dtype):
    """A mixed table: L2 then SIG on a depth, L2 then gt_plane SIG on a 2N-plane confidence, L1 on a pose, and a SIG term
    without a gradient.  U starts as NaN in a workspace exactly demon_loss_workspace_bytes long followed by a guarded tail;
    each gradient starts as NaN inside a guarded block.  Every element must come out as the restatement's bits, every
    guard unchanged, the launch count exactly one per L2 / L1 term and two per SIG term with a gradient."""
    n, h, w = 5, 33, 129
    inp = depth_inputs(n, h, w, dtype, 31)
    fl = flow_inputs(n, h, w, 3, 4, dtype, 32)
    conf_t = L.compute_confidence_map(fl["pr_flow2"], fl["gt_flow2"], 10)
    rows = (n, 3 * 1)
    pr_r, gt_r = inp["pr_rotation"], inp["gt_rotation"]
    s1, s3 = LG.sig_eps(0.01), LG.sig_eps(0.001)
    gd, gc, gr = Guarded((n, 1, h, w), dtype), Guarded((n, 2, h, w), dtype), Guarded((n, 3), dtype)
    g = {k: torch.tensor(v, dtype=dtype, device="cuda") for k, v in (("a", 0.75), ("b", -1.25), ("c", 0.5), ("d", 1.5), ("e", -0.75))}
    tab = table(term(L._L2, inp["pr_depth"], inp["gt_depth"], n, 1, h, w, weight=300.0, grad_out=g["a"], grad=gd.t),
                term(L._SIG, inp["pr_depth"], inp["gt_sig"], n, 1, h, w, s_eps=s1, weight=1500.0, grad_out=g["b"], grad=gd.t, accumulate=True),
                term(L._L2, fl["pr_conf2"], conf_t, n, 2, h, w, weight=0.3, grad_out=g["c"], grad=gc.t),
                term(L._SIG, fl["pr_conf2"], conf_t, 2 * n, 1, h, w, s_eps=s3, gt_plane=True, gt_s_eps=s3, weight=0.8, grad_out=g["d"],
                     grad=gc.t, accumulate=True),
                term(L._L1, pr_r, gt_r, 1, rows[0] * rows[1], 1, 1, weight=160.0 / n, grad_out=g["e"], grad=gr.t),
                term(L._SIG, fl["pr_flow2"], fl["gt_flow2_sig"], 2 * n, 1, h, w, s_eps=s3, weight=2.5))
    nbytes = ws_bytes(tab, dtype, True)
    elem = 4 if dtype == torch.float32 else 8
    assert nbytes == 2 * n * 10 * h * w * elem
    ws = Guarded((nbytes // elem,), dtype)
    lib = _lib.load()
    c0 = lib.demon_launch_count()
    assert call("demon_loss_backward", tab, dtype, ws.t, nbytes - elem) != 0   # one element short: refused before any launch
    assert lib.demon_launch_count() == c0
    torch.cuda.synchronize()
    assert torch.isnan(gd.t).all() and torch.isnan(gc.t).all() and torch.isnan(gr.t).all()
    assert call("demon_loss_backward", tab, dtype, ws.t, nbytes) == 0
    assert lib.demon_launch_count() - c0 == 1 + 2 + 1 + 2 + 1
    torch.cuda.synchronize()
    nd = {k: _np(v) for k, v in inp.items()}
    nf = {k: _np(v) for k, v in fl.items()}
    ct = _np(conf_t)
    T = LG.Term
    want_d = LG.table_grads([T(LG.L2, 0, nd["gt_depth"], LG.EPS, 300.0), T(LG.SIG, 0, nd["gt_sig"], LG.EPS, 1500.0, s1)], [nd["pr_depth"]],
                            [0.75, -1.25])[0]
    want_c = LG.table_grads([T(LG.L2, 0, ct, LG.EPS, 0.3), T(LG.SIG, 0, ct, LG.EPS, 0.8, s3, gt_plane=True, gt_s_eps=s3)], [nf["pr_conf2"]],
                            [0.5, 1.5])[0]
    want_r = LG.term_grad(T(LG.L1, 0, nd["gt_rotation"].reshape(1, -1), LG.EPS, 160.0 / n), nd["pr_rotation"].reshape(1, -1), -0.75)
    assert_bits(gd.t, want_d, "depth L2 + SIG")
    assert_bits(gc.t, want_c, "confidence L2 + gt_plane SIG")
    assert_bits(gr.t, want_r.reshape(n, 3), "rotation L1")
    for b in (gd, gc, gr, ws):
        assert b.guards_intact()
    # the forward: two launches whatever the table
    o = [torch.empty(2, dtype=dtype, device="cuda") for _ in range(6)]
    ftab = table(*[term(t.kind, _Ptr(t.pr), _Ptr(t.gt), t.n, t.c, t.h, t.w, s_eps=t.sig_eps, gt_plane=bool(t.gt_plane), gt_s_eps=t.gt_sig_eps,
                        weight=t.weight, out=o[i][0:1], out0=o[i][1:2]) for i, t in enumerate(tab[2])])
    fb = ws_bytes(ftab, dtype, False)
    fws = torch.empty(fb, dtype=torch.uint8, device="cuda")
    c0 = lib.demon_launch_count()
    assert call("demon_loss_forward", ftab, dtype, fws, fb) == 0
    assert lib.demon_launch_count() - c0 == 2


class _Ptr:
    """A raw device pointer standing in for a tensor in term()."""

    def __init__(self, p):
        self.p = p

    def data_ptr(self):
        return self.p


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_cabi_null_grad_out_writes_zeros_and_adds_them(dtype):
    n, h, w = 2, 17, 65
    inp = depth_inputs(n, h, w, dtype, 41)
    s1 = LG.sig_eps(0.01)
    nd = {k: _np(v) for k, v in inp.items()}
    lib = _lib.load()
    for kind, gt, want_t in ((L._L2, inp["gt_depth"], LG.Term(LG.L2, 0, nd["gt_depth"], LG.EPS, 300.0)),
                             (L._SIG, inp["gt_sig"], LG.Term(LG.SIG, 0, nd["gt_sig"], LG.EPS, 300.0, s1))):
        zero = LG.term_grad(want_t, nd["pr_depth"], None)
        assert (zero == 0).all()
        buf = Guarded((n, 1, h, w), dtype)
        tab = table(term(kind, inp["pr_depth"], gt, n, 1, h, w, s_eps=s1, weight=300.0, grad=buf.t))
        nbytes = ws_bytes(tab, dtype, True)
        ws = torch.full((max(1, nbytes),), 255, dtype=torch.uint8, device="cuda")
        assert call("demon_loss_backward", tab, dtype, ws, nbytes) == 0
        torch.cuda.synchronize()
        assert_bits(buf.t, zero, "grad_out NULL, kind %d" % kind)
        prev = torch.from_numpy(np.random.RandomState(kind).normal(0, 1, (n, 1, h, w))).to("cuda", dtype)
        buf.t.copy_(prev)
        tab = table(term(kind, inp["pr_depth"], gt, n, 1, h, w, s_eps=s1, weight=300.0, grad=buf.t, accumulate=True))
        assert call("demon_loss_backward", tab, dtype, ws, nbytes) == 0
        torch.cuda.synchronize()
        assert_bits(buf.t, _np(prev) + zero, "grad_out NULL accumulated, kind %d" % kind)
        assert buf.guards_intact()
    # a term without a gradient buffer launches nothing
    tab = table(term(L._L2, inp["pr_depth"], inp["gt_depth"], n, 1, h, w))
    c0 = lib.demon_launch_count()
    assert call("demon_loss_backward", tab, dtype, None, 0) == 0
    assert lib.demon_launch_count() == c0


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_cabi_weight_dev_replaces_the_host_weight(dtype):
    n, h, w = 3, 16, 64
    inp = depth_inputs(n, h, w, dtype, 51)
    nd = {k: _np(v) for k, v in inp.items()}
    s1 = LG.sig_eps(0.01)
    wdev = torch.tensor(0.3 * 1.7, dtype=dtype, device="cuda")
    wv = _np(wdev)[()]
    g = torch.tensor(-1.25, dtype=dtype, device="cuda")
    for kind, gt, want_t in ((L._L2, inp["gt_depth"], LG.Term(LG.L2, 0, nd["gt_depth"], LG.EPS, wv)),
                             (L._SIG, inp["gt_sig"], LG.Term(LG.SIG, 0, nd["gt_sig"], LG.EPS, wv, s1))):
        buf = Guarded((n, 1, h, w), dtype)
        out = torch.empty(2, dtype=dtype, device="cuda")
        tab = table(term(kind, inp["pr_depth"], gt, n, 1, h, w, s_eps=s1, weight=99.0, weight_dev=wdev, grad_out=g, grad=buf.t,
                         out=out[0:1], out0=out[1:2]))
        nbytes = ws_bytes(tab, dtype, True)
        ws = torch.empty(max(1, nbytes), dtype=torch.uint8, device="cuda")
        assert call("demon_loss_backward", tab, dtype, ws, nbytes) == 0
        fb = ws_bytes(tab, dtype, False)
        assert call("demon_loss_forward", tab, dtype, torch.empty(fb, dtype=torch.uint8, device="cuda"), fb) == 0
        torch.cuda.synchronize()
        assert_bits(buf.t, LG.term_grad(want_t, nd["pr_depth"], -1.25), "weight_dev kind %d" % kind)
        mean = _np(out)[0]
        unweighted = torch.empty(2, dtype=dtype, device="cuda")
        tab1 = table(term(kind, inp["pr_depth"], gt, n, 1, h, w, s_eps=s1, weight=1.0, out=unweighted[0:1], out0=unweighted[1:2]))
        assert call("demon_loss_forward", tab1, dtype, torch.empty(fb, dtype=torch.uint8, device="cuda"), fb) == 0
        assert mean == wv * _np(unweighted)[0]


# ---- the forward's SIG tiles, pixel by pixel, through the eps-0 mean ------------------------------------------------------
def sig_out0(pr, gt, planes, h, w, s_eps, gt_plane=False, gt_s_eps=0.0):
    dtype = pr.dtype
    o = torch.full((2,), float("nan"), dtype=dtype, device="cuda")
    tab = table(term(L._SIG, pr, gt, planes, 1, h, w, s_eps=s_eps, gt_plane=gt_plane, gt_s_eps=gt_s_eps, out=o[0:1], out0=o[1:2]))
    fb = ws_bytes(tab, dtype, False)
    assert call("demon_loss_forward", tab, dtype, torch.empty(fb, dtype=torch.uint8, device="cuda"), fb) == 0
    return _np(o)[1]


SEAM_SHAPES = [(h, w) for w in WIDTHS for h in HEIGHTS]
ZERO_SHAPES = [(8, h, w) for h, w in SEAM_SHAPES] + [(32, 192, 256), (64, 48, 64), (64, 6, 8), (240, 33, 129)]


def _base(planes, h, w, dtype, seed, nan=True):
    rng = np.random.RandomState(seed)
    b = rng.uniform(1.0, 2.0, (planes, h, w))
    b[rng.rand(planes, h, w) < 0.5] *= -1
    if nan:
        b[rng.rand(planes, h, w) < 0.02] = np.nan
    return _cuda(b, dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("planes,h,w", ZERO_SHAPES)
def test_forward_sig_tiles_equal_the_op_exactly(planes, h, w, dtype):
    """The prediction against the mirror op's stack of itself, NaNs included: every on-the-fly SIG value equals the op's, so
    every difference is 0 and the eps-0 mean exactly +0.  The same with the target taken on the fly (gt_plane, equal eps)."""
    base = _base(planes, h, w, dtype, planes + h + w)
    s1 = LG.sig_eps(0.01)
    v = sig_out0(base, _sig(base, s1), planes, h, w, s1)
    assert v == 0 and not np.signbit(v), v
    s3 = LG.sig_eps(0.001)
    v = sig_out0(base, base, planes, h, w, s3, gt_plane=True, gt_s_eps=s3)
    assert v == 0 and not np.signbit(v), v


def probe_positions(h, w):
    """Where a one-hot probe goes: tile corners, the last row and column of a tile (their +d neighbours lie in the halo),
    x = w-1-d and y = h-1-d for every delta, the ragged last tiles, the first and last pixel of the plane."""
    p = [(0, 0), (h - 1, w - 1), (15, 63), (16, 64), (0, 63), (15, 0), (0, 64), (16, 0), (31, 127), (0, w - 1), (h - 1, 0), (17, 70),
         (h - 1, (w - 1) // 64 * 64), ((h - 1) // 16 * 16, w - 1)]
    p += [(min(5, h - 1), w - 1 - d) for d in LG.SIG_DELTAS] + [(h - 1 - d, min(70, w - 1)) for d in LG.SIG_DELTAS]
    out = []
    for y, x in p:
        if 0 <= y < h and 0 <= x < w and (y, x) not in out:
            out.append((y, x))
    return out


PROBE_SHAPES = [(len(probe_positions(h, w)) + 3, h, w) for h, w in SEAM_SHAPES] + [(32, 192, 256), (64, 48, 64), (240, 33, 129)]


@pytest.mark.parametrize("gt_plane", [False, True], ids=["stack", "gt_plane"])
@pytest.mark.parametrize("planes,h,w", PROBE_SHAPES)
def test_forward_sig_tiles_one_hot_probes(planes, h, w, gt_plane):
    """One pixel per plane perturbed, at the positions of probe_positions in turn, planes late in the tile order included
    (the tiles a slot visits on its second and later strides).  Each probe changes at most 11 per-pixel terms; all of them
    lie within a factor 2^19 of each other, so the device's double sum is exact in any order and the eps-0 mean must be
    float32(fsum(terms) / M) bit for bit.  A skipped or doubly visited tile, or a wrong halo read, changes it."""
    dtype = torch.float32
    base = _base(planes, h, w, dtype, 7 * planes + h + w, nan=False)
    pos = probe_positions(h, w)
    pr = base.clone()
    rng = np.random.RandomState(planes + h)
    for z in range(planes):
        y, x = pos[z % len(pos)]
        pr[z, y, x] += float(rng.choice([-0.75, 0.5, 0.625]))
    s1 = LG.sig_eps(0.01)
    if gt_plane:
        got = sig_out0(pr, base, planes, h, w, s1, gt_plane=True, gt_s_eps=s1)
        terms = LG.sig_terms(_np(pr), _np(base), np.float32(0), s1, gt_plane=True, gt_s_eps=s1)
    else:
        gt = _sig(base, s1)
        got = sig_out0(pr, gt, planes, h, w, s1)
        terms = LG.sig_terms(_np(pr), _np(gt), np.float32(0), s1)
    nz = terms[terms != 0].astype(np.float64)
    assert nz.size <= 11 * planes and (nz.size > 0 or h * w == 1)
    if nz.size:   # 24 significand bits, the exponent span and the count's bits fit in a double: every partial sum is exact
        span = int(np.floor(np.log2(nz.max())) - np.floor(np.log2(nz.min())))
        assert nz.max() / nz.min() < 2.0 ** 19 and 24 + span + int(np.ceil(np.log2(nz.size + 1))) <= 53, (span, nz.size)
    want = np.float32(math.fsum(nz.tolist()) / terms.size)
    assert got.view(np.int32) == want.view(np.int32), (got, want)


# ---- the forward losses at training.py's shapes, and one CUDA graph of forward and backward ------------------------------
def _ulp32(x):
    return float(np.spacing(np.float32(abs(float(x)))))


def test_forward_losses_within_one_ulp_of_the_oracle_at_training_shapes():
    dtype = torch.float32
    fl = flow_inputs(32, 48, 64, 6, 8, dtype, 61)
    n = {k: _np(v) for k, v in fl.items()}
    for c2, c5, fs, cs, scale, l5 in (flow_combos()[0], flow_combos()[16]):
        got = L.flow_loss_block(fl["gt_flow2"], fl["gt_flow5"], fl["gt_flow2_sig"], fl["pr_flow2"], fl["pr_flow5"], fl["pr_conf2"], fl["pr_conf5"],
                                conf_diff_scale=scale, level5_factor=l5, **FLOW_ARGS)
        want = OL.flow_loss_block(n["gt_flow2"], n["gt_flow5"], n["gt_flow2_sig"], n["pr_flow2"], n["pr_flow5"], n["pr_conf2"], n["pr_conf5"],
                                  conf_diff_scale=scale, level5_factor=l5, **FLOW_ARGS)
        assert list(got) == list(want)
        for k in want:
            assert abs(float(got[k]) - float(want[k])) <= 1.01 * _ulp32(want[k]), (k, float(got[k]), float(want[k]))
    for h, w, block in ((48, 64, "dn"), (192, 256, "refine")):
        d = depth_inputs(32, h, w, dtype, 62 + h)
        nd = {k: _np(v) for k, v in d.items()}
        if block == "dn":
            got = L.depthnormal_loss_block(d["gt_depth"], d["gt_sig"], d["gt_normal"], d["gt_rotation"], d["gt_translation"], d["pr_depth"],
                                           d["pr_normal"], d["pr_rotation"], d["pr_translation"], **DN_ARGS)
            want = OL.depthnormal_loss_block(nd["gt_depth"], nd["gt_sig"], nd["gt_normal"], nd["gt_rotation"], nd["gt_translation"],
                                             nd["pr_depth"], nd["pr_normal"], nd["pr_rotation"], nd["pr_translation"], **DN_ARGS)
        else:
            got = L.depth_refine_loss_block(d["gt_depth"], d["gt_sig"], d["gt_normal"], d["pr_depth"], d["pr_normal"], **REFINE_ARGS)
            want = OL.depth_refine_loss_block(nd["gt_depth"], nd["gt_sig"], nd["gt_normal"], nd["pr_depth"], nd["pr_normal"], **REFINE_ARGS)
        assert list(got) == list(want)
        for k in want:   # one rounding of the mean; two for the products and the ratio of two such losses
            n_ulp = 2.01 if k.endswith(("loss_translation", "rot_transl_loss_ratio")) else 1.01
            assert abs(float(got[k]) - float(want[k])) <= n_ulp * _ulp32(want[k]), (block, k, float(got[k]), float(want[k]))


def test_graph_replay_of_forward_and_backward_equals_the_restatement():
    """The flow block (every option) and the refine block at training.py's shapes, forward and backward captured in one CUDA
    graph on fresh buffers, replayed: the gradients equal the restatement, not just an eager run."""
    dtype = torch.float32
    fl = flow_inputs(32, 48, 64, 6, 8, dtype, 71)
    d = depth_inputs(32, 192, 256, dtype, 72)
    fp = {k: fl[k].clone().requires_grad_(True) for k in ("pr_flow2", "pr_flow5", "pr_conf2", "pr_conf5")}
    dp, np_ = d["pr_depth"].clone().requires_grad_(True), d["pr_normal"].clone().requires_grad_(True)

    def step():
        r = L.flow_loss_block(fl["gt_flow2"], fl["gt_flow5"], fl["gt_flow2_sig"], fp["pr_flow2"], fp["pr_flow5"], fp["pr_conf2"], fp["pr_conf5"],
                              conf_diff_scale=10, level5_factor=0.0, **FLOW_ARGS)
        r.update(L.depth_refine_loss_block(d["gt_depth"], d["gt_sig"], d["gt_normal"], dp, np_, **REFINE_ARGS))
        _backward(r, ups)
    ups = upstream_tensors(dtype)
    leaves = list(fp.values()) + [dp, np_]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            for x in leaves:
                x.grad = None
            step()
    torch.cuda.current_stream().wait_stream(s)
    for x in leaves:
        x.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for x in leaves:   # the captured backward wrote into the graph's own buffers: poison them, then replay
        x.grad.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    want = want_flow(fl, flow_combos()[16])
    for k, x in fp.items():
        assert_bits(x.grad, want[k], "graph flow " + k)
    _, want_rf = want_depth_blocks(d)
    assert_bits(dp.grad, want_rf["pr_depth0"], "graph depth0")
    assert_bits(np_.grad, want_rf["pr_normal0"], "graph normal0")
    del g
