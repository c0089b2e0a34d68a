"""CPU: the table of convolution shapes that reaches every variant of the tensor-core convolution, and the datasets on which
that kernel's arithmetic is exact (both are used by tests/test_gpu_conv_variants.py).

`conv_tc_halo_kernel<PER_TAP, CIN8, MODE, N, NCLS>` has 36 instantiations (halo and per-tap mode: MODE 0 / 2 x (N 16, 32,
64, 128 with one class, N 16, 32, 64 with the four classes of a transposed convolution); 8-channel mode: MODE 0 / 2 x N 16,
32, 64, 128), and the plan of a layer adds resident weights, split-K, several N tiles, transposed-conv steps shared by 1, 2 or
4 classes and per-tap tiles of several images.  What the pipeline does is counted per CTA, at both precisions: a CTA that
loads more A stages than its ring of 2, 3 or 4 has, or more weight blocks than the weight ring's 4 slots, or that runs a
second work item (a CTA moving on to its next tile, with its resident weights reused).  VARIANTS is a table of small shapes;
the planner's own description of each (demon_debug_describe_conv, no device needed) must together reach every one of those
targets, so a planner change that leaves a target untested fails here and names it.

The exact datasets: x, w in {-1, 0, 1} (`int`), x = i + j 2^-11 (`alo`: A_lo = 0 or +-2^-11 after the kernel's truncating
split) or w = i + j 2^-11 (`wlo`: W_lo = 0 or +-2^-11 after the host's round-to-nearest-even split), i, j in {-1, 0, 1},
integer bias.  The dropped term A_lo W_lo is zero, every product is exact, and every partial sum is a multiple of 2^-11 of
magnitude < 2^13 (K <= 8000), i.e. fits 24 bits: no accumulation order or rounding mode changes it.  So 3xTF32 must equal
float32(leaky(float64 reference)) bit for bit, while single-pass TF32, which truncates the 2^-11 parts away, must differ on
`alo` and `wlo`.  test_exact_datasets_emulated pins that property with a numpy model of the kernel's arithmetic.
"""
import ctypes
import re

import numpy as np
import pytest

from demon_b200 import _lib

FP32, X3TF32, TF32 = 0, 1, 2
TC_PRECISIONS = (X3TF32, TF32)
MODE_OF = {X3TF32: 2, TF32: 0}

# (B, H, W, Cin, Cout, kh, kw, sy, sx, deconv, in_off, out_off).  H, W: input size; deconv rows are k4 s2 (kh, kw, sy, sx
# ignored).  The input slice starts at channel in_off of a pixel of in_off + Cin + 4 channels (8-channel rows: the kernel's
# 8-channel mode reads whole 8-channel pixels, so pitch 8, offset 0), the output slice at channel out_off of a pixel of
# out_off + Cout + 4 channels.
VARIANTS = [
    # 8-channel mode
    (2, 16, 8, 8, 16, 3, 3, 1, 1, 0, 0, 32),       # N 16, resident weights
    (1, 32, 16, 8, 24, 9, 1, 2, 1, 0, 0, 4),       # conv1y-like, N 32 (Cout 24: ragged N tile)
    (1, 16, 8, 8, 48, 1, 3, 1, 1, 0, 0, 64),       # N 64
    (1, 16, 8, 8, 96, 3, 1, 1, 1, 0, 0, 512),      # two N tiles of 64, one per CTA
    (17, 32, 16, 8, 96, 3, 3, 1, 1, 0, 0, 64),     # two N tiles: each CTA runs several items and wraps the weight ring
    (17, 64, 64, 8, 16, 1, 3, 1, 1, 0, 0, 32),     # 544 tiles: each CTA reuses its resident weights and wraps the A ring
    (33, 32, 16, 8, 96, 1, 3, 1, 1, 0, 0, 128),    # N 128
    # halo mode, one class
    (1, 16, 8, 32, 16, 1, 3, 1, 1, 0, 32, 4),      # N 16, resident weights
    (1, 32, 16, 32, 24, 1, 9, 1, 2, 0, 64, 32),    # conv1x-like, N 32
    (1, 32, 16, 32, 16, 3, 3, 2, 2, 0, 4, 64),     # netRefine/conv1-like: four stride-parity planes
    (1, 16, 8, 32, 48, 1, 3, 1, 1, 0, 128, 8),     # N 64
    (1, 16, 8, 32, 96, 1, 3, 1, 1, 0, 256, 256),   # two N tiles
    (1, 16, 8, 512, 16, 1, 3, 1, 1, 0, 512, 32),   # split-K
    (2, 32, 16, 64, 64, 7, 1, 2, 1, 0, 64, 64),    # conv2y-like, two chunks
    (33, 32, 16, 32, 96, 1, 3, 1, 1, 0, 32, 128),  # N 128
    (1, 16, 8, 256, 16, 1, 3, 1, 1, 0, 256, 4),    # eight chunks through 4 A stages
    (1, 32, 16, 128, 16, 1, 9, 1, 2, 0, 128, 64),  # four chunks through 3 A stages (TF32)
    (1, 32, 16, 128, 48, 1, 7, 1, 2, 0, 4, 256),   # four chunks through 3 A stages (3xTF32)
    (17, 64, 64, 64, 16, 3, 3, 2, 2, 0, 64, 512),  # four planes, two chunks per tile through 2 A stages, 272 tiles on
                                                   # 132 CTAs reusing their resident weights
    # halo mode, transposed convolutions (four classes)
    (1, 16, 8, 32, 16, 4, 4, 2, 2, 1, 64, 32),     # N 16: steps of 4, 2 and 1 classes
    (1, 16, 8, 32, 24, 4, 4, 2, 2, 1, 32, 4),      # refine0-like, N 32
    (1, 16, 8, 32, 48, 4, 4, 2, 2, 1, 4, 64),      # N 64: steps of at most 2 classes
    (1, 16, 8, 128, 64, 4, 4, 2, 2, 1, 128, 4),    # refine1-like, four chunks
    # per-tap mode, one class
    (1, 5, 7, 32, 16, 1, 3, 1, 1, 0, 32, 4),       # N 16, rows and columns that do not fill the tile
    (3, 5, 7, 32, 16, 3, 3, 1, 1, 0, 4, 32),       # several images per tile, the last tile ragged
    (1, 5, 7, 32, 24, 1, 3, 1, 1, 0, 64, 64),      # N 32
    (1, 5, 7, 32, 48, 3, 1, 1, 1, 0, 128, 128),    # N 64
    (1, 5, 7, 32, 96, 1, 3, 1, 1, 0, 256, 8),      # two N tiles
    (1, 6, 8, 32, 48, 3, 3, 2, 2, 0, 0, 512),      # weight ring
    (1, 6, 8, 256, 16, 3, 3, 2, 2, 0, 256, 32),    # split-K
    (3, 12, 16, 128, 256, 1, 5, 1, 2, 0, 128, 256),  # conv4x-like, ragged images
    (33, 19, 21, 32, 96, 1, 3, 1, 1, 0, 512, 64),  # N 128
    # per-tap mode, transposed convolutions
    (1, 5, 7, 32, 16, 4, 4, 2, 2, 1, 32, 32),      # N 16
    (1, 5, 7, 32, 24, 4, 4, 2, 2, 1, 64, 4),       # N 32
    (1, 5, 7, 32, 48, 4, 4, 2, 2, 1, 4, 128),      # N 64
    (2, 6, 8, 512, 64, 4, 4, 2, 2, 1, 0, 256),     # refine4-like, split-K
]

_PLAN_RE = re.compile(r"halo (\S+) mode (\d) n_tile (\d+) x(\d+) steps (\d+) x (\d+) chunks sa (\d) .* tiles (\d+) ksplit (\d+) "
                      r"wres (\d) tb (\d+) th (\d+) tw (\d+) \|")


def pitches(row):
    """(in_pitch, out_pitch) of a VARIANTS row."""
    B, H, W, Cin, Cout, kh, kw, sy, sx, deconv, in_off, out_off = row
    in_pitch = 8 if Cin == 8 else in_off + Cin + 4
    return in_pitch, out_off + Cout + 4


def out_size(row):
    B, H, W, Cin, Cout, kh, kw, sy, sx, deconv = row[:10]
    return (2 * H, 2 * W) if deconv else (-(-H // sy), -(-W // sx))


def geometry(row):
    """(kh, kw, sy, sx) the entry is called with."""
    return (4, 4, 2, 2) if row[9] else tuple(row[5:9])


def describe(row, precision):
    """The planner's description of a VARIANTS row, parsed; None if the row gets no tensor-core plan."""
    B, H, W, Cin, Cout = row[:5]
    kh, kw, sy, sx = geometry(row)
    in_pitch, out_pitch = pitches(row)
    buf = ctypes.create_string_buffer(8192)
    _lib.load().demon_debug_describe_conv(B, H, W, Cin, in_pitch, Cout, out_pitch, kh, kw, sy, sx, row[9], precision, buf, 8192)
    text = buf.value.decode()
    m = _PLAN_RE.match(text)
    if not m:
        return None
    kind, mode, n, ntiles, nsteps, chunks, sa, tiles, ksplit, wres, tb, th, tw = m.groups()
    widths = sorted({bin(int(c, 16)).count("1") for c in re.findall(r"\[c([0-9a-f]+) ", text)})
    return dict(kind=kind, mode=int(mode), N=int(n), n_tiles=int(ntiles), nsteps=int(nsteps), chunks=int(chunks), sa=int(sa),
                tiles=int(tiles), ksplit=int(ksplit), wres=int(wres), tb=int(tb), th=int(th), tw=int(tw), widths=widths, text=text)


def tc_error_bound(precision, Cin, kh, kw, deconv, ksplit):
    """The coefficient of the tensor-core convolution's per-element error bound |err| <= bound * S, S = sum |x||w| + |b| over
    the terms of an output element; Cin is the channel count the kernel reads (a layer's cin_buf), ksplit the plan's.  With
    n8 = the number of K = 8 wgmma slices summed into an output element:

    * 3xTF32: A_hi = trunc(A) and A_lo = A - A_hi (exact), |A_lo| < 2^-10 |A|, and the tensor cores truncate A_lo to TF32:
      2^-20 |A|.  W_hi = rne(W), |W_lo| <= 2^-11 |W|, truncated to TF32: 2^-21 |W|.  The dropped A_lo W_lo: 2^-21 |A W|.  The
      split costs at most 2^-19 S.  Every one of the 3 n8 wgmma rounds twice (its internal sum and the accumulator add), at
      most one float32 ulp of a partial sum <= S each, 2^-23 S; split-K adds ksplit sums, the epilogue the bias add and the
      leaky ReLU's product: 2 more.  |err| <= (2^-19 + (2 * 3 n8 + ksplit + 2) 2^-23) S.
    * TF32: both operands truncated to TF32, 2^-10 relative each: 2^-9 S, and n8 wgmma: |err| <= (2^-9 + (2 n8 + ksplit + 2) 2^-23) S.

    The split terms follow from the operand formats alone.  The accumulation terms do not: NVIDIA does not document how a
    wgmma rounds its internal sum, and "at most one float32 ulp of S per wgmma" is an assumption about Hopper's tensor
    cores that rests on measurement (tests/test_gpu_conv_variants.py: test_variant_realistic)."""
    n8 = (4 * Cin // 8) if deconv else ((-(-kh * kw // 4)) * 4 if Cin == 8 else kh * kw * Cin // 8)
    split, mult = (2.0 ** -19, 3) if precision == X3TF32 else (2.0 ** -9, 1)
    return split + (2 * mult * n8 + ksplit + 2) * 2.0 ** -23


SMS = 132    # the launch grid is min(work items, SMs): an H100 SXM's 132 (a GPU with fewer SMs gives each CTA more work)
W_RING = 4   # weight ring slots of the kernel (kRing)


def cta_work(d):
    """What the busiest CTA of a launch does: (work items, A-stage loads, weight-block loads).  A work item is a (tile,
    K slice) pair, items are dealt to the CTAs round robin; an item loads one A stage per 32-channel chunk of its K slice
    (halo and 8-channel mode) or per step of every chunk (per-tap mode), and one weight block per step of every chunk unless
    the weights are resident."""
    items = -(-d["tiles"] * d["ksplit"] // SMS)
    chunks = d["chunks"] // d["ksplit"]
    a_loads = items * chunks * (d["nsteps"] if d["kind"] == "per-tap" else 1)
    return items, a_loads, 0 if d["wres"] else items * chunks * d["nsteps"]


def features(row, d):
    """The targets a row's plan reaches.  The pipeline targets count what a CTA actually does: an A ring of `sa` stages is
    only exercised past its first round when one CTA loads more than `sa` stages, the weight ring when it loads more than
    W_RING blocks, resident weights are only reused when a CTA runs a second work item."""
    B, deconv = row[0], row[9]
    Ho, Wo = (row[1], row[2]) if deconv else out_size(row)
    kind, mode = d["kind"], "mode %d" % d["mode"]
    f = {("instantiation", kind, mode, "N %d" % d["N"], "%d class(es)" % (4 if deconv else 1))}
    if kind != "cin8":
        f |= {(kind, "resident weights %d" % d["wres"]), (kind, "split-K %s" % (d["ksplit"] > 1)),
              (kind, "several N tiles %s" % (d["n_tiles"] > 1))}
    items, a_loads, w_loads = cta_work(d)
    if a_loads > d["sa"]:
        f.add((kind, mode, "a CTA wraps the A ring of %d stages" % d["sa"]))
    if items > 1:
        f.add((kind, mode, "a CTA runs several work items"))
        if d["wres"]:
            f.add((kind, mode, "a CTA reuses its resident weights for a later work item"))
    if w_loads > W_RING:
        f.add((kind, mode, "a CTA wraps the weight ring"))
    if deconv:
        f |= {(kind, "transposed-conv step of %d classes" % w) for w in d["widths"]}
        f.add((kind, "transposed-conv steps of at most %d classes" % max(d["widths"])))
    if kind == "per-tap":
        if d["tb"] > 1 and B % d["tb"]:
            f.add((kind, "tile of several images, the last ragged"))
        if Ho % d["th"] or Wo % d["tw"]:
            f.add((kind, "image rows or columns that do not fill the tile"))
    return f


def required_targets():
    t = set()
    for kind in ("halo", "per-tap", "cin8"):
        for mode in (0, 2):
            for n, ncls in ((16, 1), (32, 1), (64, 1), (128, 1), (16, 4), (32, 4), (64, 4)):
                if kind == "cin8" and ncls == 4:
                    continue
                t.add(("instantiation", kind, "mode %d" % mode, "N %d" % n, "%d class(es)" % ncls))
    for kind in ("halo", "per-tap"):
        t |= {(kind, "resident weights 0"), (kind, "resident weights 1"), (kind, "split-K True"), (kind, "split-K False"),
              (kind, "several N tiles True"), (kind, "several N tiles False")}
        t |= {(kind, "transposed-conv step of %d classes" % w) for w in (1, 2, 4)}
        t |= {(kind, "transposed-conv steps of at most %d classes" % w) for w in (2, 4)}
    t |= {("per-tap", "tile of several images, the last ragged"), ("per-tap", "image rows or columns that do not fill the tile")}
    # what a CTA does, at both precisions.  Per-tap stages are 16 KB and 8-channel halos small, so those modes always get 4
    # A stages; the halo mode's larger stages reach 2 and 3.
    stages = {"halo": (2, 3, 4), "per-tap": (4,), "cin8": (4,)}
    for kind in ("halo", "per-tap", "cin8"):
        for mode in ("mode 0", "mode 2"):
            t |= {(kind, mode, "a CTA wraps the A ring of %d stages" % sa) for sa in stages[kind]}
            t |= {(kind, mode, "a CTA runs several work items"), (kind, mode, "a CTA reuses its resident weights for a later work item"),
                  (kind, mode, "a CTA wraps the weight ring")}
    return t


def test_every_row_gets_a_tensor_core_plan_at_both_precisions():
    for row in VARIANTS:
        for prec in TC_PRECISIONS:
            d = describe(row, prec)
            assert d is not None, (row, prec)
            assert d["mode"] == MODE_OF[prec], (row, d["text"])
            macs = row[0] * np.prod(out_size(row)) * row[3] * row[4] * (4 if row[9] else row[5] * row[6])
            assert macs <= 3e8, row   # small enough for a float64 reference


def test_variants_reach_every_kernel_instantiation_and_plan_feature():
    reached = set()
    for row in VARIANTS:
        for prec in TC_PRECISIONS:
            reached |= features(row, describe(row, prec))
    missing = sorted(required_targets() - reached)
    assert not missing, "targets no VARIANTS row reaches any more: %s" % missing


def test_slice_offsets_include_the_networks():
    offs = {r[10] for r in VARIANTS} | {r[11] for r in VARIANTS}
    assert {32, 64, 128, 256, 512} <= offs
    assert all(o % 4 == 0 for o in offs)


# ---- the exact datasets ---------------------------------------------------------------------------------------------
DATASETS = ("int", "alo", "wlo")
LO = 2.0 ** -11


def exact_data(name, xshape, wshape, nbias, rng):
    """(x, w, bias) float32 arrays of dataset `name` (see the module docstring)."""
    def tern(shape):
        return rng.integers(-1, 2, shape).astype(np.float64)
    x, w = tern(xshape), tern(wshape)
    if name == "alo":
        x += tern(xshape) * LO
    elif name == "wlo":
        w += tern(wshape) * LO
    b = rng.integers(-2, 3, nbias).astype(np.float64)
    out = tuple(a.astype(np.float32) for a in (x, w, b))
    assert all(np.array_equal(o, a) for o, a in zip(out, (x, w, b)))
    return out


def _trunc(a):
    return (np.asarray(a, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _rne(a):   # tc_prepare's tf32_round_h
    u = np.asarray(a, np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0xFFF + ((u >> 13) & 1)) & 0xFFFFE000).astype(np.uint32)).view(np.float32)


def _rz32(v):
    """float64 -> float32 rounded toward zero (the least favourable rounding an accumulator could use)."""
    f = v.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(v)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f.astype(np.float64)


def emulate_dot(a, w, three):
    """A model of the kernel's dot product over the last axis: 3xTF32 (A_hi = trunc(A), A_lo = A - A_hi, W_hi = rne(W),
    W_lo = W - W_hi, the tensor cores truncate every operand to TF32) or single-pass TF32 (both operands truncated), one
    wgmma per 8 products whose sum is rounded toward zero to float32 and added to the float32 accumulator, again rounded
    toward zero."""
    a, w = np.asarray(a, np.float32), np.asarray(w, np.float32)
    if three:
        ah = _trunc(a); al = _trunc(a - ah)
        wh = _rne(w); wl = _trunc(w - wh); wh = _trunc(wh)
        pairs = ((ah, wl), (al, wh), (ah, wh))   # the kernel's issue order
    else:
        pairs = ((_trunc(a), _trunc(w)),)
    K = a.shape[-1]
    acc = np.zeros(a.shape[:-1])
    for k0 in range(0, K, 8):
        for p, q in pairs:
            s = (p[..., k0:k0 + 8].astype(np.float64) * q[..., k0:k0 + 8].astype(np.float64)).sum(-1)   # exact here
            acc = _rz32(acc + _rz32(s))
    return acc


def test_exact_datasets_emulated():
    """At the network's largest K (4608 = 512 channels x 9 taps), 3xTF32 reproduces the float64 dot product exactly on all
    three datasets, and single-pass TF32 misses it on `alo` and `wlo` (so those datasets do run through the lo terms)."""
    rng = np.random.default_rng(0)
    K, draws = 4608, 20
    for name in DATASETS:
        x, w, _ = exact_data(name, (draws, K), (draws, K), 1, rng)
        exact = (x.astype(np.float64) * w.astype(np.float64)).sum(-1)
        assert np.array_equal(emulate_dot(x, w, True), exact), name
        single = emulate_dot(x, w, False)
        if name == "int":
            assert np.array_equal(single, exact)
        else:   # a draw can hit the exact sum by chance: the truncation errors of its terms cancel
            assert np.count_nonzero(single != exact) >= draws - 2, name
