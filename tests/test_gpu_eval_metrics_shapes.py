"""The PRDC tile kernels and the device Frechet distance at the size of the FID-50k evaluation, against float64
(pytest -m gpu).

PRDC (metrics/prdc.py:_compute_prdc_cuda, csrc/metrics.cu) replaces the reference's three N x N sklearn distance matrices
by 64 x 64 fp64 distance tiles reduced on the fly: row_sqnorm_kernel, then prdc_radii_kernel (per row, the k+1 smallest
distances in per-thread sorted lists, merged across the 16 lanes of a half-warp by "pop the global minimum; the lowest
owning lane pops") once for the real and once for the fake set, then prdc_cross_kernel (per fake column the number of
real rows whose radius holds it, per real row "any fake inside its own radius" and "nearest fake inside the real
radius", through shared / global atomics and shuffles).  The outputs each launch is handed (sqnorm_ws, radii, col_count,
row_any, row_cov) are checked element by element, and compute_prdc's four values as the product reports them.

Cases, each at a size the product runs:
1. FID-50k, train split: 50 000 real x 50 000 fake 2048-d features, k = 5 (WORKER.evaluate's nearest_k); 782 row tiles x
   782 column tiles, the last one 16 wide (50 000 = 781 * 64 + 16).
2. The valid split and the folder evaluator: 10 000 real (the CIFAR-10 test split) x 50 000 fake, so the real and fake
   sets run on different grids.
3. Mode collapse and memorisation, 4 000 x 4 000 (62 full tiles and one of 32), k = 5.  Groups of bitwise-identical fake
   rows, placed in one lane's list (the same (c % 64) / 4, in one tile and across tiles), in different lanes of one
   half-warp, in different column tiles and in different row CTAs, with fewer than k+1 copies (the radius is a genuine
   neighbour behind a run of exact ties in the merge) and with k+1 or more (the radius is rounding-level).  Identical
   rows give bit-identical distances, so a merge that pops every owner of a tied minimum moves the radius by a rank.
   Memorised rows: for a real row i whose (k+1)-th neighbour (self included) is the real row m, a bitwise copy of m goes
   into the fake set.  The radius pass and the cross pass then evaluate r_i and d(i, copy) from the same operands in the
   same order (the same fma chain, then acc + acc, |x|^2 + |y|^2 and one subtraction in both kernels), so the two are
   bit-identical and, the comparison being strict, the pair is outside.  These pairs are certain-out, for every real row
   whose (k+1)-th neighbour is m, and so is (m, j) against the radius of every fake row j whose (k+1)-th neighbour is
   the copy (fma and the additions commute).  The counts of the copies' columns are asserted exactly.
4. Both sides of the kernel's k limit (kMaxK1 = 8 entries per list): k = 1, 3 and 7 (7 fills the list) on the kernels,
   and k = 8, which sgb_prdc_radii refuses and compute_prdc sends to its host tensor path; at n = k+1 (every row's list
   holds the whole set), 64 (one tile) and 65 (a tile plus a one-row tile), D = 2048.

Features: seeded on the device, non-negative and correlated like pooled post-ReLU Inception features (per-dimension scale
0.5..1.5, 32 shared factors), around 300 class centres, so that k-NN radii (d^2 ~ 430) sit far below the bulk distance
(d^2 ~ 6 800).  The fake set drops a quarter of the modes, shifts half of the rest and puts 15 % of its samples around
centres of no real mode.  They are drawn in fp32, the Inception output type, and handed over as float64, as the worker
does.  Cases 1-3 assert precision, recall and coverage in [0.05, 0.95] and density in (0.05, 2): no decision set is
trivially all-in or all-out.  Every buffer a test hands a kernel starts as a sentinel (NaN, bytes 0xAB; col_count too,
which the launch must zero), so a row or column no thread writes fails.

Reference: plain float64 torch on the GPU, in row blocks of 4096: d^2 = |x|^2 + |y|^2 - 2 x.y by cuBLAS DGEMM, clamped at
0, the self-distance 0 for X vs X, the radius the (k+1)-th smallest d^2 of a row (topk, largest=False).  Nothing on the
reference side calls the library.

Decision margins.  PRDC is made of strict comparisons d < r, and two correct fp64 evaluations can disagree on a pair whose
distance is within rounding of the radius, so each decision is exact except inside a rigorous margin, in the d^2 domain:
* One evaluation of d^2 in any summation order: |x|^2 and |y|^2 are sums of D products (error <= gamma_D each), 2 x.y is
  (<= 2 gamma_D |x||y| <= gamma_D (|x|^2 + |y|^2)), and the two additions add <= 3u (|x|^2 + |y|^2) (u = 2^-53,
  d^2 <= 2 (|x|^2 + |y|^2)).  So |err| <= EPS (|x|^2 + |y|^2) with EPS = 2 gamma_{D+2}, gamma_n = n u / (1 - n u): twice
  the bound of one dot product, because d^2 is assembled from three sums.  Clamping at 0 only moves it closer.
* The kernel's and the reference's d^2 of a pair differ by <= 2 EPS (|x_i|^2 + |y_j|^2); a k-th smallest value moves by
  no more than the values it is taken from, so the radii differ by <= 2 EPS (|x_i|^2 + max_k |x_k|^2) (the radius check,
  plus 5u r^2 for the kernel's sqrt and the test's squaring).
* The kernel compares fl(sqrt(d^2)) < fl(sqrt(r^2)): false whenever d^2 >= r^2, true whenever d^2 < r^2 (1 - 5u).
* So for a decision against the radius of row i of set X:  delta_ij = 2 EPS (|x_i|^2 + |y_j|^2)
  + 2 EPS (|x_i|^2 + max_k |x_k|^2) + 5u r_i^2.  A pair is certain-in if d^2_ref < r^2_ref - delta, certain-out if
  d^2_ref >= r^2_ref + delta, ambiguous otherwise.  Then: count_lo <= col_count <= count_lo + (ambiguous in the column);
  row_any / row_cov are 1 where the row has a certain-in pair and 0 where it has neither certain-in nor ambiguous pairs
  (row_cov: min_j d_ij < r_i is "some pair inside"); each of the four values lies between the values of the certain
  decisions and of the certain plus ambiguous ones, at most (ambiguous pairs) / N apart.
* sqnorm_ws: |rn - |x|^2_ref| <= 2 gamma_D |x|^2.
The number of ambiguous pairs of each case is printed and must be <= 1e-6 of the pairs, so the margin does not hollow out
the check (EPS (|x|^2 + |y|^2) ~ 2e-8 against radii d^2 ~ 430).

Frechet distance (metrics/fid.py:frechet_distance_device: tr sqrt(S1 S2) as sum sqrt(lambda(S1^1/2 S2 S1^1/2)), two
cuSOLVER symmetric eigendecompositions) against frechet_inception_distance (the reference's scipy sqrtm, float64) on the
same moments, each finalised by MomentsAccumulator from 2048-d features (the recipe of the FID-50k moments test, a small
mean shift and scale between the sets):
* full rank, 50 000 vs 50 000, FID ~ 23 while tr S1 + tr S2 ~ 4 600, the regime where the final subtraction cancels;
  called as WORKER.evaluate calls it, the reference statistics arriving as numpy arrays.  Bound 1e-10 (tr S1 + tr S2);
* rank deficient, 50 000 vs 1 000 (< D: S2 singular, sqrtm ill-conditioned), called as the folder evaluator calls it.
  Bound 1e-6 (tr S1 + tr S2).
Both bounds are estimates.  On an H100 80GB HBM3 (700 W) these cases agreed with scipy to 1e-15 and 4e-9 of
tr S1 + tr S2, and the same form with LAPACK's eigh in place of cuSOLVER to 1e-15 and 1.4e-8 on sets drawn like these;
the eigenvalues near zero of the singular case are resolved only to ~sqrt(u ||M||) each.  Both bounds sit far inside
the +-0.5 % FID target, which is asserted too.
"""
import numpy as np
import pytest
import torch

from test_gpu_norm_shapes import _cuda

pytestmark = pytest.mark.gpu

f64 = torch.float64
D = 2048
K_EVAL = 5                      # WORKER.evaluate's nearest_k
MODES, FACTORS, NOISE = 300, 32, 0.35
BLOCK = 4096                    # reference row block
U = 2.0 ** -53
EPS = 2.0 * (D + 2) * U / (1.0 - (D + 2) * U)     # one evaluation of d^2: |err| <= EPS (|x|^2 + |y|^2)
SQRT_REL = 5.0 * U              # fl(sqrt) on the kernel side, squaring of the kernel radius on the test side
AMB_FRAC = 1e-6
FID_TR_REL = {"full-rank": 1e-10, "rank-deficient": 1e-6}
FID_TARGET = 5e-3               # the +-0.5 % FID target
SENTINEL_U8 = 0xAB
SENTINEL_I32 = 0xABABABAB - (1 << 32)


# ------------------------------------------------------------------------------------------------ features
def _space(dev):
    """Per-dimension scale and the class centres (in units of the scale), shared by the real and fake sets."""
    g = torch.Generator(device=dev).manual_seed(21)
    std = 0.5 + torch.rand(D, generator=g, device=dev)
    return std, 1.2 * torch.randn(MODES, D, generator=g, device=dev)


def _features(space, n, seed, fake=False):
    """n features, fp32 values handed over as float64: std * max(0, 3 + centre + NOISE * (0.6 z + 0.8 shared factor))."""
    std, centres = space
    dev = std.device
    g = torch.Generator(device=dev).manual_seed(seed)
    if fake:
        kept = torch.rand(MODES, generator=g, device=dev).argsort()[:3 * MODES // 4]       # a quarter of the modes dropped
        moved = (torch.rand(len(kept), 1, generator=g, device=dev) < 0.5).to(centres.dtype)  # half of the rest shifted
        c = centres[kept] + 0.25 * moved * torch.randn(len(kept), D, generator=g, device=dev)
        cen = c[torch.randint(0, len(kept), (n,), generator=g, device=dev)]
        off = torch.rand(n, generator=g, device=dev) < 0.15                                 # off-manifold samples
        cen[off] = 1.2 * torch.randn(int(off.sum()), D, generator=g, device=dev)
    else:
        cen = centres[torch.randint(0, MODES, (n,), generator=g, device=dev)]
    shared = torch.randn(n, FACTORS, generator=g, device=dev)
    z = 0.6 * torch.randn(n, D, generator=g, device=dev) + 0.8 * shared[:, torch.arange(D, device=dev) % FACTORS]
    return (std * (3.0 + cen + NOISE * z).clamp(min=0.0)).float().to(f64)


# ------------------------------------------------------------------------------------------------ float64 reference
def _d2(a, b, a2, b2):
    return torch.addmm(a2[:, None] + b2[None, :], a, b.t(), alpha=-2.0).clamp_(min=0.0)


def _ref_radii(x, k1):
    """Per row of x: |x|^2, the k1-th smallest d^2 to the rows of x (self zeroed), the row it belongs to, and whether
    that row is separated from the (k1-1)-th and (k1+1)-th by more than the kernel / reference disagreement can bridge
    (then the kernel's k1-th smallest is the same row)."""
    n = x.shape[0]
    x2 = (x * x).sum(1)
    r2 = torch.empty(n, dtype=f64, device=x.device)
    arg = torch.empty(n, dtype=torch.long, device=x.device)
    sep = torch.empty(n, dtype=torch.bool, device=x.device)
    x2max = x2.max()
    for s in range(0, n, BLOCK):
        e = min(s + BLOCK, n)
        d = _d2(x[s:e], x, x2[s:e], x2)
        d[torch.arange(e - s, device=x.device), torch.arange(s, e, device=x.device)] = 0.0
        v, idx = torch.topk(d, min(k1 + 1, n), dim=1, largest=False)
        del d
        r2[s:e], arg[s:e] = v[:, k1 - 1], idx[:, k1 - 1]
        gap = 4.0 * EPS * (x2[s:e] + x2max)
        ok = torch.ones(e - s, dtype=torch.bool, device=x.device)
        if k1 >= 2:
            ok &= v[:, k1 - 1] - v[:, k1 - 2] > gap
        if v.shape[1] > k1:
            ok &= v[:, k1] - v[:, k1 - 1] > gap
        sep[s:e] = ok
    return dict(x2=x2, r2=r2, arg=arg, sep=sep, tol=2.0 * EPS * (x2 + x2max) + SQRT_REL * r2)


def _memorised_pairs(memorised, rr, rf, dev):
    """The pairs whose kernel distance is bit-identical to the radius it is compared with, for each real row m copied
    bitwise into fake column c: (i, c) for every real row i with m at its radius (against r_real[i]), and (m, j) for
    every fake row j with c at its radius (against r_fake[j]: fma and the additions commute, so swapping the two
    operands changes no bit).  Only rows whose radius row is certain (sep) are taken; the rest stay ambiguous."""
    pr, pf = [], []
    for m, c in memorised:
        pr += [(int(i), c) for i in torch.nonzero((rr["arg"] == m) & rr["sep"]).flatten()]
        pf += [(m, int(j)) for j in torch.nonzero((rf["arg"] == c) & rf["sep"]).flatten()]
    return [torch.tensor(p, dtype=torch.long, device=dev).reshape(-1, 2) for p in (pr, pf)]


def _certain_out(lo_in, lo_out, pairs, s, e):
    sel = (pairs[:, 0] >= s) & (pairs[:, 0] < e)
    if bool(sel.any()):
        i, j = pairs[sel, 0] - s, pairs[sel, 1]
        lo_in[i, j], lo_out[i, j] = False, True


def _ref_cross(real, fake, rr, rf, designed_real, designed_fake):
    """Bounds on the cross outputs from certain / ambiguous decisions (module docstring).  designed_real / designed_fake:
    [P, 2] (real row, fake column) pairs whose distance equals the real / fake radius bit for bit on the kernel side
    (_memorised_pairs): certain-out."""
    nr, nf = real.shape[0], fake.shape[0]
    dev = real.device
    out = dict(count_lo=torch.zeros(nf, dtype=torch.long, device=dev), amb_col=torch.zeros(nf, dtype=torch.long, device=dev))
    for name in ("cov_in", "cov_amb", "any_in", "any_amb"):
        out[name] = torch.zeros(nr, dtype=torch.bool, device=dev)
    n_amb = 0
    for s in range(0, nr, BLOCK):
        e = min(s + BLOCK, nr)
        d = _d2(real[s:e], fake, rr["x2"][s:e], rf["x2"])
        pair_m = 2.0 * EPS * (rr["x2"][s:e, None] + rf["x2"][None, :])
        # against the real radius: density / precision (per column), coverage (per row)
        m = pair_m + (rr["tol"][s:e])[:, None]
        r2 = rr["r2"][s:e, None]
        lo_in, lo_out = d < r2 - m, d >= r2 + m
        _certain_out(lo_in, lo_out, designed_real, s, e)
        amb = ~(lo_in | lo_out)
        out["count_lo"] += lo_in.sum(0)
        out["amb_col"] += amb.sum(0)
        out["cov_in"][s:e], out["cov_amb"][s:e] = lo_in.any(1), amb.any(1)
        n_amb += int(amb.sum())
        # against the fake radius: recall (per row)
        m = pair_m + rf["tol"][None, :]
        r2 = rf["r2"][None, :]
        lo_in, lo_out = d < r2 - m, d >= r2 + m
        _certain_out(lo_in, lo_out, designed_fake, s, e)
        amb = ~(lo_in | lo_out)
        out["any_in"][s:e], out["any_amb"][s:e] = lo_in.any(1), amb.any(1)
        n_amb += int(amb.sum())
        del d, pair_m, m, lo_in, lo_out, amb
    out["n_amb"] = n_amb
    return out


# ------------------------------------------------------------------------------------------------ the kernels
def _kernel_outputs(real, fake, k):
    """sgb_prdc_radii on both sets and sgb_prdc_cross, every output buffer starting as a sentinel."""
    from sgb200 import _lib as L
    (nr, Dr), nf = real.shape, fake.shape[0]
    dev = real.device
    nan = lambda n: torch.full((n,), float("nan"), dtype=f64, device=dev)  # noqa: E731
    o = dict(rn=nan(nr), fn=nan(nf), r_real=nan(nr), r_fake=nan(nf),
             col_count=torch.full((nf,), SENTINEL_I32, dtype=torch.int32, device=dev),
             row_any=torch.full((nr,), SENTINEL_U8, dtype=torch.uint8, device=dev),
             row_cov=torch.full((nr,), SENTINEL_U8, dtype=torch.uint8, device=dev))
    L.call("sgb_prdc_radii", L.ptr(real), nr, Dr, k, L.ptr(o["rn"]), L.ptr(o["r_real"]), L.stream_ptr())
    L.call("sgb_prdc_radii", L.ptr(fake), nf, Dr, k, L.ptr(o["fn"]), L.ptr(o["r_fake"]), L.stream_ptr())
    L.call("sgb_prdc_cross", L.ptr(real), L.ptr(o["rn"]), L.ptr(fake), L.ptr(o["fn"]), L.ptr(o["r_real"]), L.ptr(o["r_fake"]),
           nr, nf, Dr, L.ptr(o["col_count"]), L.ptr(o["row_any"]), L.ptr(o["row_cov"]), L.stream_ptr())
    torch.cuda.synchronize()
    return o


def _ratio(err, tol):
    """max err / tol; NaN (a sentinel left in place) counts as infinitely far."""
    r = err / tol
    return float("inf") if bool(torch.isnan(r).any()) else float(r.max())


def _flag_faults(got, certain, possible):
    """Rows where a 0/1 output is outside {0, 1}, 0 on a certain-in row, or 1 on a row with no possible pair."""
    return int(((got > 1) | ((got == 0) & certain) | ((got == 1) & ~(certain | possible))).sum())


def _check_prdc(case, real, fake, k, memorised=(), spread=True):
    """Kernel outputs and compute_prdc against the float64 decision bounds.  memorised: (real row m, fake column c) with
    fake[c] a bitwise copy of real[m]."""
    from sgb200.metrics import prdc
    nr, nf = real.shape[0], fake.shape[0]
    dev = real.device
    rr, rf = _ref_radii(real, k + 1), _ref_radii(fake, k + 1)
    designed, designed_fake = _memorised_pairs(memorised, rr, rf, dev)
    ref = _ref_cross(real, fake, rr, rf, designed, designed_fake)
    lo, hi = ref["count_lo"], ref["count_lo"] + ref["amb_col"]
    report = {}
    if k + 1 <= 8:
        o = _kernel_outputs(real, fake, k)
        worst = {}
        for name, got, want in (("sqnorm real", o["rn"], rr["x2"]), ("sqnorm fake", o["fn"], rf["x2"])):
            worst[name] = _ratio((got - want).abs(), 2.0 * (D * U / (1.0 - D * U)) * want)
        for name, got, r in (("radii real", o["r_real"], rr), ("radii fake", o["r_fake"], rf)):
            worst[name] = _ratio((got * got - r["r2"]).abs(), r["tol"])
        cc = o["col_count"].long()
        faults = {"col_count": int(((cc < lo) | (cc > hi)).sum()),
                  "row_any": _flag_faults(o["row_any"], ref["any_in"], ref["any_amb"]),
                  "row_cov": _flag_faults(o["row_cov"], ref["cov_in"], ref["cov_amb"])}
        if designed.shape[0]:
            cols = designed[:, 1]
            assert int(ref["amb_col"][cols].sum()) == 0, "a memorised column also holds an ambiguous pair"
            faults["memorised columns"] = int((cc[cols] != lo[cols]).sum())
        report = "worst / bound %s, faults %s" % ({n: "%.3g" % v for n, v in worst.items()}, faults)
        if memorised:
            report += ", memorised pairs %d against r_real, %d against r_fake" % (designed.shape[0], designed_fake.shape[0])
    else:
        # the lists hold kMaxK1 = 8 entries: the entry point refuses k + 1 > 8 and compute_prdc takes the host path
        from sgb200 import _lib as L
        ws, rad = torch.empty(nr, dtype=f64, device=dev), torch.empty(nr, dtype=f64, device=dev)
        with pytest.raises(RuntimeError):
            L.call("sgb_prdc_radii", L.ptr(real), nr, D, k, L.ptr(ws), L.ptr(rad), L.stream_ptr())
        report = "host tensor path"
    got = prdc.compute_prdc(real, fake, k)
    mean = lambda t, n: float(t.sum()) / n  # noqa: E731
    bounds = {"precision": (mean(lo > 0, nf), mean(hi > 0, nf)),
              "recall": (mean(ref["any_in"], nr), mean(ref["any_in"] | ref["any_amb"], nr)),
              "density": (mean(lo, nf) / k, mean(hi, nf) / k),
              "coverage": (mean(ref["cov_in"], nr), mean(ref["cov_in"] | ref["cov_amb"], nr))}
    print("PRDC %s (%d real x %d fake, k = %d): ambiguous pairs %d of %d; %s; %s" % (
        case, nr, nf, k, ref["n_amb"], nr * nf, report,
        ", ".join("%s %.6f [%.6f, %.6f]" % (n, got[n], b[0], b[1]) for n, b in bounds.items())))
    assert ref["n_amb"] <= AMB_FRAC * nr * nf
    if k + 1 <= 8:
        for name, v in worst.items():
            assert v <= 1.0, (name, v)
        assert not any(faults.values()), faults
    for name, (b0, b1) in bounds.items():
        assert b0 - 1e-12 <= got[name] <= b1 + 1e-12, (name, got[name], b0, b1)
    if spread:
        for name in ("precision", "recall", "coverage"):
            assert 0.05 <= got[name] <= 0.95, (name, got[name])
        assert 0.05 < got["density"] < 2.0, got["density"]


# ------------------------------------------------------------------------------------------------ 1, 2. evaluation sizes
@pytest.mark.parametrize("split,n_real,n_fake", [("train", 50000, 50000), ("valid", 10000, 50000)])
def test_prdc_at_fid50k_size_vs_float64(split, n_real, n_fake):
    dev = _cuda()
    sp = _space(dev)
    real, fake = _features(sp, n_real, 1), _features(sp, n_fake, 2, fake=True)
    _check_prdc("FID-50k " + split, real, fake, K_EVAL)


# ------------------------------------------------------------------------------------------------ 3. ties and memorisation
N_COLLAPSE = 4000
# groups of bitwise-identical fake rows (the first is the source); lane of column c in a tile: (c % 64) // 4
TIED_GROUPS = [
    [128, 129, 130],                                   # one lane's list, one tile
    [260, 324, 708, 2180],                             # one lane (c % 64 = 4) across column tiles / row CTAs
    [512, 516, 520],                                   # three lanes of one half-warp, one tile
    [3100, 3300],                                      # two lanes, two tiles
    [1000, 1001, 1005, 1194, 3990],                    # k copies: same lane, next lane, another tile, the ragged tile
    [1500, 1504, 1508, 1564, 1632, 2700],              # k + 1 copies: the radius is rounding-level
    [2000, 2004, 2008, 2012, 2016, 2020, 2576, 2577, 2578, 2579],   # 10 copies over 6 lanes and 2 tiles
]
MEMO_ROWS = [5, 70, 777, 1500, 2049, 3200, 3968, 3999]  # real rows in different row CTAs, the last in the ragged tile
MEMO_COLS = [50, 700, 1800, 2500, 3020, 3500, 3700, 3999]


def test_prdc_mode_collapse_ties_and_memorised_rows_vs_float64():
    dev = _cuda()
    sp = _space(dev)
    k = K_EVAL
    real, fake = _features(sp, N_COLLAPSE, 3), _features(sp, N_COLLAPSE, 4, fake=True)
    used = [c for grp in TIED_GROUPS for c in grp] + MEMO_COLS
    assert len(set(used)) == len(used) and max(used) < N_COLLAPSE
    for grp in TIED_GROUPS:
        fake[grp[1:]] = fake[grp[0]].clone()
    rr = _ref_radii(real, k + 1)
    memorised = []
    for i, col in zip(MEMO_ROWS, MEMO_COLS):
        assert bool(rr["sep"][i]), "memorised row %d: its (k+1)-th neighbour is within rounding of the next" % i
        m = int(rr["arg"][i])
        fake[col] = real[m]
        memorised.append((m, col))
    _check_prdc("mode collapse + memorisation", real, fake, k, memorised)


# ------------------------------------------------------------------------------------------------ 4. the k limit
@pytest.mark.parametrize("n", ["k+1", 64, 65])
@pytest.mark.parametrize("k", [1, 3, 7, 8])
def test_prdc_both_sides_of_the_kernel_k_limit_vs_float64(k, n):
    dev = _cuda()
    n = k + 1 if n == "k+1" else n
    sp = _space(dev)
    _check_prdc("k limit", _features(sp, n, 10 + k), _features(sp, n, 20 + k, fake=True), k, spread=False)


# ------------------------------------------------------------------------------------------------ Frechet distance
def _fid_features(g, std, n, shift, scale):
    """fp32, >= 0, per-dimension mean ~3x the standard deviation, 32 shared factors (the FID-50k moments test's recipe)."""
    dev = std.device
    shared = torch.randn(n, FACTORS, generator=g, device=dev)
    z = 0.6 * torch.randn(n, D, generator=g, device=dev) + 0.8 * shared[:, torch.arange(D, device=dev) % FACTORS]
    return (std * (3.0 + shift + scale * z.clamp(min=-3.0))).float()


def _moments(f):
    from sgb200.metrics import fid
    acc = fid.MomentsAccumulator(D, f.device)
    for s in range(0, f.shape[0], 256):
        acc.update(f[s:s + 256])
    return acc.finalize()


@pytest.fixture(scope="module")
def fid_reference_moments():
    """Per-dimension scale and the moments of the 50 000 reference features."""
    dev = _cuda()
    g = torch.Generator(device=dev).manual_seed(12)
    std = 0.5 + torch.rand(D, generator=g, device=dev)
    mu, sigma = _moments(_fid_features(g, std, 50000, 0.0, 1.0))
    yield std, mu, sigma
    torch.cuda.empty_cache()


@pytest.mark.parametrize("kind,n", [("full-rank", 50000), ("rank-deficient", 1000)])
def test_frechet_distance_device_vs_scipy_sqrtm(fid_reference_moments, kind, n):
    from sgb200.metrics import fid
    std, mu_ref, sigma_ref = fid_reference_moments
    g = torch.Generator(device=std.device).manual_seed(13 + n)
    m, s = _moments(_fid_features(g, std, n, 0.05, 1.03))
    if kind == "full-rank":
        # WORKER.evaluate: generated moments on the device, the pre-computed reference statistics as numpy arrays
        mu_np, sigma_np = mu_ref.cpu().numpy(), sigma_ref.cpu().numpy()
        got = fid.frechet_distance_device(m, s, torch.as_tensor(mu_np, device=m.device),
                                          torch.as_tensor(sigma_np, device=m.device))
        args = (m.cpu().numpy(), s.cpu().numpy(), mu_np, sigma_np)
    else:
        # the folder evaluator: dset1's and the small dset2's moments, both on the device
        got = fid.frechet_distance_device(mu_ref, sigma_ref, m, s)
        args = (mu_ref.cpu().numpy(), sigma_ref.cpu().numpy(), m.cpu().numpy(), s.cpu().numpy())
    want = float(fid.frechet_inception_distance(*args))
    tr = float(np.trace(args[1]) + np.trace(args[3]))
    bound = FID_TR_REL[kind] * tr
    print("FID %s (50000 vs %d): device %.10g, scipy %.10g, tr S1 + tr S2 %.6g, |diff| %.3g = %.3g of the bound "
          "(bound %.3g = %.2g of the 0.5 %% target)" % (kind, n, got, want, tr, abs(got - want), abs(got - want) / bound,
                                                        bound, bound / (FID_TARGET * want)))
    if kind == "full-rank":
        assert 1.0 < want < 30.0 and tr > 1000.0          # the regime where the subtraction cancels
    assert bound <= 0.1 * FID_TARGET * want
    assert abs(got - want) <= bound
