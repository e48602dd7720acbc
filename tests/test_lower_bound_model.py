"""Exact CPU model of the filtered sweep's lower bound (derp_cost.cuh: ssdApprox, sqrtApprox, lowerBoundOfCost) against
the exact path's arithmetic (evalCost's exact branch, computeSSD in oracle/derp_oracle.cpp).

The bound pass is only correct if its number never exceeds the exact cost.  Its proof (derp_cost.cuh, DESIGN.md §4)
rests on per-term error constants, on the l2 aggregate of 27 terms with the rounding of both fp32 sums and of
sqrt.approx, and on the kept-set decision of lowerBoundOfCost.  This file re-computes both paths bit for bit in numpy:
  * exact path: fp32 weights (1-xw)(1-yw) ... without FMA, left-to-right four-product sum, (ushort) truncation,
    (d0*d0 + d1*d1) + d2*d2 per sample, ssd += s in dx-outer / dy-inner order;
  * cheap path: x-lerps then y-lerps as fma(w, b - a, a), differences against dst + addend and the bias, fma
    accumulation in the lanes of accB / accBR / accBs and the final adds of ssdApprox;
  * FMA emulated exactly (fp64 product, TwoSum, correction of the double rounding at fp32 midpoints; checked against
    fractions.Fraction below); the real bilerp V exactly in extended precision (weights are multiples of 2^-24,
    texels 16-bit integers: 64 significant bits);
  * sqrt.approx at a relative error of 2^-22 in either direction (the figure the kernel's comment relies on; the PTX
    ISA's stated bound for sqrt.approx.f32 is not larger).
The constants kErrB, kErrU, the final factor and the +0.5 addend are read from the kernel sources, so the model follows
any edit of them."""
import functools
import os
import re
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "facebook360_dep_b200", "csrc")
F32 = np.float32
LD = np.longdouble
SQRT_REL = 2.0 ** -22
EXTREMES = np.array([0, 1, 2, 32767, 32768, 65533, 65534, 65535], np.float32)
# the per-term claims of the proof (derp_cost.cuh, above kErrB)
CLAIM_BILERP, CLAIM_LERP, CLAIM_MID, CLAIM_TERM = 0.0273, 0.0234, 0.5507, 0.56


@functools.lru_cache(maxsize=1)
def kernel_constants():
    with open(os.path.join(CSRC, "derp_cost.cuh")) as f:
        cost = f.read()
    with open(os.path.join(CSRC, "derp_refine.cuh")) as f:
        refine = f.read()
    kerr_b = float(re.search(r"constexpr float kErrB = ([0-9.eE+-]+)f;", cost).group(1))
    kerr_u = float(re.search(r"constexpr float kErrU = ([0-9.eE+-]+)f;", cost).group(1))
    factor = float(re.search(r"/ conf \* ([0-9.eE+-]+)f;", cost).group(1))
    # the lower-bound pass loads the destination tile and the pixel's bias with an explicit addend (sweepLowerKernel)
    lower = refine[refine.index("sweepLowerKernel"):refine.index("struct SeedArgs")]
    tile = re.findall(r"loadDstTile\([^;]*?,\s*([0-9.eE+-]+)f\);", lower)
    pixel = re.findall(r"loadPixelState\([^;]*?,\s*ps,\s*([0-9.eE+-]+)f\);", lower)
    assert len(tile) == 1 and len(pixel) == 1 and tile == pixel, \
        "sweepLowerKernel must pass one literal addend to loadDstTile and loadPixelState: %s %s" % (tile, pixel)
    return kerr_b, kerr_u, factor, float(tile[0])


# ---- exact fp32 arithmetic ------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """RN32(a * b + c) exactly, elementwise on float32 arrays.  a * b is exact in fp64; s + err == a * b + c exactly
    (TwoSum); RN32(s) differs from RN32(s + err) only when s is an fp32 midpoint and err != 0."""
    a, b, c = (np.asarray(v, F32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    err = (p - (s - bb)) + (c64 - bb)
    r = s.astype(F32)
    r64 = r.astype(np.float64)
    toward = np.where(s > r64, F32(np.inf), F32(-np.inf)).astype(F32)
    other = np.nextafter(r, toward)
    mid = (s != r64) & ((r64 + other.astype(np.float64)) * 0.5 == s)
    up = mid & (err * (s - r64) > 0)
    return np.where(up, other, r).astype(F32)


def lerp(a, b, w):
    """lerp1 / lerp2 of derp_cost.cuh: fma(w, b - a, a)."""
    return fma32(w, np.asarray(b, F32) - np.asarray(a, F32), a)


def bilerp_exact(p00, p01, p10, p11, xw, yw):
    """bilerp of CvUtil.h:83-86 as the exact path runs it: fp32, no FMA, left to right; float result."""
    one = F32(1)
    xm, ym = one - xw, one - yw
    w00, w01, w10, w11 = xm * ym, xw * ym, xm * yw, xw * yw
    return ((p00 * w00 + p01 * w01) + p10 * w10) + p11 * w11


def bilerp_cheap(p00, p01, p10, p11, xw, yw):
    return lerp(lerp(p00, p01, xw), lerp(p10, p11, xw), yw)


def bilerp_real(p00, p01, p10, p11, xw, yw):
    """The real-valued bilerp V with the fp32 weights: exact in extended precision (see the module docstring)."""
    x, y = np.asarray(xw, LD), np.asarray(yw, LD)
    return (((1 - x) * (1 - y)) * np.asarray(p00, LD) + (x * (1 - y)) * np.asarray(p01, LD)
            + ((1 - x) * y) * np.asarray(p10, LD) + (x * y) * np.asarray(p11, LD))


def weights_from_positions(p):
    """(xw or yw) = p - round(p) + 0.5 in fp32, as fetchWarp / evalCost form them (roundBiased2)."""
    p = np.asarray(p, F32)
    t = np.floor(p.astype(np.float64) + 0.5).astype(F32)  # floor(RZ(p + .5)) == roundf(p) for p >= 0
    return ((p - t) + F32(0.5)).astype(F32)


# ---- one source: exact and cheap sums ---------------------------------------------------------------------------------
def exact_sums(blk, qb, dst, dbias, xw, yw):
    """Exact path's unscaled (biased, unbiased) fp32 sums.  blk (N,4,4,3) colour texels (rows, cols), qb (N,2,2,3) bias
    texels, dst (N,3,3,3) destination patch (rows, cols), dbias (N,3), xw / yw (N,)."""
    x, y = xw[:, None], yw[:, None]
    bias = dbias - np.floor(bilerp_exact(qb[:, 0, 0], qb[:, 0, 1], qb[:, 1, 0], qb[:, 1, 1], x, y))
    sb = np.zeros(len(xw), F32)
    su = np.zeros(len(xw), F32)
    for c in range(3):      # dx outer
        for r in range(3):  # dy inner
            t = np.floor(bilerp_exact(blk[:, r, c], blk[:, r, c + 1], blk[:, r + 1, c], blk[:, r + 1, c + 1], x, y))
            d = dst[:, r, c] - t
            u = d - bias
            dd, uu = d * d, u * u
            sb = sb + ((dd[:, 0] + dd[:, 1]) + dd[:, 2])
            su = su + ((uu[:, 0] + uu[:, 1]) + uu[:, 2])
    return sb, su


def cheap_sums(blk, qb, dst, dbias, xw, yw, addend):
    """ssdApprox: unscaled (biased, bias-compensated) fp32 sums of the cheap path."""
    h = F32(addend)
    x, y = xw[:, None], yw[:, None]
    bias = (dbias + h) - bilerp_cheap(qb[:, 0, 0], qb[:, 0, 1], qb[:, 1, 0], qb[:, 1, 1], x, y)
    z = np.zeros(len(xw), F32)
    acc_b = [z, z]           # accB lanes (B, G): dx outer, dy inner
    acc_u = [z, z]
    acc_rb = [z, z, z]       # accBR lanes (R of dy = -1, 0) and accBs (R of dy = +1): one accumulator per row
    acc_ru = [z, z, z]
    for c in range(3):
        for r in range(3):
            a = bilerp_cheap(blk[:, r, c], blk[:, r, c + 1], blk[:, r + 1, c], blk[:, r + 1, c + 1], x, y)
            d = (dst[:, r, c] + h) - a
            u = d - bias
            for ch in range(2):
                acc_b[ch] = fma32(d[:, ch], d[:, ch], acc_b[ch])
                acc_u[ch] = fma32(u[:, ch], u[:, ch], acc_u[ch])
            acc_rb[r] = fma32(d[:, 2], d[:, 2], acc_rb[r])
            acc_ru[r] = fma32(u[:, 2], u[:, 2], acc_ru[r])
    sb = ((acc_b[0] + acc_b[1]) + (acc_rb[0] + acc_rb[1])) + acc_rb[2]
    su = ((acc_u[0] + acc_u[1]) + (acc_ru[0] + acc_ru[1])) + acc_ru[2]
    return sb, su


def slot_errors(case):
    """Per source: the worst |rB - sqrt(sB_exact)| over the sqrt.approx error, the worst rU - sqrt(sU_exact), and
    whether ul * factor <= sU_exact with the worst (largest) rU.  sB_exact / sU_exact are the exact path's fp32 sums."""
    kerr_b, kerr_u, factor, addend = kernel_constants()
    eb, eu = exact_sums(*case)
    cb, cu = cheap_sums(*case, addend)
    root_b = np.sqrt(eb.astype(np.float64))
    rb = np.sqrt(cb.astype(np.float64))
    err_b = np.maximum(np.abs(rb * (1 + SQRT_REL) - root_b), np.abs(rb * (1 - SQRT_REL) - root_b))
    ru_hi = np.nextafter((np.sqrt(cu.astype(np.float64)) * (1 + SQRT_REL)).astype(F32), F32(np.inf))
    err_u = ru_hi.astype(np.float64) - np.sqrt(eu.astype(np.float64))
    ul = np.maximum(ru_hi - F32(kerr_u), F32(0))
    ul = ul * ul
    ok_u = ul.astype(np.float64) * factor <= eu.astype(np.float64)
    return err_b, err_u, ok_u, eb, cb


# ---- FMA emulation check ----------------------------------------------------------------------------------------------
def _rn32_fraction(q):
    """Round a Fraction to the nearest fp32, ties to even (normal range)."""
    if q == 0:
        return 0.0
    sign = -1 if q < 0 else 1
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    scale = Fraction(2) ** (23 - e)
    m = q * scale
    fl = m.numerator // m.denominator
    rem = m - fl
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
        fl += 1
    return sign * float(Fraction(fl) / scale)


def test_fma_emulation_is_exact():
    rng = np.random.RandomState(0)
    n = 4000
    w = weights_from_positions(rng.uniform(1, 5000, n))
    a = rng.randint(0, 65536, n).astype(F32) + rng.randint(0, 2 ** 10, n).astype(F32) / F32(2 ** 10)
    b = (rng.uniform(-65535, 65535, n)).astype(F32)
    c = (rng.uniform(-1e5, 1e5, n)).astype(F32)
    # products landing on fp32 midpoints of the sum: c chosen so that a*b + c is a midpoint +- a small residue
    k = n // 2
    base = (a[:k].astype(np.float64) * b[:k].astype(np.float64))
    c[:k] = (np.round(base).astype(np.float64) * 0 - base.astype(F32).astype(np.float64)).astype(F32)
    got = fma32(w * 0 + a, b, c)
    for i in range(n):
        want = _rn32_fraction(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
        assert float(got[i]) == want, (i, a[i], b[i], c[i], got[i], want)
    # exact ties of the fp64 sum: 2^24 + 1 + tiny residue
    one = np.array([1.0], F32)
    big = np.array([16777216.0], F32)
    for res in (2.0 ** -30, -(2.0 ** -30)):
        av = np.array([1.0 + 2.0 ** -23], F32)
        bv = np.array([1.0 + 2.0 ** -23 * (1 if res > 0 else -1)], F32)
        want = _rn32_fraction(Fraction(float(av[0])) * Fraction(float(bv[0])) + Fraction(float(big[0])))
        assert float(fma32(av, bv, big)[0]) == want
    assert float(fma32(one, one, big)[0]) == 16777216.0  # 2^24 + 1: a tie, even


# ---- per-term claims ------------------------------------------------------------------------------------------------
def weight_grid():
    """fp32 weights from positions p on a dense grid, with exact half-integers and the fp32 values either side."""
    frac = np.concatenate([np.linspace(0, 1, 401), [0.5, 0.25, 0.75]])
    ps = []
    for k in (1.0, 2.0, 37.0, 1023.0, 65535.0, 1048575.0, 3999999.0):
        p = (k + frac).astype(F32)
        ps += [p, np.nextafter(p, F32(np.inf)), np.nextafter(p, F32(0))]
    p = np.concatenate(ps)
    p = p[(p >= 1.0) & (p < 4.0e6)]
    w = np.unique(weights_from_positions(p))
    assert np.all(np.modf(w.astype(np.float64) * 2 ** 24)[0] == 0), "weights are multiples of 2^-24"
    return w


def per_term(q, xw, yw, dst, addend):
    """Errors of one (sample, channel) term: q (N,4) texels, xw / yw / dst (N,)."""
    p00, p01, p10, p11 = (q[:, i] for i in range(4))
    b = bilerp_exact(p00, p01, p10, p11, xw, yw)
    a = bilerp_cheap(p00, p01, p10, p11, xw, yw)
    v = bilerp_real(p00, p01, p10, p11, xw, yw)
    t = np.floor(b)
    e_bilerp = np.abs(b.astype(LD) - v)
    e_lerp = np.abs(a.astype(LD) - v)
    e_mid = np.abs(t.astype(LD) - (a.astype(LD) - LD(0.5)))
    d_cheap = (dst + F32(addend)) - a
    e_term = np.abs(d_cheap.astype(np.float64) - (dst - t).astype(np.float64))
    return np.stack([e_bilerp.astype(np.float64), e_lerp.astype(np.float64), e_mid.astype(np.float64), e_term], 1)


def worst_per_term():
    _, _, _, addend = kernel_constants()
    rng = np.random.RandomState(7)
    w = weight_grid()
    quads = np.array(np.meshgrid(*[EXTREMES] * 4, indexing="ij")).reshape(4, -1).T.astype(F32)
    worst = np.zeros(4)
    best_cases = []
    # extreme texel quadruples x weight pairs x destinations {0, 65535}
    for rep in range(6):
        xw = w[rng.randint(0, len(w), len(quads))]
        yw = w[rng.randint(0, len(w), len(quads))]
        dst = np.where(rng.rand(len(quads)) < 0.5, F32(0), F32(65535))
        e = per_term(quads, xw, yw, dst, addend)
        worst = np.maximum(worst, e.max(0))
        best_cases.append((quads, xw, yw, dst, e[:, 2]))
    # random quadruples, half of them near full scale
    n = 400000
    q = rng.randint(0, 65536, (n, 4)).astype(F32)
    q[: n // 2] = (65535 - rng.randint(0, 64, (n // 2, 4))).astype(F32)
    xw = w[rng.randint(0, len(w), n)]
    yw = w[rng.randint(0, len(w), n)]
    dst = rng.randint(0, 65536, n).astype(F32)
    e = per_term(q, xw, yw, dst, addend)
    worst = np.maximum(worst, e.max(0))
    best_cases.append((q, xw, yw, dst, e[:, 2]))
    # coordinate search from the worst hits of the truncation-midpoint error
    qs, xs, ys, ds = (np.concatenate([c[i] for c in best_cases]) for i in range(4))
    score = np.concatenate([c[4] for c in best_cases])
    top = np.argsort(score)[-512:]
    q, xw, yw, dst = qs[top].copy(), xs[top].copy(), ys[top].copy(), ds[top].copy()
    cur = per_term(q, xw, yw, dst, addend)[:, 2]
    for it in range(300):
        q2, x2, y2 = q.copy(), xw.copy(), yw.copy()
        k = rng.randint(0, 6, len(q))
        sel = k < 4
        step = rng.choice([-3, -1, 1, 3], len(q)).astype(F32)
        q2[sel, k[sel]] = np.clip(q2[sel, k[sel]] + step[sel], 0, 65535)
        x2[k == 4] = np.nextafter(x2[k == 4], np.where(step[k == 4] > 0, F32(1), F32(0)).astype(F32))
        y2[k == 5] = np.nextafter(y2[k == 5], np.where(step[k == 5] > 0, F32(1), F32(0)).astype(F32))
        e = per_term(q2, x2, y2, dst, addend)
        better = e[:, 2] > cur
        q[better], xw[better], yw[better], cur[better] = q2[better], x2[better], y2[better], e[better, 2]
        worst = np.maximum(worst, e.max(0))
    return worst


def test_per_term_claims(capsys):
    worst = worst_per_term()
    claims = (CLAIM_BILERP, CLAIM_LERP, CLAIM_MID, CLAIM_TERM)
    names = ("|fl32(bilerp) - V|", "|a - V|", "|t - (a - 1/2)|", "|d' - d| per term")
    with capsys.disabled():
        for name, got, claim in zip(names, worst, claims):
            print("\n  per-term %-20s max %.6f   claim %.4f" % (name, got, claim), end="")
        print()
    for name, got, claim in zip(names, worst, claims):
        assert got <= claim, (name, got, claim)


def test_bias_term_claim():
    """The bias difference of the cheap path against the exact one (dBias + addend - lerp vs dBias - trunc(bilerp))."""
    _, _, _, addend = kernel_constants()
    rng = np.random.RandomState(11)
    w = weight_grid()
    n = 200000
    q = rng.randint(0, 65536, (n, 4)).astype(F32)
    q[: n // 4] = EXTREMES[rng.randint(0, len(EXTREMES), (n // 4, 4))]
    xw, yw = w[rng.randint(0, len(w), n)], w[rng.randint(0, len(w), n)]
    dbias = rng.randint(0, 65536, n).astype(F32)
    exact = dbias - np.floor(bilerp_exact(q[:, 0], q[:, 1], q[:, 2], q[:, 3], xw, yw))
    cheap = (dbias + F32(addend)) - bilerp_cheap(q[:, 0], q[:, 1], q[:, 2], q[:, 3], xw, yw)
    assert np.abs(cheap.astype(np.float64) - exact).max() <= CLAIM_TERM


# ---- per-source aggregate -------------------------------------------------------------------------------------------
def constant_cases(rng, n, contrast):
    """Constant source and destination patches: every term's midpoint error has the same sign.  contrast (n,) = dst -
    src level; the bias compensation is pushed the other way so that the unbiased differences are as large as possible."""
    w = weight_grid()
    src = np.where(contrast >= 0, 0, -contrast) + rng.randint(0, 2, n) * 0
    src = np.clip(src, 0, 65535).astype(F32)
    dstl = np.clip(src + contrast, 0, 65535).astype(F32)
    blk = np.broadcast_to(src[:, None, None, None], (n, 4, 4, 3)).astype(F32).copy()
    dst = np.broadcast_to(dstl[:, None, None, None], (n, 3, 3, 3)).astype(F32).copy()
    qlev = np.where(contrast >= 0, 65535, 0).astype(F32)
    qb = np.broadcast_to(qlev[:, None, None, None], (n, 2, 2, 3)).astype(F32).copy()
    dbias = np.broadcast_to((65535 - qlev)[:, None], (n, 3)).astype(F32).copy()
    xw, yw = w[rng.randint(0, len(w), n)], w[rng.randint(0, len(w), n)]
    return [blk, qb, dst, dbias, xw, yw]


def search_cases(rng, n, iters):
    """Hill climb on |rB - sqrt(sB_exact)| from high-contrast near-constant patches: mutate texels, destination and
    weights, keep what increases the error."""
    kerr_b, _, _, _ = kernel_constants()
    w = weight_grid()
    case = constant_cases(rng, n, np.where(rng.rand(n) < 0.5, 65535, -65535) - rng.randint(0, 4, n) * np.sign(rng.rand(n) - 0.5))
    case[0] = np.clip(case[0] + rng.randint(-40, 41, case[0].shape), 0, 65535).astype(F32)
    cur = slot_errors(case)[0]
    for it in range(iters):
        c2 = [a.copy() for a in case]
        kind = rng.randint(0, 4, n)
        i = np.arange(n)
        r, c, ch = rng.randint(0, 4, n), rng.randint(0, 4, n), rng.randint(0, 3, n)
        step = rng.choice([-7, -2, -1, 1, 2, 7], n)
        m = kind == 0
        c2[0][i[m], r[m], c[m], ch[m]] = np.clip(c2[0][i[m], r[m], c[m], ch[m]] + step[m], 0, 65535)
        m = kind == 1
        c2[2][i[m], r[m] % 3, c[m] % 3, ch[m]] = np.clip(c2[2][i[m], r[m] % 3, c[m] % 3, ch[m]] + step[m], 0, 65535)
        m = kind == 2
        c2[4][m] = w[rng.randint(0, len(w), int(m.sum()))]
        m = kind == 3
        c2[5][m] = w[rng.randint(0, len(w), int(m.sum()))]
        e = slot_errors(c2)[0]
        better = e > cur
        for a, b in zip(case, c2):
            a[better] = b[better]
        cur = np.where(better, e, cur)
    return case


def test_per_source_aggregate(capsys):
    kerr_b, kerr_u, factor, _ = kernel_constants()
    rng = np.random.RandomState(3)
    n = 20000
    contrast = np.concatenate([np.linspace(-65535, 65535, n // 2).round(), rng.randint(-65535, 65536, n // 2)])
    cases = [constant_cases(rng, n, contrast), search_cases(rng, 2048, 120)]
    worst_b, worst_u, all_ok = 0.0, -np.inf, True
    for case in cases:
        err_b, err_u, ok_u, eb, cb = slot_errors(case)
        worst_b = max(worst_b, float(err_b.max()))
        worst_u = max(worst_u, float(err_u.max()))
        all_ok &= bool(ok_u.all())
    with capsys.disabled():
        print("\n  aggregate |rB - sqrt(sB_exact)| max %.4f   kErrB %.4f   margin %.4f" % (worst_b, kerr_b, kerr_b - worst_b))
        print("  aggregate rU - sqrt(sU_exact)   max %.4f   kErrU %.4f   margin %.4f" % (worst_u, kerr_u, kerr_u - worst_u))
    assert worst_b <= kerr_b
    assert all_ok, "(max(rU - kErrU, 0))^2 * factor exceeds the exact unbiased sum"


# ---- lowerBoundOfCost ----------------------------------------------------------------------------------------------
def kernel_bound(rb, lb, keep, conf):
    """lowerBoundOfCost restated in fp32 on the slots (rb[i], lb[i]) in slot order."""
    kerr_b, _, factor, _ = kernel_constants()
    two_err = F32(2) * F32(kerr_b)
    n = len(rb)
    r1 = r2 = r3 = F32(-1)
    l1 = l2 = t1 = t2 = rest_r = rest_t = F32(0)
    for i in range(n):
        a, b = F32(rb[i]), F32(lb[i])
        rest_r = F32(rest_r + (l2 if a > r2 else b))
        rest_t = F32(rest_t + min(b, t2))
        if a > r1:
            r3, r2, l2, r1, l1 = r2, r1, l1, a, b
        elif a > r2:
            r3, r2, l2 = r2, a, b
        elif a > r3:
            r3 = a
        if b > t1:
            t2, t1 = t1, b
        elif b > t2:
            t2 = b
    if n == 1:
        kept = l1
    elif n == 2:
        kept = l2 if F32(r1 - r2) > two_err else t2
    else:
        kept = rest_r if F32(r2 - r3) > two_err else rest_t
    scale = F32(1) / (F32(65535) * F32(65535))
    k = F32(keep)
    return F32(F32(F32(F32(F32(kept * scale) / k) * F32(F32(1) / k)) / F32(conf)) * F32(factor))


def pair_less(x, y):
    return x[0] < y[0] or (not (y[0] < x[0]) and x[1] < y[1])


def reference_cost(sb, su, keep, conf):
    """What the exact path returns for these fp32 sums: the `keep` smallest (biased, unbiased) scaled pairs in pairLess
    order, their unbiased mean, / keep / conf.  Exact real arithmetic on the fp32 scaled pairs, then the smallest value
    an fp32 evaluation of it can round to (relative 2^-24 per operation, keep + 4 operations)."""
    scale = F32(1) / (F32(65535) * F32(65535))
    pairs = [(F32(b * scale), F32(u * scale)) for b, u in zip(sb, su)]
    order = sorted(range(len(pairs)), key=functools.cmp_to_key(lambda i, j: -1 if pair_less(pairs[i], pairs[j]) else (1 if pair_less(pairs[j], pairs[i]) else 0)))
    kept = sum(Fraction(float(pairs[i][1])) for i in order[:keep])
    exact = kept / keep / keep / Fraction(float(conf))
    return float(exact) * (1 - (keep + 4) * 2.0 ** -24)


def fuzz_slots(rng, n, kerr_b):
    """Exact fp32 sums for n sources whose roots sit at and around 2 kErrB separations, slot roots perturbed by up to
    kErrB (the aggregate bound) and lower bounds <= the exact unbiased sums, with unbiased sums of very different sizes."""
    base = rng.uniform(0, 3.4e5)
    gaps = rng.choice([0.0, 1e-3, 2 * kerr_b - 1e-3, 2 * kerr_b, 2 * kerr_b + 1e-3, 4 * kerr_b, 50.0, 5e4], n)
    roots = np.clip(base + np.cumsum(gaps) * rng.choice([-1, 1]), 0, None)
    rng.shuffle(roots)
    sb = (roots.astype(np.float64) ** 2).astype(F32)
    mag = rng.choice([0.0, 3e3, 1e6, 1e9, 4.6e11], n)
    su = (mag * rng.uniform(0.5, 1.0, n)).astype(F32)
    true_root = np.sqrt(sb.astype(np.float64))
    e = rng.choice([-kerr_b, kerr_b, 0.0], n) * rng.choice([1.0, 1.0, rng.uniform()], n)
    rb = (true_root + e).astype(F32)
    over = np.abs(rb.astype(np.float64) - true_root) > kerr_b
    rb[over] = np.nextafter(rb[over], true_root[over].astype(F32))
    rb = np.maximum(rb, F32(0))
    lb = np.where(rng.rand(n) < 0.7, su, (su * rng.uniform(0, 1, n)).astype(F32)).astype(F32)
    return sb, su, rb, lb


@pytest.mark.parametrize("n", list(range(1, 11)))
def test_lower_bound_of_cost_branches(n):
    kerr_b, _, _, _ = kernel_constants()
    rng = np.random.RandomState(100 + n)
    keep = max(1, n - 2)
    bad = []
    for trial in range(1500):
        sb, su, rb, lb = fuzz_slots(rng, n, kerr_b)
        conf = float(rng.choice([1.0, 1.0 / 12.0 / 65025.0, 3.7e-3]))
        got = float(kernel_bound(rb, lb, keep, conf))
        want = reference_cost(sb, su, keep, conf)
        if got > want:
            bad.append((got, want, rb.tolist(), lb.tolist(), sb.tolist(), su.tolist()))
    assert not bad, "%d of 1500 bounds exceed the exact cost, e.g. %s" % (len(bad), bad[0])
