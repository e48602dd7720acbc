"""Exact CPU model of the filtered sweep's two-row lower bound (derp_cost.cuh: ssdLowerRows, sqrtApprox, KeptBound)
against the exact path's arithmetic (evalCost's exact branch, computeSSD in oracle/derp_oracle.cpp).

The bound pass forms, per source, a lower bound of the bias-compensated sum from the 18 terms of the sample rows dy = 0
and dy = +1 only, and per pixel the sum of the keep = max(1, n - 2) smallest per-source bounds.  Its proof
(derp_cost.cuh above kErrURows, DESIGN.md §4): the 18 terms are a subset of the 27 non-negative terms of the exact sum;
each cheap term is within 0.56 of the exact one (the per-term claims that test_lower_bound_model.py checks; the samples
are formed with the same x-lerp / y-lerp / two-subtraction arithmetic); so the l2 error of the two rows is at most
2 * 0.56 * sqrt(18) < kErrURows, and the rest (fp32 sums, sqrt.approx, scale, divisions) is relative and covered by the
final factor 1 - 2^-16.  This file re-computes both paths bit for bit in numpy (FMA emulated exactly, sqrt.approx at
2^-22 in either direction), with per-sample weights formed from positions as evalCost forms them (P -1, P, P +1 in
fp32), on constant patches of every contrast up to 65535 and on hill-climbed patches, and checks the pixel bound
against the reference's robust mean on random slot sets.  kErrURows, the final factor and the +0.5 addend are read from
the kernel sources."""
import functools
import os
import re

import numpy as np
import pytest

from tests.test_lower_bound_model import (CSRC, F32, SQRT_REL, bilerp_cheap, bilerp_exact, fma32, kernel_constants,
                                          reference_cost)


@functools.lru_cache(maxsize=1)
def row_constants():
    with open(os.path.join(CSRC, "derp_cost.cuh")) as f:
        cost = f.read()
    kerr = float(re.search(r"constexpr float kErrURows = ([0-9.eE+-]+)f;", cost).group(1))
    kept = cost[cost.index("struct KeptBound"):]
    factor = float(re.search(r"/ conf \* ([0-9.eE+-]+)f;", kept).group(1))
    _, _, _, addend = kernel_constants()  # the literal sweepLowerKernel passes to loadDstTile and loadPixelState
    return kerr, factor, addend


def sample_weights(pos):
    """(xw or yw) of the samples d = -1, 0, +1 around positions pos (N,): P + d in fp32, then p - round(p) + 0.5."""
    p = np.asarray(pos, F32)
    out = []
    for d in (-1, 0, 1):
        q = (p + F32(d)).astype(F32)
        t = np.floor(q.astype(np.float64) + 0.5).astype(F32)
        out.append(((q - t) + F32(0.5)).astype(F32))
    return np.stack(out, 1)


def random_positions(rng, n):
    base = rng.choice([2.0, 37.0, 1023.0, 65535.0, 1048575.0, 3999990.0], n)
    frac = np.where(rng.rand(n) < 0.3, rng.choice([0.0, 0.25, 0.5, 0.75], n), rng.rand(n))
    p = (base + frac).astype(F32)
    nudge = rng.randint(-1, 2, n)
    p = np.where(nudge > 0, np.nextafter(p, F32(np.inf)), np.where(nudge < 0, np.nextafter(p, F32(0)), p))
    return p.astype(F32)


# ---- one source ---------------------------------------------------------------------------------------------------
def exact_sum_u(blk, qb, dst, dbias, xw, yw):
    """Exact path's unscaled unbiased fp32 sum over all 27 terms, and the exact (real) sum of the 18 terms of the rows
    dy = 0 and dy = +1.
    blk (N,4,4,3), qb (N,2,2,3), dst (N,3,3,3), dbias (N,3), xw / yw (N,3) per sample column / row."""
    cx, cy = xw[:, 1:2], yw[:, 1:2]
    bias = dbias - np.floor(bilerp_exact(qb[:, 0, 0], qb[:, 0, 1], qb[:, 1, 0], qb[:, 1, 1], cx, cy))
    su = np.zeros(len(xw), F32)
    row = np.zeros(len(xw), np.float64)
    for c in range(3):      # dx outer
        for r in range(3):  # dy inner
            x, y = xw[:, c:c + 1], yw[:, r:r + 1]
            t = np.floor(bilerp_exact(blk[:, r, c], blk[:, r, c + 1], blk[:, r + 1, c], blk[:, r + 1, c + 1], x, y))
            u = (dst[:, r, c] - t) - bias
            uu = u * u
            su = su + ((uu[:, 0] + uu[:, 1]) + uu[:, 2])
            if r >= 1:
                row += (u.astype(np.float64) ** 2).sum(1)  # integers: exact in fp64
    return su, row


def cheap_row_u(blk, qb, dst, dbias, xw, yw, addend):
    """ssdLowerRows: the unscaled bias-compensated fp32 sum of the rows dy = 0 and dy = +1, in the kernel's lanes (B, G)
    and R and its order (per column: row dy = 0, then row dy = +1)."""
    h = F32(addend)
    cx, cy = xw[:, 1:2], yw[:, 1:2]
    bias = (dbias + h) - bilerp_cheap(qb[:, 0, 0], qb[:, 0, 1], qb[:, 1, 0], qb[:, 1, 1], cx, cy)
    z = np.zeros(len(xw), F32)
    acc = [z, z, z]  # acc lanes (B, G), accR
    for c in range(3):
        for r in (1, 2):
            s = bilerp_cheap(blk[:, r, c], blk[:, r, c + 1], blk[:, r + 1, c], blk[:, r + 1, c + 1], xw[:, c:c + 1],
                             yw[:, r:r + 1])
            u = ((dst[:, r, c] + h) - s) - bias
            for ch in range(3):
                acc[ch] = fma32(u[:, ch], u[:, ch], acc[ch])
    return (acc[0] + acc[1]) + acc[2]


def source_errors(case):
    """Per source: the worst rU - sqrt(exact two-row sum) over the sqrt.approx error, and whether the slot's lower bound
    ul = max(rU - kErrURows, 0)^2, times the final factor, stays <= the exact path's full unbiased sum."""
    kerr, factor, addend = row_constants()
    su, row = exact_sum_u(*case)
    cu = cheap_row_u(*case, addend)
    ru_hi = np.nextafter((np.sqrt(cu.astype(np.float64)) * (1 + SQRT_REL)).astype(F32), F32(np.inf))
    err = ru_hi.astype(np.float64) - np.sqrt(row)
    ul = np.maximum(ru_hi - F32(kerr), F32(0))
    ul = ul * ul
    ok = ul.astype(np.float64) * factor <= su.astype(np.float64)
    return err, ok


def constant_cases(rng, n, contrast):
    """Constant source and destination patches (every term's midpoint error has the same sign), bias pushed the other
    way so that the unbiased differences are as large as possible.  contrast (n,) = dst - src level."""
    src = np.clip(np.where(contrast >= 0, 0, -contrast), 0, 65535).astype(F32)
    dstl = np.clip(src + contrast, 0, 65535).astype(F32)
    blk = np.broadcast_to(src[:, None, None, None], (n, 4, 4, 3)).astype(F32).copy()
    dst = np.broadcast_to(dstl[:, None, None, None], (n, 3, 3, 3)).astype(F32).copy()
    qlev = np.where(contrast >= 0, 65535, 0).astype(F32)
    qb = np.broadcast_to(qlev[:, None, None, None], (n, 2, 2, 3)).astype(F32).copy()
    dbias = np.broadcast_to((65535 - qlev)[:, None], (n, 3)).astype(F32).copy()
    xw, yw = sample_weights(random_positions(rng, n)), sample_weights(random_positions(rng, n))
    return [blk, qb, dst, dbias, xw, yw]


def search_cases(rng, n, iters):
    """Hill climb on rU - sqrt(exact two-row sum) from high-contrast near-constant patches: mutate the texels of rows
    1..3, the destination rows dy = 0 and +1, the bias texels and the positions; keep what increases the error."""
    contrast = np.where(rng.rand(n) < 0.5, 65535, -65535) - rng.randint(0, 4, n) * np.sign(rng.rand(n) - 0.5)
    case = constant_cases(rng, n, contrast)
    case[0] = np.clip(case[0] + rng.randint(-40, 41, case[0].shape), 0, 65535).astype(F32)
    cur = source_errors(case)[0]
    i = np.arange(n)
    for _ in range(iters):
        c2 = [a.copy() for a in case]
        kind = rng.randint(0, 5, n)
        r, c, ch = rng.randint(1, 4, n), rng.randint(0, 4, n), rng.randint(0, 3, n)
        step = rng.choice([-7, -2, -1, 1, 2, 7], n)
        m = kind == 0
        c2[0][i[m], r[m], c[m], ch[m]] = np.clip(c2[0][i[m], r[m], c[m], ch[m]] + step[m], 0, 65535)
        m = kind == 1
        rd = 1 + (r[m] % 2)
        c2[2][i[m], rd, c[m] % 3, ch[m]] = np.clip(c2[2][i[m], rd, c[m] % 3, ch[m]] + step[m], 0, 65535)
        m = kind == 2
        c2[1][i[m], r[m] % 2, c[m] % 2, ch[m]] = np.clip(c2[1][i[m], r[m] % 2, c[m] % 2, ch[m]] + step[m], 0, 65535)
        m = kind == 3
        c2[4][m] = sample_weights(random_positions(rng, int(m.sum())))
        m = kind == 4
        c2[5][m] = sample_weights(random_positions(rng, int(m.sum())))
        e = source_errors(c2)[0]
        better = e > cur
        for a, b in zip(case, c2):
            a[better] = b[better]
        cur = np.where(better, e, cur)
    return case


def random_cases(rng, n):
    """Unstructured patches: random texels, destination and bias, half of them near full scale."""
    blk = rng.randint(0, 65536, (n, 4, 4, 3)).astype(F32)
    blk[: n // 2] = (65535 - rng.randint(0, 64, (n // 2, 4, 4, 3))).astype(F32)
    qb = rng.randint(0, 65536, (n, 2, 2, 3)).astype(F32)
    dst = rng.randint(0, 65536, (n, 3, 3, 3)).astype(F32)
    dbias = rng.randint(0, 65536, (n, 3)).astype(F32)
    return [blk, qb, dst, dbias, sample_weights(random_positions(rng, n)), sample_weights(random_positions(rng, n))]


def test_sample_weights_follow_the_kernel():
    """The centre sample's weight is p - round(p) + 0.5 (roundf rounds halves up).  The side samples' weights can
    differ from it where the fp32 addition P + 1 crosses a power of two and rounds, which is why the model carries one
    weight per sample column and row."""
    p = np.array([2.5, 37.25, 1048575.75, 3999990.5], F32)
    w = sample_weights(p)
    assert np.array_equal(w[:, 1], np.array([0.0, 0.75, 0.25, 0.0], F32))
    w = sample_weights(random_positions(np.random.RandomState(1), 100000))
    assert (w[:, 2] != w[:, 1]).any()


def test_row_bound_per_source(capsys):
    kerr, _, _ = row_constants()
    rng = np.random.RandomState(5)
    n = 20000
    contrast = np.concatenate([np.linspace(-65535, 65535, n // 2).round(), rng.randint(-65535, 65536, n // 2)])
    worst, all_ok = -np.inf, True
    for case in (constant_cases(rng, n, contrast), random_cases(rng, n), search_cases(rng, 2048, 150)):
        err, ok = source_errors(case)
        worst = max(worst, float(err.max()))
        all_ok &= bool(ok.all())
    with capsys.disabled():
        print("\n  rows dy = 0, +1: rU - sqrt(exact sum)   max %.4f   kErrURows %.4f   margin %.4f" % (worst, kerr, kerr - worst))
    assert worst <= kerr
    assert all_ok, "(max(rU - kErrURows, 0))^2 * factor exceeds the exact unbiased sum"


# ---- KeptBound -------------------------------------------------------------------------------------------------------
def kept_bound(lb, keep, conf):
    """KeptBound restated in fp32 on the per-source lower bounds in slot order."""
    _, factor, _ = row_constants()
    t1 = t2 = rest = F32(0)
    for b in lb:
        b = F32(b)
        rest = F32(rest + min(b, t2))
        if b > t1:
            t2, t1 = t1, b
        elif b > t2:
            t2 = b
    n = len(lb)
    kept = t1 if n == 1 else (t2 if n == 2 else rest)
    scale = F32(1) / (F32(65535) * F32(65535))
    k = F32(keep)
    return F32(F32(F32(F32(F32(kept * scale) / k) * F32(F32(1) / k)) / F32(conf)) * F32(factor))


@pytest.mark.parametrize("n", list(range(1, 16)) + [40])
def test_kept_bound_never_exceeds_the_cost(n):
    """Random exact sums (biased sums independent of the unbiased ones, so that every kept set occurs) and per-source
    lower bounds <= the unbiased sums; the pixel bound must not exceed what the exact path returns."""
    rng = np.random.RandomState(200 + n)
    keep = max(1, n - 2)
    bad = []
    for trial in range(600 if n < 40 else 200):
        sb = (rng.choice([0.0, 1e3, 1e6, 1e9, 4.6e11], n) * rng.uniform(0.5, 1.0, n)).astype(F32)
        su = (rng.choice([0.0, 3e3, 1e6, 1e9, 4.6e11], n) * rng.uniform(0.5, 1.0, n)).astype(F32)
        lb = np.where(rng.rand(n) < 0.7, su, (su * rng.uniform(0, 1, n)).astype(F32)).astype(F32)
        conf = float(rng.choice([1.0, 1.0 / 12.0 / 65025.0, 3.7e-3]))
        got = float(kept_bound(lb, keep, conf))
        want = reference_cost(sb, su, keep, conf)
        if got > want:
            bad.append((got, want, lb.tolist(), sb.tolist(), su.tolist()))
    assert not bad, "%d bounds exceed the exact cost, e.g. %s" % (len(bad), bad[0])


def test_kept_bound_sums_the_keep_smallest():
    rng = np.random.RandomState(9)
    for n in list(range(1, 16)) + [40, 63]:
        lb = rng.randint(0, 1000, n).astype(F32)
        keep = max(1, n - 2)
        want = np.sort(lb)[:keep].sum() / (F32(65535) * F32(65535)) / keep / keep
        got = float(kept_bound(lb, keep, 1.0))
        assert abs(got - want) <= 4e-5 * want + 1e-30, (n, got, want)  # the factor 1 - 2^-16 and fp32 roundings
