"""CPU model of sweep form 5's half-precision pass 1 (FastHitterKH in csrc/tpt_fast.cu, operands from build_half_pairs
in csrc/tpt_scene_pack.h): exact emulation of every binary16 operation, the per-sphere constants with their error bound,
and the FP32 candidate test of forms 2 and 4 it must contain. Used by tools/half_sweep_study.py and the tests."""
from __future__ import annotations

import numpy as np

U = 2.0 ** -11                  # unit roundoff of binary16
ORIGIN_BOUND = 16.0             # kHalfOriginBound
_LIMIT = 30000.0


def round_half(x, mode: int = 0) -> np.ndarray:
    """float64 -> nearest binary16 value (mode 0, ties to even), or rounded up (+1) / down (-1); as float64."""
    x = np.asarray(x, np.float64)
    ax = np.abs(x)
    e = np.floor(np.log2(np.where(ax > 0, ax, 1.0)))
    # log2 can be off by one next to powers of two: fix the exponent so that ax is in [2^e, 2^(e+1))
    e = np.where(np.ldexp(1.0, e.astype(int)) > ax, e - 1, e)
    e = np.where(np.ldexp(1.0, (e + 1).astype(int)) <= ax, e + 1, e)
    q = np.ldexp(1.0, (np.maximum(e, -14) - 10).astype(int))
    k = x / q
    k = np.ceil(k) if mode > 0 else np.floor(k) if mode < 0 else np.rint(k)
    return np.copysign(k * q, x)


def hfma(a, b, c) -> np.ndarray:
    """One binary16 FMA (a*b + c rounded once to nearest even) of binary16 inputs, emulated exactly: the product is exact
    in float64 and the sum's rounding error is recovered with TwoSum; when float64 rounded the sum onto a binary16
    tie, the error's sign decides the direction."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)
    c = np.asarray(c, np.float64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    r = round_half(s)
    tie = np.abs(s - r) == np.abs(round_half(s, 1) - round_half(s, -1)) / 2
    nudge = np.where(err > 0, np.nextafter(s, np.inf), np.nextafter(s, -np.inf))
    return np.where(tie & (err != 0), round_half(nudge), r)


def hadd(a, b) -> np.ndarray:
    return hfma(a, 1.0, b)


def sphere_constants(centers, r2):
    """(S, R'^2, R'', E, gate) per sphere: R'^2, E and the gate as build_half_pairs computes them (before rounding to
    binary16); R'' is the widened radius of the "wholly behind" test the study compares (not in the kernel)."""
    c = np.asarray(centers, np.float32).astype(np.float64)
    r2 = np.asarray(r2, np.float32).astype(np.float64)
    S = np.sqrt((c * c).sum(axis=1))
    Om = ORIGIN_BOUND
    E = U * (5.01 * S + 4.01 * Om) + 2.0 ** -20
    Rw = np.sqrt(r2 + (S * S + Om * Om + r2) * 2.0 ** -15)
    Rp2 = (Rw + 1.4143 * E) ** 2 / (1.0 - U) * (1.0 + 2.0 ** -20)
    Rb = (Rw * (1.0 + 2.0 ** -20) + (S + Om) * 2.0 ** -21 + U * 5.02 * (S + Om) + 2.0 ** -20) / (1.0 - 4.02 * U)
    ok = ((S + Om + 1.0) ** 2 <= _LIMIT) & (Rp2 <= _LIMIT)
    return S, Rp2, Rb, E, ok


def scene_ok(centers, r2) -> bool:
    """build_half_pairs' gate: at most 64 padded spheres and every sphere's intermediates well inside binary16."""
    n = len(r2)
    return (n + 3) // 4 * 4 <= 64 and bool(sphere_constants(centers, r2)[4].all())


def ray_basis(o, d):
    """The kernel's per-ray FP32 constants: the basis (u, v) around d (sample_light_cone's), o.u, o.v, o.d. The kernel
    contracts some of these products into FMAs; the bound does not depend on which."""
    o = np.asarray(o, np.float32)
    d = np.asarray(d, np.float32)
    one = np.float32(1)
    sgn = np.copysign(one, d[:, 2])
    a = (-one / (sgn + d[:, 2])).astype(np.float32)
    b = d[:, 0] * d[:, 1] * a
    u = np.stack([one + sgn * d[:, 0] * d[:, 0] * a, sgn * b, -sgn * d[:, 0]], axis=1).astype(np.float32)
    v = np.stack([b, sgn + d[:, 1] * d[:, 1] * a, -d[:, 1]], axis=1).astype(np.float32)
    dot = lambda x, y: (x[:, 0] * y[:, 0] + x[:, 1] * y[:, 1] + x[:, 2] * y[:, 2]).astype(np.float32)
    return u, v, dot(o, u), dot(o, v), dot(o, d)


def in_bound(o, d) -> np.ndarray:
    """Rays the half pass may take (the kernel's per-lane test before its warp vote)."""
    o = np.asarray(o, np.float32)
    d = np.asarray(d, np.float32)
    oo = (o * o).sum(axis=1, dtype=np.float32)
    dd = (d * d).sum(axis=1, dtype=np.float32)
    return (oo <= np.float32(ORIGIN_BOUND ** 2)) & (np.abs(dd - np.float32(1)) <= np.float32(2.0 ** -18))


def half_pass(centers, r2, o, d, behind: bool = False):
    """Emulated pass 1 of form 5: (candidate [rays, spheres] bool, xu, xv, q) with every binary16 rounding the kernel
    does. behind=True adds the "wholly behind the origin" test s.d - o.d + R'' >= 0 (study only)."""
    c = np.asarray(centers, np.float32).astype(np.float64)
    _, Rp2, Rb, _, _ = sphere_constants(centers, r2)
    X, Y, Z = (round_half(c[:, k])[None, :] for k in range(3))
    NR2 = round_half(-Rp2, -1)[None, :]
    NRB = round_half(-Rb, -1)[None, :]
    u, v, ou, ov, od = ray_basis(o, d)
    h = lambda x: round_half(np.asarray(x, np.float64))[:, None]
    d = np.asarray(d, np.float32)
    xu = hfma(X, h(u[:, 0]), hfma(Y, h(u[:, 1]), hfma(Z, h(u[:, 2]), h(-ou))))
    xv = hfma(X, h(v[:, 0]), hfma(Y, h(v[:, 1]), hfma(Z, h(v[:, 2]), h(-ov))))
    q = hfma(xu, xu, hfma(xv, xv, NR2))
    cand = np.signbit(q)
    if behind:
        nw = hfma(X, h(-d[:, 0]), hfma(Y, h(-d[:, 1]), hfma(Z, h(-d[:, 2]), hadd(NRB, h(od)))))
        cand &= np.signbit(nw)
    return cand, xu, xv, q


def exact_xuv(centers, o, d):
    """xu, xv in float64 from the FP32 basis: what the half chain approximates."""
    c = np.asarray(centers, np.float32).astype(np.float64)
    u, v, _, _, _ = ray_basis(o, d)
    x = c[None, :, :] - np.asarray(o, np.float32).astype(np.float64)[:, None, :]
    return (x * u.astype(np.float64)[:, None, :]).sum(axis=2), (x * v.astype(np.float64)[:, None, :]).sum(axis=2)


def fp32_candidates(centers, r2, o, d):
    """Form 4's pass 1 (the expanded form in FP32, FMA-contracted like the kernel): its candidate set [rays, spheres],
    which contains every sphere its pass 2 accepts."""
    f = np.float32
    c = np.asarray(centers, f)
    r2 = np.asarray(r2, f)
    K = ((c.astype(np.float64) ** 2).sum(axis=1) - r2.astype(np.float64)).astype(f)
    o = np.asarray(o, f)
    d = np.asarray(d, f)

    def fma(a, b, cc):
        return (a.astype(np.float64) * b.astype(np.float64) + cc.astype(np.float64)).astype(f)
    nod = -fma(o[:, 0], d[:, 0], fma(o[:, 1], d[:, 1], o[:, 2] * d[:, 2]))
    oo = fma(o[:, 0], o[:, 0], fma(o[:, 1], o[:, 1], o[:, 2] * o[:, 2]))
    C = lambda k: c[None, :, k]
    nb = fma(C(0), d[:, None, 0], fma(C(1), d[:, None, 1], fma(C(2), d[:, None, 2], np.broadcast_to(nod[:, None], (len(o), len(c))))))
    negc = fma(C(0), 2 * o[:, None, 0], fma(C(1), 2 * o[:, None, 1], fma(C(2), 2 * o[:, None, 2], (-K[None, :] - oo[:, None]).astype(f))))
    discr = fma(nb, nb, negc)
    rej = np.signbit(discr) | (np.signbit(nb) & np.signbit(negc))
    return ~rej


def exact_accepts(centers, r2, o, d, tmin: float = 0.001):
    """Spheres a ray hits at some t > tmin, in float64: the set the candidates must contain (up to FP32 rounding)."""
    c = np.asarray(centers, np.float32).astype(np.float64)
    r2 = np.asarray(r2, np.float32).astype(np.float64)
    o = np.asarray(o, np.float32).astype(np.float64)
    d = np.asarray(d, np.float32).astype(np.float64)
    x = c[None] - o[:, None]
    nb = (x * d[:, None]).sum(axis=2)
    discr = nb * nb - (x * x).sum(axis=2) + r2[None]
    sq = np.sqrt(np.maximum(discr, 0))
    return (discr > 0) & (nb + sq > tmin)
