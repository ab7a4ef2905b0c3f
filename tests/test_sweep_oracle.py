"""A float64 nearest-hit oracle for the fast kernels' sphere sweeps (tpt_fast.cu: SerialHitter<false>, FastHitterK,
FastHitterK2, FastHitterK2C), checked here against exact rational arithmetic, plus the ray and scene generators the GPU
file (test_gpu_sweep_oracle.py) feeds to tpt_debug_hit.

Semantics (every fast form): for a ray {o, d} and a sphere {s, R = fl32(r*r)} (tpt_scene_pack.h stores r^2 rounded to
float32) let nb = (s - o).d, c = |s - o|^2 - R, D = nb^2 - c. If D > 0, t = nb - sqrt(D), and if t <= tMin then
t = nb + sqrt(D); the sphere is accepted when tMin < t < best. tMin = 1e-3, tMax = 1e7, and on equal t the lowest id wins
(strict '<' in ascending id order). Only spheres < count are real; the padded ones are left out of the oracle.

Error bounds (u = 2^-24). Every fused multiply-add rounds once: a chain p_k = fl(t_k + p_{k-1}) of exact products t_k
(two float32 factors) has |computed p_k - p_k| <= e_k with e_k = e_{k-1} + u (|p_k| + e_{k-1}), since the computed
partial sum is at most |p_k| + e_{k-1} in magnitude and its rounding adds at most u times that (running error analysis,
Higham ch. 3, on the partial sums the float32 form actually forms, not on a blanket gamma_n (|s| + |o|)^2). Per
(ray, sphere), with the oracle's nb, c the exact values of the float32 inputs:

  reference form (sphere_discr<false>; forms 0 and 3's pass 2): co = fl32(s - o) is formed first; the oracle computes it
      exactly (an IEEE subtraction), so its rounding enters as the known |nb(co) - nb| and |c(co) - c|. Then
      nb = fma(co_x, d_x, fma(co_y, d_y, co_z d_z)) and -c = fma(-co_x, co_x, fma(-co_y, co_y, fma(-co_z, co_z, R)))
      are two chains with the bound above.
  expanded form (FastHitterK / FastHitterK2; forms 1 and 2): nod = -fma(o_x, d_x, fma(o_y, d_y, o_z d_z)),
      nb = fma(s_x, d_x, fma(s_y, d_y, fma(s_z, d_z, nod))), oo = the same chain for o.o, K = fl32(|s|^2 - R) from
      double (its rounding |K - (|s|^2 - R)| is known exactly), c = fma(-2 s_x o_x ... fl(K + oo)); the errors of nod,
      oo and K enter their chains as the starting e_0.
  On a scene that passes the expanded-form gate (forms 0, 1 and 2 run there) the oracle uses the larger of the two bounds
  for every form. On a scene that fails it only forms 0 and 3 run, and both decide every hit in the reference form
  (form 3's pass 1 only ever adds candidates: its margin is what covers the expanded form's error, and form 3 == form 0
  on every ray is what tests it), so the reference bound alone applies there. Either way the oracle adds 2^-46 of the
  magnitudes for its own float64 rounding. The blanket 22u(|s| + |o|)^2 of the kernel comments is NOT used: the
  stress scene's ground sphere (|s| = 1000) would make every ray that leaves it undecidable, while the partial sums
  see that K = |s|^2 - R ~ 0 and s.o ~ 0 there.

  The discriminant D = fma(nb, nb, -c) rounds once, which keeps its sign. Over the box nb +- E_nb, c +- E_c it lies in
  [D_lo, D_hi]. The kernels take sqrt.approx.ftz.f32 (one MUFU.SQRT on sm_90). The PTX ISA documents the approximate
  square-root family of the MUFU unit to about 2^-23 relative (rsqrt.approx.f32: 2^-22.9); the oracle allows
  rho = 2^-22 + u for it and the rounding of D (the GPU tests check every returned t against the resulting bound, so a
  wrong assumption here fails them), so sqrt(D) in [sqrt(D_lo)(1-rho),
  sqrt(D_hi)(1+rho)], and one more u |t| for the subtraction nb -+ sqrt. That gives enclosures [t-_lo, t-_hi], [t+_lo, t+_hi]
  of the computed roots anywhere in the box. Per sphere the outcome is then decided when one of these holds, else it is
  ambiguous:
      reject          D_hi <= 0, or t+_hi < tMin (both roots at or below tMin)
      accept, t-      D_lo > FLT_MIN (no flush to zero) and t-_lo > tMin
      accept, t+      D_lo > FLT_MIN, t-_hi < tMin and t+_lo > tMin
  A ray is WELL-CONDITIONED when no sphere is ambiguous and the winner's t_hi is below every other accepted sphere's t_lo
  (spheres bit-identical to the winner excepted: they produce the same t bits and lose the tie). For such a ray every
  form must return the oracle's id, with a t inside [t_lo, t_hi].
"""
from fractions import Fraction
import decimal

import numpy as np
import pytest

from test_oracle import golden_scene
from test_gpu_fast import surface_rays

U = 2.0 ** -24
T_MIN = float(np.float32(1e-3))
T_MAX = float(np.float32(1e7))
FLT_MIN = float(np.finfo(np.float32).tiny)
RHO = 2.0 ** -22 + U
SLACK = 2.0 ** -46
PAD = 10000.0
MARGIN = 2.0 ** -17          # form 3's pass-1 margin: 2^-17 (|s|^2 + o.o)


def scene_arrays(spheres):
    """(centres float32 [n,3], r^2 float32 [n]) exactly as tpt_scene_pack.h stages them."""
    raw = np.asarray(spheres).view(np.float32).reshape(-1, 5)
    r = raw[:, 3].copy()
    return np.ascontiguousarray(raw[:, :3]), (r * r).astype(np.float32)


def gate_passes(spheres):
    """tpt_set_scene's expanded-form gate: every sphere has |s|^2 <= 128 + 2 r^2 (in double)."""
    raw = np.asarray(spheres).view(np.float32).reshape(-1, 5).astype(np.float64)
    return bool(((raw[:, :3] ** 2).sum(1) <= 128.0 + 2.0 * raw[:, 3] ** 2).all())


def _groups(centres, r2):
    """Per sphere, the lowest id of the spheres with bit-identical {centre, r^2} (exact duplicates)."""
    key = np.concatenate([centres.view(np.uint32), r2.view(np.uint32)[:, None]], 1)
    _, first, inv = np.unique(key, axis=0, return_index=True, return_inverse=True)
    return first[inv.reshape(-1)]


def _chain(terms, x0=None, e0=None):
    """Running error of a float32 fma chain fl(t_1 + fl(t_2 + ... fl(t_n + x0))) whose terms t_k are exact products:
    the exact partial sums p_k and the bound e_k = e_{k-1} + u (|p_k| + e_{k-1}) on |computed p_k - p_k| (each step
    rounds once; the computed partial sum is at most |p_k| + e_{k-1} in magnitude). Without x0 the innermost term is a
    plain product, rounded once. Returns (p_n, e_n)."""
    if x0 is None:
        p, e = terms[0], U * np.abs(terms[0])
        terms = terms[1:]
    else:
        p, e = x0, e0
    for t in terms:
        p = t + p
        e = e + U * (np.abs(p) + e)
    return p, e


def pair_bounds(o, d, s, r2, expanded=True):
    """Exact (float64) nb, c of rays o, d [R,1,3] against spheres s [1,S,3], r2 [1,S], and bounds on how far the
    float32 forms' computed nb, c can be from them: the larger of the reference and expanded forms' running-error bounds,
    or the reference form's alone when `expanded` is False (a scene that fails the gate)."""
    co = s - o
    nb = (co * d).sum(-1)
    c = (co * co).sum(-1) - r2
    # reference form: co = fl32(s - o) is computed exactly here (IEEE subtraction), then the two fma chains
    co32 = (s.astype(np.float32) - o.astype(np.float32)).astype(np.float64)
    x, y, z = co32[..., 0], co32[..., 1], co32[..., 2]
    dx, dy, dz = d[..., 0], d[..., 1], d[..., 2]
    q, eq = _chain([z * dz, y * dy, x * dx])
    enb_ref = np.abs(q - nb) + eq
    p, ep = _chain([-z * z, -y * y, -x * x], r2 + 0 * x, 0.0)
    ec_ref = np.abs(-p - c) + ep
    # expanded form: nod = -(o.d), nb = s.d + nod; oo = o.o, c = -2 s.o + fl(K + oo), K = fl32(|s|^2 - r^2) from double
    ox, oy, oz = o[..., 0], o[..., 1], o[..., 2]
    sx, sy, sz = s[..., 0], s[..., 1], s[..., 2]
    a, ea = _chain([oz * dz, oy * dy, ox * dx])
    b, eb = _chain([sz * dz, sy * dy, sx * dx], -a, ea)
    enb_exp = np.abs(b - nb) + eb
    oo, eo = _chain([oz * oz, oy * oy, ox * ox])
    Kd = (s * s).sum(-1) - r2
    K32 = Kd.astype(np.float32).astype(np.float64)
    k0 = K32 + oo
    ek0 = eo + U * (np.abs(k0) + eo)
    cx, ecx = _chain([-2 * sz * oz, -2 * sy * oy, -2 * sx * ox], k0, ek0)
    ec_exp = np.abs(cx - c) + ecx
    mag = (s * s).sum(-1) + (o * o).sum(-1) + (co * co).sum(-1) + r2
    if not expanded:
        enb_exp, ec_exp = enb_ref, ec_ref
    enb = np.maximum(enb_ref, enb_exp) + SLACK * (np.sqrt(mag) + 1)
    ec = np.maximum(ec_ref, ec_exp) + SLACK * (mag + 1)
    return nb, c, enb, ec


def classify(nb, c, enb, ec):
    """Outcome per pair: 0 reject, 1 accept t-, 2 accept t+, -1 ambiguous; with the enclosure [tlo, thi] of the chosen
    root and its float64 value t (inf for a reject)."""
    nlo, nhi = nb - enb, nb + enb
    n2lo = np.where((nlo <= 0) & (nhi >= 0), 0.0, np.minimum(nlo * nlo, nhi * nhi))
    n2hi = np.maximum(nlo * nlo, nhi * nhi)
    dlo = n2lo - (c + ec)
    dhi = n2hi - (c - ec)
    slack = SLACK * (n2hi + np.abs(c) + ec)
    dlo, dhi = dlo - slack, dhi + slack
    sqlo = np.sqrt(np.maximum(dlo, 0.0)) * (1 - RHO)
    sqhi = np.sqrt(np.maximum(dhi, 0.0)) * (1 + RHO)
    tm_lo, tm_hi = nlo - sqhi, nhi - sqlo
    tp_lo, tp_hi = nlo + sqlo, nhi + sqhi
    w = U * np.maximum(np.abs(tm_lo), np.abs(tm_hi))
    tm_lo, tm_hi = tm_lo - w, tm_hi + w
    w = U * np.maximum(np.abs(tp_lo), np.abs(tp_hi))
    tp_lo, tp_hi = tp_lo - w, tp_hi + w
    D = nb * nb - c
    sq = np.sqrt(np.maximum(D, 0.0))
    out = np.full(nb.shape, -1, np.int8)
    rej = (dhi <= 0) | (tp_hi < T_MIN)
    pos = dlo > FLT_MIN
    am = pos & (tm_lo > T_MIN)
    ap = pos & (tm_hi < T_MIN) & (tp_lo > T_MIN)
    out[ap] = 2
    out[am] = 1
    out[rej] = 0
    tlo = np.where(am, tm_lo, np.where(ap, tp_lo, np.inf))
    thi = np.where(am, tm_hi, np.where(ap, tp_hi, np.inf))
    t = np.where(am, nb - sq, np.where(ap, nb + sq, np.inf))
    far = (out > 0) & (tlo >= T_MAX)          # beyond tMax: never accepted (not reached by any scene here)
    out[far] = np.where(thi[far] >= T_MAX, 0, -1)
    return out, t, tlo, thi


def nearest_hit(rays, spheres, expanded=None, pairs_per_chunk=1 << 21):
    """The oracle. rays float32 [n,6] {o, d}; spheres as given to set_scene (real spheres only); expanded: whether the
    expanded form's bound applies (default: the scene passes the gate). Returns a dict of id (int, -1 = no hit), t, tlo,
    thi (float64; tMax for no hit) and well (bool) per ray."""
    centres, r2 = scene_arrays(spheres)
    if expanded is None:
        expanded = gate_passes(spheres)
    s = centres.astype(np.float64)[None]
    R2 = r2.astype(np.float64)[None]
    grp = _groups(centres, r2)
    n, S = len(rays), len(r2)
    res = dict(id=np.full(n, -1, np.int64), t=np.full(n, T_MAX), tlo=np.full(n, T_MAX), thi=np.full(n, T_MAX),
               well=np.zeros(n, bool))
    step = max(1, pairs_per_chunk // max(S, 1))
    for a in range(0, n, step):
        r = rays[a:a + step].astype(np.float64)
        o, d = r[:, None, :3], r[:, None, 3:]
        out, t, tlo, thi = classify(*pair_bounds(o, d, s, R2, expanded))
        m = len(r)
        ok = (out >= 0).all(1)
        w = np.argmin(t, 1)                                   # first minimum = lowest id among exact ties
        rows = np.arange(m)
        hit = np.isfinite(t[rows, w])
        # runner-up: every other accepted sphere that is not a bit-identical copy of the winner
        other = grp[None, :] != grp[w][:, None]
        ru = np.where(other, tlo, np.inf).min(1)
        sep = ~hit | (thi[rows, w] < ru)
        res["id"][a:a + m] = np.where(hit, grp[w], -1)
        res["t"][a:a + m] = np.where(hit, t[rows, w], T_MAX)
        res["tlo"][a:a + m] = np.where(hit, tlo[rows, w], T_MAX)
        res["thi"][a:a + m] = np.where(hit, thi[rows, w], T_MAX)
        res["well"][a:a + m] = ok & sep
    return res


def pad_possible(rays, count):
    """Rays on which form 0's padded sphere (centre 10000^3, r^2 = 0) is not certainly rejected (its D may round >= 0)."""
    simd = (count + 3) // 4 * 4
    if simd == count:
        return np.zeros(len(rays), bool)
    r = rays.astype(np.float64)
    s = np.full((1, 1, 3), PAD)
    out, *_ = classify(*pair_bounds(r[:, None, :3], r[:, None, 3:], s, np.zeros((1, 1))))
    return out[:, 0] != 0


# ---- scenes --------------------------------------------------------------------------------------------------------
def make_scene(count, layout, seed=0):
    """A runtime scene of `count` spheres with one exact duplicate pair (ids dup, dup + 1; count >= 2).
    compact: passes the expanded-form gate (tpt_set_scene: |s|^2 <= 128 + 2 r^2): a ground sphere (0,-100.5,-1) r=100 and
             small spheres with |s| <= 8.
    spread:  fails it: a giant sphere (0,-1000,0) r=1000 whose surface is the scene's floor, and small spheres on a grid
             that reaches |s| >> 11 (like the stress scene).
    Returns (spheres, materials, camera, dup) with dup = -1 when there is no pair."""
    import toypathtracer_b200 as tpt
    rng = np.random.default_rng(seed * 7919 + count * 2 + (layout == "spread"))
    sph = np.zeros(count, tpt.SPHERE_DTYPE)
    mats = np.zeros(count, tpt.MATERIAL_DTYPE)
    big = count >= 3
    first = 1 if big else 0
    k = count - first
    if layout == "compact":
        if big:
            sph[0] = ((0, -100.5, -1), 100, 0)
        rmax = float(np.clip(7.0 / max(k, 1) ** (1 / 3), 0.25, 1.0))
        dirs = rng.normal(size=(k, 3)); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        cen = dirs * 8.0 * rng.random(k)[:, None] ** (1 / 3)
        cen[:, 1] = np.abs(cen[:, 1]) * 0.5
        rad = rmax * (0.4 + 0.6 * rng.random(k))
    else:
        if big:
            sph[0] = ((0, -1000, 0), 1000, 0)
        side = int(np.ceil(np.sqrt(max(k, 1))))
        pitch = max(1.0, 24.0 / side)              # small scenes are spread wide too: the gate must fail
        g = np.arange(k)
        rad = 0.2 + 0.15 * rng.random(k)
        x = ((g % side) - side / 2 + 0.15 + 0.7 * rng.random(k)) * pitch
        z = ((g // side) - side / 2 + 0.15 + 0.7 * rng.random(k)) * pitch - side * pitch / 4
        cen = np.stack([x, rad, z], 1)
        if k >= 1:
            cen[0] = (20.0, 0.8, -15.0); rad[0] = 0.8     # fails the gate whatever the count
    sph["center"][first:] = cen
    sph["radius"][first:] = rad
    dup = -1
    if count >= 2:
        cand = np.arange(first, count - 1)
        cand = cand[cand % 64 != 63]                       # keep the pair inside one 64-sphere chunk
        dup = int(rng.choice(cand)) if len(cand) else first
        sph[dup + 1] = sph[dup]
    sph["invRadius"] = (np.float32(1) / sph["radius"]).astype(np.float32)
    t = rng.random(count)
    mats["type"] = np.where(t < 0.6, 0, np.where(t < 0.85, 1, 2))
    mats["albedo"] = 0.2 + 0.7 * rng.random((count, 3))
    mats["roughness"] = np.where(mats["type"] == 1, 0.5 * rng.random(count), 0)
    mats["ri"] = np.where(mats["type"] == 2, 1.5, 0)
    if big:
        mats[0] = (0, (0.5, 0.5, 0.5), (0, 0, 0), 0, 0)
    nl = min(4, max(0, count - 3))
    if nl:
        lights = rng.choice(np.arange(first, count), nl, replace=False)
        lights = lights[(lights != dup) & (lights != dup + 1)]
        mats["type"][lights] = 0
        mats["emissive"][lights] = (8, 7, 6)
    cam = tpt.make_camera((0, 6, 14), (0, 0.5, -2), (0, 1, 0), 50, 16 / 9, 0.02, 14)
    return sph, mats, cam, dup


# ---- ray generators ------------------------------------------------------------------------------------------------
def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _gap_ok(o, centres, radii, tol, grp, skip):
    """Distance from each origin o[i] to every sphere surface outside group skip[i] exceeds tol[i]."""
    from scipy.spatial import cKDTree
    c = centres.astype(np.float64); r = radii.astype(np.float64)
    small = r < 50
    ok = np.ones(len(o), bool)
    for j in np.nonzero(~small)[0]:                  # the giant / ground spheres: check against every origin
        g = np.abs(np.linalg.norm(o - c[j], axis=1) - r[j])
        ok &= (g > tol) | (skip == grp[j])
    idx = np.nonzero(small)[0]
    if len(idx):
        tree = cKDTree(c[idx])
        reach = r[idx].max() + tol.max() + 1e-3
        for i, near in enumerate(tree.query_ball_point(o, reach)):
            if not ok[i] or not near:
                continue
            jj = idx[near]
            g = np.abs(np.linalg.norm(o[i] - c[jj], axis=1) - r[jj])
            ok[i] = ((g > tol[i]) | (grp[jj] == skip[i])).all()
    return ok


def aimed_rays(spheres, seed, tries=96):
    """For each real sphere k (the higher id of an exact duplicate pair stands for the lower one): a ray from outside it,
    aimed at its centre, whose origin lies delta = clip(0.2 r, 0.01, 0.2) (later tries: 0.05 r and 0.02 r, at least 0.005 and 0.002) from k's surface and more than 2 delta from every
    other sphere surface. The first root along the ray is then k's, at t = delta, and every other sphere's hit is beyond
    2 delta: k is the unique, well-conditioned nearest hit. Returns (rays float32 [m,6], target ids [m]); spheres for which
    no such origin was found in `tries` random directions are left out (none in the scenes used here)."""
    rng = np.random.default_rng(seed)
    centres, r2 = scene_arrays(spheres)
    radii = np.asarray(spheres).view(np.float32).reshape(-1, 5)[:, 3].astype(np.float64)
    grp = _groups(centres, r2)
    n = len(radii)
    todo = np.nonzero(grp == np.arange(n))[0]
    out_r, out_k = [], []
    for it in range(tries):
        if not len(todo):
            break
        nrm = _unit(rng.normal(size=(len(todo), 3)))
        delta = (np.clip(0.2 * radii[todo], 0.01, 0.2) if it < tries // 3 else np.clip(0.05 * radii[todo], 0.005, 0.05)
                 if it < 2 * tries // 3 else np.clip(0.02 * radii[todo], 0.002, 0.02))
        o = (centres[todo].astype(np.float64) + nrm * (radii[todo] + delta)[:, None]).astype(np.float32)
        d = _unit(centres[todo].astype(np.float64) - o.astype(np.float64)).astype(np.float32)
        # a bit-identical copy of k is k itself (same t bits, lower id wins): its surface is not an obstacle
        ok = _gap_ok(o.astype(np.float64), centres, radii, 2 * delta, grp, todo)
        out_r.append(np.concatenate([o[ok], d[ok]], 1)); out_k.append(todo[ok])
        todo = todo[~ok]
    return np.concatenate(out_r).astype(np.float32), np.concatenate(out_k)


def near_tangent_rays(spheres, n, seed, band=4.0):
    """Rays whose exact discriminant against a chosen sphere k lies within +-band times form 3's pass-1 margin
    2^-17 (|s_k|^2 + o.o), both signs, log-uniform in [band/1000, band] margins: origins at camera distance (8..20 from
    k) and on other spheres' surfaces. Returns (rays, k, D/margin as built)."""
    rng = np.random.default_rng(seed)
    centres, r2 = scene_arrays(spheres)
    radii = np.asarray(spheres).view(np.float32).reshape(-1, 5)[:, 3].astype(np.float64)
    c64 = centres.astype(np.float64)
    k = rng.integers(0, len(radii), n)
    cam = rng.random(n) < 0.5
    o = np.empty((n, 3))
    o[cam] = c64[k[cam]] + _unit(rng.normal(size=(int(cam.sum()), 3))) * rng.uniform(8, 20, (int(cam.sum()), 1))
    m = rng.integers(0, len(radii), int((~cam).sum()))
    o[~cam] = c64[m] + _unit(rng.normal(size=(len(m), 3))) * radii[m, None]
    o = o.astype(np.float32).astype(np.float64)
    s = c64[k]
    margin = MARGIN * ((s * s).sum(1) + (o * o).sum(1))
    frac = band * 10.0 ** (-3 * rng.random(n)) * np.where(rng.random(n) < 0.5, -1, 1)
    b2 = r2[k].astype(np.float64) - frac * margin                       # D = R - b^2 for a unit direction
    w = s - o
    L = np.linalg.norm(w, axis=1)
    good = (b2 > 0) & (L > np.sqrt(np.maximum(b2, 0)) + 1e-3)
    w = w / L[:, None]
    p = _unit(np.cross(w, rng.normal(size=(n, 3))))
    sin = np.sqrt(np.maximum(b2, 0)) / L
    d = np.sqrt(np.clip(1 - sin ** 2, 0, 1))[:, None] * w + sin[:, None] * p
    rays = np.concatenate([o, d], 1).astype(np.float32)[good]
    return rays, k[good], frac[good]


def tmin_rays(spheres, n, seed):
    """Origins within 3e-3 of a sphere surface, inside and outside (distance e, log-uniform 2e-4..3e-3 of both signs),
    directions half straight in/out, half random: the first root falls at or near tMin = 1e-3."""
    rng = np.random.default_rng(seed)
    centres, _ = scene_arrays(spheres)
    radii = np.asarray(spheres).view(np.float32).reshape(-1, 5)[:, 3].astype(np.float64)
    k = rng.integers(0, len(radii), n)
    nrm = _unit(rng.normal(size=(n, 3)))
    e = 2e-4 * 15.0 ** rng.random(n) * np.where(rng.random(n) < 0.5, -1, 1)
    o = centres[k].astype(np.float64) + nrm * (radii[k] + e)[:, None]
    d = np.where((rng.random(n) < 0.5)[:, None], nrm * np.where(rng.random(n) < 0.5, -1, 1)[:, None],
                 _unit(rng.normal(size=(n, 3))))
    return np.concatenate([o, _unit(d)], 1).astype(np.float32), k, e


def degenerate_rays(spheres, seed):
    """Axis-aligned directions with exact +-0 components, origins exactly at sphere centres, origins at |o| ~ 1e3."""
    rng = np.random.default_rng(seed)
    centres, _ = scene_arrays(spheres)
    axes = []
    for a in range(3):
        for sgn in (1.0, -1.0):
            for zs in ((0.0, 0.0), (-0.0, 0.0), (0.0, -0.0), (-0.0, -0.0)):
                v = [zs[0], zs[1]]
                v.insert(a, sgn)
                axes.append(v)
    axes = np.array(axes, np.float32)
    o1 = centres[rng.integers(0, len(centres), 16)]                       # at a centre
    o2 = np.array([[0, 6, 14], [0.5, 1.0, 0.0], [0, 0, 0], [-0.0, 0.25, -0.0]], np.float32)
    far = _unit(rng.normal(size=(8, 3))) * 1000.0                          # |o| ~ 1e3, looking back at the scene
    rays = [np.concatenate([np.repeat(oo[None], len(axes), 0), axes], 1) for oo in np.concatenate([o1, o2])]
    rays.append(np.concatenate([far, _unit(-far + rng.normal(size=far.shape))], 1))
    rays.append(np.concatenate([far, _unit(-far)], 1))
    return np.concatenate(rays).astype(np.float32)


def pad_aimed_rays(n, seed):
    """Rays aimed exactly (in float64, then rounded) at the padding point (10000, 10000, 10000)."""
    rng = np.random.default_rng(seed)
    o = rng.uniform(-12, 12, (n, 3)); o[:, 1] = np.abs(o[:, 1])
    o = o.astype(np.float32).astype(np.float64)
    return np.concatenate([o, _unit(PAD - o)], 1).astype(np.float32)


# ---- exact rational reference ----------------------------------------------------------------------------------------
_TMIN_Q = Fraction(T_MIN)


def exact_hit(ray, centres, r2):
    """Exact outcome per sphere (0 reject / 1 t- / 2 t+), sign of D, and the winner, from the float32 inputs as rationals;
    the winning t is compared in 120-digit decimal (exact up to equal values, which only bit-identical spheres produce)."""
    o = [Fraction(float(v)) for v in ray[:3]]
    d = [Fraction(float(v)) for v in ray[3:]]
    outs, signs, ts = [], [], []
    ctx = decimal.Context(prec=120)
    for s, R in zip(centres, r2):
        co = [Fraction(float(s[i])) - o[i] for i in range(3)]
        nb = sum(co[i] * d[i] for i in range(3))
        c = sum(x * x for x in co) - Fraction(float(R))
        D = nb * nb - c
        signs.append((D > 0) - (D < 0))
        out, t = 0, None
        if D > 0:
            a = nb - _TMIN_Q                       # t- > tMin <=> a > sqrt(D);  t+ > tMin <=> a > -sqrt(D)
            if a > 0 and a * a > D:
                out = 1
            elif a >= 0 or a * a < D:
                out = 2
            if out:
                sq = ctx.sqrt(ctx.divide(decimal.Decimal(D.numerator), decimal.Decimal(D.denominator)))
                nbd = ctx.divide(decimal.Decimal(nb.numerator), decimal.Decimal(nb.denominator))
                t = nbd - sq if out == 1 else nbd + sq
        outs.append(out)
        ts.append(t)
    best, bid = None, -1
    for i, t in enumerate(ts):
        if t is not None and t < decimal.Decimal(T_MAX) and (best is None or t < best):
            best, bid = t, i
    return outs, signs, bid, best


# ---- tests -----------------------------------------------------------------------------------------------------------
def _exact_check_scenes():
    import toypathtracer_b200 as tpt
    out = []
    for layout in ("compact", "spread"):
        sph, mats, cam, dup = make_scene(20, layout, seed=3)
        out.append((f"{layout}20", sph))
    s = tpt.stress_scene(64, 36, count=20)
    out.append(("stress20", s[0]))
    return out


def test_oracle_matches_exact_rational_arithmetic():
    """~2 000 rays x 20 spheres: on every ray the oracle calls well-conditioned, the sign of D, the root choice and the
    winner equal the exact result, and the exact t lies inside the oracle's bound; the bounds hold on EVERY ray (the exact
    nb, c of each pair inside the box is what makes that so, and the exact outcome must be one the box allows)."""
    total, well_total = 0, 0
    for name, sph in _exact_check_scenes():
        centres, r2 = scene_arrays(sph)
        sets = [surface_rays(sph, 240, 1), near_tangent_rays(sph, 200, 2)[0], tmin_rays(sph, 150, 3)[0],
                degenerate_rays(sph, 4)[::3], pad_aimed_rays(16, 5), aimed_rays(sph, 6)[0]]
        rays = np.concatenate(sets)
        rays = rays[np.isfinite(rays).all(1)]
        ora = nearest_hit(rays, sph)
        r = rays.astype(np.float64)
        outs_o, *_ = classify(*pair_bounds(r[:, None, :3], r[:, None, 3:], centres.astype(np.float64)[None],
                                           r2.astype(np.float64)[None]))
        for i, ray in enumerate(rays):
            outs, signs, bid, best = exact_hit(ray, centres, r2)
            for j in range(len(r2)):
                if outs_o[i, j] >= 0:
                    assert outs_o[i, j] == outs[j], (name, i, j, outs_o[i, j], outs[j])
                    if outs[j] == 0:
                        pass
                    else:
                        assert signs[j] > 0
            if ora["well"][i]:
                well_total += 1
                assert ora["id"][i] == bid, (name, i, ora["id"][i], bid)
                if bid >= 0:
                    assert decimal.Decimal(ora["tlo"][i]) <= best <= decimal.Decimal(ora["thi"][i]), (name, i)
        total += len(rays)
    assert total >= 2000
    assert well_total > 0.5 * total, (well_total, total)


def test_oracle_sees_the_duplicate_tie():
    """An exact duplicate pair ties on every ray: the oracle reports the lower id, well-conditioned."""
    sph, mats, cam, dup = make_scene(40, "compact", seed=1)
    rays, k = aimed_rays(sph, 7)
    sel = k == dup
    assert sel.sum() == 1
    res = nearest_hit(rays[sel], sph)
    assert res["well"].all() and (res["id"] == dup).all()


@pytest.mark.parametrize("layout", ["compact", "spread"])
@pytest.mark.parametrize("count", [1, 2, 3, 7, 46, 130])
def test_scene_generator(layout, count):
    """make_scene: compact passes the expanded-form gate, spread fails it, one exact duplicate pair in one chunk."""
    sph, mats, cam, dup = make_scene(count, layout)
    assert len(sph) == count and np.isfinite(sph["center"]).all()
    assert gate_passes(sph) == (layout == "compact")
    if count >= 2:
        assert sph[dup].tobytes() == sph[dup + 1].tobytes() and dup // 64 == (dup + 1) // 64
        assert len(np.unique(np.asarray(sph).view(np.uint8).reshape(count, 20), axis=0)) == count - 1


@pytest.mark.parametrize("layout", ["compact", "spread"])
def test_aimed_rays_hit_their_sphere(layout):
    """Every real sphere gets an aimed ray, and the oracle agrees: its target, uniquely and well-conditioned."""
    sph, mats, cam, dup = make_scene(150, layout, seed=2)
    rays, k = aimed_rays(sph, 8)
    assert set(k) == set(range(150)) - {dup + 1}
    res = nearest_hit(rays, sph)
    assert res["well"].all()
    assert (res["id"] == k).all()
    delta = np.linalg.norm(rays[:, :3].astype(np.float64) - sph["center"][k], axis=1) - sph["radius"][k]
    assert (res["tlo"] <= delta * (1 + 1e-4)).all() and (res["thi"] >= delta * (1 - 1e-4)).all()
    assert (delta >= 0.0019).all()


def test_aimed_rays_on_reference_and_stress_scenes(libs):
    for sph in (golden_scene()[0], libs.stress_scene(64, 36, count=300)[0]):
        rays, k = aimed_rays(sph, 9)
        centres, r2 = scene_arrays(sph)
        assert len(set(k)) == len(np.unique(_groups(centres, r2)))
        res = nearest_hit(rays, sph)
        assert res["well"].all() and (res["id"] == k).all()


@pytest.mark.parametrize("layout", ["compact", "spread"])
def test_near_tangent_rays_land_in_the_band(layout):
    """The near-tangent set: exact D against its sphere within +-4 margins, both signs well represented, and a good share
    within the expanded form's own error bound (where form 3's margin decides)."""
    sph, *_ = make_scene(100, layout, seed=4)
    rays, k, frac = near_tangent_rays(sph, 2000, 10)
    assert len(rays) > 1800
    centres, r2 = scene_arrays(sph)
    r = rays.astype(np.float64)
    s = centres[k].astype(np.float64)
    nb = ((s - r[:, :3]) * r[:, 3:]).sum(1)
    c = ((s - r[:, :3]) ** 2).sum(1) - r2[k]
    D = nb * nb - c
    margin = MARGIN * ((s * s).sum(1) + (r[:, :3] ** 2).sum(1))
    q = D / margin
    assert (np.abs(q) <= 4.5).all()
    assert (q > 0).mean() > 0.3 and (q < 0).mean() > 0.3
    _, _, enb, ec = pair_bounds(r[:, None, :3], r[:, None, 3:], s[:, None], r2[k].astype(np.float64)[:, None])
    inside = np.abs(D) < (2 * np.abs(nb) * enb[:, 0] + ec[:, 0])
    assert inside.mean() > 0.2


def test_tmin_rays_straddle_the_surface():
    sph, *_ = make_scene(60, "compact", seed=5)
    rays, k, e = tmin_rays(sph, 1000, 11)
    centres, _ = scene_arrays(sph)
    dist = np.linalg.norm(rays[:, :3].astype(np.float64) - centres[k], axis=1) - sph["radius"][k]
    assert (np.abs(dist) < 3.1e-3).all() and (dist > 0).mean() > 0.3 and (dist < 0).mean() > 0.3
    res = nearest_hit(rays, sph)
    assert 0.2 < res["well"].mean() < 1.0


def test_degenerate_and_pad_aimed_rays():
    sph, *_ = make_scene(45, "compact", seed=6)
    rays = degenerate_rays(sph, 12)
    d = rays[:, 3:]
    assert ((d == 0) & np.signbit(d)).any() and ((d == 0) & ~np.signbit(d)).any()
    centres, _ = scene_arrays(sph)
    assert (rays[:, None, :3] == centres[None]).all(2).any()
    assert (np.linalg.norm(rays[:, :3], axis=1) > 900).any()
    res = nearest_hit(rays, sph)
    assert res["well"].mean() > 0.5
    pad = pad_aimed_rays(64, 13)
    assert pad_possible(pad, 45).all()                         # 45 spheres pad to 48: form 0 may return 45..47 there
    assert not pad_possible(pad, 44).any()                     # no padding, nothing to hit
    assert not pad_possible(surface_rays(sph, 2000, 14), 45).any()


def test_well_conditioned_fraction_of_surface_rays(libs):
    """The oracle decides most rays a path tracer produces: >= 0.9 of the surface/camera rays on the reference scene,
    the stress scene's first 1024 spheres and both synthetic layouts."""
    cases = [("reference", golden_scene()[0]), ("stress1024", libs.stress_scene(64, 36, count=1024)[0]),
             ("compact300", make_scene(300, "compact")[0]), ("spread300", make_scene(300, "spread")[0])]
    for name, sph in cases:
        rays = surface_rays(sph, 3000 if len(sph) < 1000 else 1000, 15)
        rays = rays[np.isfinite(rays).all(1)]
        res = nearest_hit(rays, sph)
        frac = res["well"].mean()
        print(f"{name}: well-conditioned {frac:.4f} of {len(rays)} surface/camera rays")
        assert frac >= 0.9, (name, frac)
        assert 0.2 < (res["id"][res["well"]] >= 0).mean() < 0.95
