"""The pose solver (K10 GNC-TLS yaw + K11 COTE, quatro.hpp:388-572, 585-747, 806-936, teaser/utils.h:151-166) on cliques built to hit
the places where pose_kernel can go wrong: the GNC control flow (the mu <= 0 exit, iteration caps, cost thresholds 0 and inf, GNC
factors 1 / 1.0001 / 100, the 1e-16 -> 1e-2 noise-bound substitution, max r^2 at nb^2/2 (1 -+ 2^-20)), yaw at 0 / 90 / 180 and
+-179.99 degrees, near-reflection H, zero chain vectors; COTE with tied events, consensus back to 0 in mid-sweep, a non-dyadic range,
signed zeros, targets 4e5 / 5e6 m out, median candidate sets of 1 ... 4100 members (including upper-end events); rotation-inlier COTE
with 0, 1, all and a wrapping run of inliers; the RyRx prior in both branches; cliques of 2 ... 32768 members on both sides of the
shared-memory / workspace switch at 4096.

The float64 restatement below is written from the reference text, not from the oracle:
- GNC-TLS: H as an exactly rounded sum (math.fsum), the yaw as the maximiser of trace(R H) in long double, and, per iteration, the
  margin of every decision against an error bound of the implementation under test (see _gnc_error_model).
- everything downstream of R (chain -> rotation inliers -> COTE inputs -> sweep -> median -> masks -> final list) in Python floats in
  the kernel's operation order: exact float64, so given an implementation's R and rotation mask it must agree bit for bit.

CPU: the oracle's yaw lies within its bound of the exact one, its discrete outputs equal the restatement's wherever every margin holds,
and everything downstream of its R is bit-identical.  GPU (-m gpu, through the C-ABI): the same for qb200_solve_pose, plus one mixed
qb200_solve_batch_each wave through 1 and 4 lanes that must be byte-identical to the single-pair calls."""
import math

import numpy as np
import pytest

from quatro_b200.capi import (COTE_MEDIAN, COTE_WEIGHTED_MEAN, INLIER_NONE, MEM_HOST, SET_LISTS, Handle, ListBuffers, Params,
                              QuatroB200Error, default_params)
from support import P4

U = 2.0 ** -53
LD = np.longdouble
SAFE = 1e3            # a discrete decision is compared only where its margin exceeds SAFE x its propagated error bound
WELL_CONDITIONED = 1e-9


def _prm(**kw):
    """Default params with rot_noise_bound explicit (0 would latch on the device and be 2 noise_bound per call in the oracle)."""
    p = default_params()
    p.rot_noise_bound = 0.6
    for k, v in kw.items():
        if k == "RyRx":
            p.use_pre_estimated_RyRx = 1
            for i, e in enumerate(np.asarray(v, float).ravel()):
                p.RyRx[i] = float(e)
        else:
            setattr(p, k, v)
    return p


# ==== float64 restatement =====================================================================================================
def chain_tims(a4, b4, clique):
    """quatro.hpp:828-843: x_i = src(leaf) - src(root), y_i = tgt(leaf) - tgt(root), leaf = the next member (cyclic); XY rows."""
    cl = np.asarray(clique, np.int64)
    lf = np.roll(cl, -1)
    A, B = a4[:, :2].astype(np.float64), b4[:, :2].astype(np.float64)
    return A[lf] - A[cl], B[lf] - B[cl]


class _Margins:
    """Smallest ratio margin / error bound over every recorded decision (inf: every decision exact)."""

    def __init__(self):
        self.ratio = math.inf

    def add(self, margin, err):
        margin, err = np.asarray(margin, np.float64), np.asarray(err, np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            r = np.where(err > 0, margin / err, np.inf)
        r = np.where(np.isnan(r), 0.0, r)                  # an undefined error bound is no margin
        if r.size:
            self.ratio = min(self.ratio, float(np.min(r)))


def _gnc_error_model(c, kind):
    """Rounding steps between a product x w y and the implementation's H entry.  The device sums per thread chains of ceil(c / 256)
    terms, then 5 shuffle levels and 8 warp partials: |dH| <= (ceil(c/256) + 13) u sum|terms|.  The oracle sums sequentially:
    (c - 1) u sum|terms|, and its Jacobi SVD adds a few u ||H||.  +2 covers the restatement's own rounded products."""
    if kind == "device":
        return -(-c // 256) + 13 + 2, 0.0
    return c - 1 + 2, 32.0


def _r2_error(xn, yn, r2, eps):
    """Bound on |implementation r^2 - r^2| for a yaw error eps: 2 |x| |r| eps + |x|^2 eps^2 + the rounding of the residual."""
    if not eps < math.inf:
        return np.full(len(xn), math.inf)
    return 2 * xn * np.sqrt(r2) * eps + (xn * eps) ** 2 + 8 * U * (xn + yn) ** 2


def ref_gnc(x, y, p, kind="device"):
    """solveForRotation2D (quatro.hpp:430-572) in exact / long double arithmetic.  Returns the yaw of the last rotation, the bound
    on |implementation yaw - yaw| (eps), the iteration count, the weights' >= 0.4 mask, the cost, why the loop ended, and the smallest
    ratio margin / error over every decision: r^2 vs th1 / th2, the weight vs 0.4, cost_diff vs the threshold, 2 max r^2 / nb^2 - 1
    vs 0 at iteration 0.  Every error is propagated from eps (a yaw error moves r^2 by 2 |x| |r| eps) and from mu's error."""
    c = len(x)
    nb2 = p.rot_noise_bound * p.rot_noise_bound
    if nb2 < 1e-16:
        nb2 = 1e-2
    ksum, ksvd = _gnc_error_model(c, kind)
    x0, x1, y0, y1 = x[:, 0], x[:, 1], y[:, 0], y[:, 1]
    xn, yn = np.hypot(x0, x1), np.hypot(y0, y1)
    axy = np.abs(x0 * y0) + np.abs(x0 * y1) + np.abs(x1 * y0) + np.abs(x1 * y1)
    w = np.ones(c, LD)
    dw = np.zeros(c)                      # bound on |implementation weight - w|
    mu, rel_mu, prev, cost, cost_err_prev = 1.0, 0.0, math.inf, math.inf, 0.0
    yaw, eps, iters, exit_, nn, hn, S, cond0 = LD(0), 0.0, 0, "max_iterations", 0.0, 0.0, 0.0, 0.0
    m = _Margins()
    for it in range(p.rotation_max_iterations):
        iters = it + 1
        wd = w.astype(np.float64)
        t00, t01, t10, t11 = x0 * wd * y0, x0 * wd * y1, x1 * wd * y0, x1 * wd * y1
        cc = math.fsum(np.concatenate([t00, t11]).tolist())
        ss = math.fsum(np.concatenate([t01, -t10]).tolist())
        S = math.fsum(np.abs(np.concatenate([t00, t01, t10, t11])).tolist())
        hn = math.sqrt(math.fsum(t00.tolist()) ** 2 + math.fsum(t01.tolist()) ** 2 + math.fsum(t10.tolist()) ** 2 + math.fsum(t11.tolist()) ** 2)
        nn = math.hypot(cc, ss)
        if it == 0:
            cond0 = nn / hn if hn > 0 else 0.0
        yaw = np.arctan2(LD(ss), LD(cc)) if nn > 0 else LD(0)
        prop = math.fsum((dw * axy).tolist())
        if nn > 0:
            eps0 = (ksum * U * S + ksvd * U * hn) / nn + 8 * U
            eps = eps0 + prop / nn
        else:   # H = 0 exactly (every weight or chain vector 0): the identity everywhere; cc = ss = 0 with H != 0: every yaw maximises
            eps0 = eps = 0.0 if S == 0 and prop == 0 else math.inf
        cs, sn = np.cos(yaw), np.sin(yaw)
        dx = y0.astype(LD) - (cs * x0 - sn * x1)
        dy = y1.astype(LD) - (sn * x0 + cs * x1)
        r2 = dx * dx + dy * dy
        r2d = r2.astype(np.float64)
        E = _r2_error(xn, yn, r2d, eps)
        E0 = _r2_error(xn, yn, r2d, eps0)
        if it == 0:
            j = int(np.argmax(r2))
            q = 2 * r2[j] / nb2 - 1
            m.add(abs(float(q)), 2 * E[j] / nb2 + 4 * U)
            mu = float(1 / (2 * float(r2d[j]) / nb2 - 1))
            rel_mu = (2 * E[j] / nb2 + 4 * U) / max(abs(float(q)), 1e-300)
            if mu <= 0:
                exit_ = "mu"
                break
        th1 = (mu + 1) / mu * nb2
        th2 = mu / (mu + 1) * nb2
        th_err = rel_mu / (mu + 1) + 4 * U
        m.add(np.abs(r2d - th1), E + th1 * th_err)
        m.add(np.abs(r2d - th2), E + th2 * th_err)
        cost = float(np.sum(w * r2))
        cost_err = float(np.sum(wd * E + r2d * dw)) + (ksum + 2) * U * abs(cost)
        K = nb2 * mu * (mu + 1)
        with np.errstate(divide="ignore", invalid="ignore"):
            mid = np.sqrt(LD(K) / r2) - LD(mu)
        w_new = np.where(r2 >= th1, LD(0), np.where(r2 <= th2, LD(1), mid))
        inter = (r2 > th2) & (r2 < th1)
        with np.errstate(divide="ignore", invalid="ignore"):
            dw = np.where(inter, 0.5 * np.sqrt(K / r2d) * (E0 / r2d + 2 * rel_mu) + 4 * U * (mu + 1), 0.0)
        w = w_new
        r2_04 = K / (0.4 + mu) ** 2                 # w = 0.4 <=> r^2 = K / (0.4 + mu)^2
        m.add(np.where(inter, np.abs(r2d - r2_04), np.inf), E + r2_04 * (2 * rel_mu + 8 * U))
        cost_diff = abs(cost - prev)
        thr = p.rotation_cost_threshold
        if math.isfinite(cost_diff) and math.isfinite(thr) and thr > 0:
            m.add(abs(cost_diff - thr), cost_err + cost_err_prev)
        mu = mu * p.rotation_gnc_factor
        prev, cost_err_prev = cost, cost_err
        if cost_diff < thr:
            exit_ = "cost"
            break
    mask = (w >= 0.4).astype(np.uint8)
    return dict(yaw=yaw, eps=eps, iters=iters, mask=mask, n_rot=len(rot_inliers(mask)), cost=cost, exit=exit_, ratio=m.ratio,
                safe=m.ratio > SAFE, nb2=nb2, nn=nn, hn=hn, S=S, mu0=mu, cond0=cond0)


def rot_inliers(mask):
    """quatro.hpp:857-874: member i is a rotation inlier when TIM i-1 and TIM i both are (i = 0 checks TIM c-1)."""
    c = len(mask)
    return [i for i in range(c) if mask[c - 1 if i == 0 else i - 1] and mask[i]]


def _div(a, b):
    if b != 0.0:
        return a / b
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def ref_cote(X, rng, median):
    """Quatro::estimate (quatro.hpp:618-747): events (X - range, +) and (X + range, -) in insertion order, sorted stably by value
    (D3), swept sequentially in Python floats in the reference's operation order; the first minimum of x_cost; the literal "median"
    candidate set h[min_idx - j], j < n_card (upper-end events included), with D5 for n_card <= 1."""
    N = len(X)
    X = [float(v) for v in X]
    vals = []
    for v in X:
        vals += [v - rng, v + rng]
    order = sorted(range(2 * N), key=lambda k: vals[k])
    weight = 1.0 / (rng * rng)
    ris = 0.0
    for _ in range(N):
        ris += rng
    dxw = dwc = sx = sxx = 0.0
    card = min_idx = min_card = 0
    min_cost = min_xhat = 0.0
    cards, dwc_at_zero = [], []
    for k, e in enumerate(order):
        idx, eps = e >> 1, (1 if e % 2 == 0 else -1)
        Xi = X[idx]
        card += eps
        dwc += eps * weight
        dxw += eps * weight * Xi
        ris -= eps * rng
        sx += eps * Xi
        sxx += eps * Xi * Xi
        xh = _div(dxw, dwc)
        cost = card * xh * xh + sxx - 2 * sx * xh + ris
        if k == 0 or cost < min_cost:
            min_cost, min_idx, min_card, min_xhat = cost, k, card, xh
        cards.append(card)
        if card == 0:
            dwc_at_zero.append(dwc)
    est, cand, ambiguous, upper_cand = min_xhat, [], False, False
    if median and min_card > 0:
        ev = [order[min_idx - j] for j in range(min_card)]
        upper_cand = any(e % 2 for e in ev)
        cand = sorted(X[e >> 1] for e in ev)
        n = len(cand)
        mid = [cand[0]] if n == 1 else [cand[n // 2 - 1], cand[n // 2]]
        est = cand[0] if n == 1 else (cand[n // 2 - 1] + cand[n // 2]) / 2.0
        # equal values of different sign (+-0.0) have no defined order in a sort: the sign of a zero median is then unspecified
        zeros = [math.copysign(1.0, v) for v in cand if v == 0.0]
        ambiguous = n > 1 and any(v == 0.0 for v in mid) and len(set(zeros)) > 1
    inl = np.array([abs(v - est) <= rng for v in X], np.uint8)
    ties = [(vals[order[k]] == vals[order[k + 1]]) and (order[k] % 2 != order[k + 1] % 2) for k in range(2 * N - 1)]
    return est, inl, dict(n_card=min_card, min_idx=min_idx, cards=cards, dwc_at_zero=dwc_at_zero, ambiguous=ambiguous,
                          upper_cand=upper_cand, order=order, vals=vals, mixed_tie=ties)


def ref_downstream(a4, b4, clique, p, R, rot_mask):
    """quatro.hpp:857-930 given the implementation's full rotation R (row-major 3 x 3, Rz times the prior) and rotation mask: rotation
    inliers, the COTE inputs X = tgt - (scale R) (RyRx src) [RyRx only in the branch without rotation inliers; (1.0 R) x src summed
    left to right as the kernel does], COTE per axis, the ANDed mask and the final inlier ids."""
    clique = np.asarray(clique, np.int64)
    c = len(clique)
    rl = rot_inliers(rot_mask)
    use_rot = bool(p.using_rot_inliers_when_estimating_cote) and len(rl) > 0
    mem = clique[rl] if use_rot else clique
    s = a4[mem, :3].astype(np.float64)
    b = b4[mem, :3].astype(np.float64)
    sx, sy, sz = s[:, 0].copy(), s[:, 1].copy(), s[:, 2].copy()
    if not use_rot:
        Q = [float(p.RyRx[i]) for i in range(9)] if p.use_pre_estimated_RyRx else [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
        sx, sy, sz = (Q[0] * sx + Q[1] * sy + Q[2] * sz, Q[3] * sx + Q[4] * sy + Q[5] * sz, Q[6] * sx + Q[7] * sy + Q[8] * sz)
    rng = p.cote_noise_bound * math.sqrt(p.cbar2)
    N = len(mem)
    tm = np.ones(N, np.uint8)
    t, X, info = [], [], []
    for ax in range(3):
        r = [float(R[ax][k]) for k in range(3)]
        Xa = b[:, ax] - (1.0 * r[0] * sx + 1.0 * r[1] * sy + 1.0 * r[2] * sz)
        e, inl, d = ref_cote(Xa, rng, p.cote_mode == COTE_MEDIAN)
        t.append(e); X.append(Xa); info.append(d)
        tm &= inl
    tmask = np.zeros(c, np.uint8)
    tmask[:N] = tm
    final = mem[tm.astype(bool)].astype(np.int32)
    return dict(t=np.array(t), tmask=tmask, n_final=len(final), final=final, N=N, use_rot=use_rot, rot_list=rl, X=X, axes=info)


def rotation_of(res):
    return np.array(res.T[:], np.float64).reshape(4, 4).T[:3, :3].copy()


def yaw_of(R, p):
    """Yaw of an implementation's rotation: R = Rz(yaw) RyRx, so Rz = R RyRx^T."""
    Rz = np.asarray(R, LD)
    if p.use_pre_estimated_RyRx:
        Q = np.array([p.RyRx[i] for i in range(9)], LD).reshape(3, 3)
        Rz = Rz @ Q.T
    return np.arctan2(Rz[1, 0], Rz[0, 0])


def yaw_gap(a, b):
    d = (LD(a) - LD(b)) % (2 * LD(np.pi))
    return float(min(d, 2 * LD(np.pi) - d))


# ==== constructions ===========================================================================================================
def _rot_exact(xy, quarter):
    """Rotation by quarter x 90 degrees without rounding."""
    x, y = xy[:, 0].copy(), xy[:, 1].copy()
    for _ in range(quarter % 4):
        x, y = -y, x
    return np.stack([x, y], 1)


def _line(c, resid=None, quarter=0, t=(3.0, -2.0, 1.5), z=None, spacing=0.5, zsrc=None):
    """Source points on the x axis at i * spacing; targets = the source rotated by quarter x 90 degrees plus t, with TIM i displaced
    by resid[i] along the line (sum 0: the chain is cyclic).  Every chain vector and residual is parallel to the line, so
    H01 - H10 = 0 and the yaw is exactly quarter x 90 degrees in every implementation; r_i^2 = resid[i]^2 exactly.  z: target z
    offsets (the z COTE inputs, since R's z row is exactly (0, 0, 1))."""
    r = np.zeros(c) if resid is None else np.asarray(resid, float)
    assert len(r) == c and r.sum() == 0.0
    e = np.concatenate([[0.0], np.cumsum(r[:-1])])
    a = np.zeros((c, 3))
    a[:, 0] = np.arange(c) * spacing
    if zsrc is not None:
        a[:, 2] = zsrc
    b = np.zeros((c, 3))
    b[:, :2] = _rot_exact(np.stack([a[:, 0] + e, np.zeros(c)], 1), quarter) + np.asarray(t[:2])
    b[:, 2] = (a[:, 2] if z is None else np.asarray(z, float)) + t[2]
    a4, b4 = P4(a), P4(b)
    assert np.array_equal(a4[:, :2].astype(float), a[:, :2]) and np.array_equal(b4[:, :2].astype(float), b[:, :2]), "inexact line"
    return a4, b4, np.arange(c)


def _mask_resid(mask, big=4.0):
    """TIM residuals 0 where mask is 1 and +-big elsewhere, summing to 0."""
    out = [i for i, v in enumerate(mask) if not v]
    assert len(out) != 1
    vals = [big, -big] * ((len(out) - 3) // 2) + [big, big, -2 * big] if len(out) % 2 else [big, -big] * (len(out) // 2)
    r = np.zeros(len(mask))
    r[out] = vals
    return r


def _Rz(deg):
    t = np.deg2rad(deg)
    return np.array([[np.cos(t), -np.sin(t), 0], [np.sin(t), np.cos(t), 0], [0, 0, 1]])


def _Ry(deg):
    t = np.deg2rad(deg)
    return np.array([[np.cos(t), 0, np.sin(t)], [0, 1, 0], [-np.sin(t), 0, np.cos(t)]])


def _scene(seed, c, L=None, yaw=None, outliers=0.3, noise=0.02, t=(12.0, -7.0, 1.0), extent=40.0, prior=None):
    """Random matched pairs: inliers b = Rz(yaw) prior a + t + noise, outliers uniform; the clique is a sorted random c-subset of L."""
    rng = np.random.default_rng(seed)
    L = L or c
    yaw = rng.uniform(-180, 180) if yaw is None else yaw
    a = rng.uniform(-extent, extent, (L, 3)) * [1, 1, 0.1]
    Rf = _Rz(yaw) @ (np.eye(3) if prior is None else prior)
    b = a @ Rf.T + np.asarray(t) + rng.normal(0, noise, (L, 3))
    out = rng.random(L) < outliers
    b[out] = rng.uniform(-extent, extent, (int(out.sum()), 3)) * [1, 1, 0.1] + np.asarray(t)
    clique = np.sort(rng.choice(L, c, replace=False))
    return P4(a), P4(b), clique


def _near_reflection(seed, n=64, eta=2.0 ** -20):
    """Sources in four-fold symmetric dyadic sets (sum x x^T = s I exactly); targets = a reflection plus eta x a rotation: H is a
    reflection-like matrix with ||(cc, ss)|| ~ eta ||H||."""
    rng = np.random.default_rng(seed)
    v = rng.integers(-512, 512, (n, 2)) / 64.0
    pts = np.concatenate([v, _rot_exact(v, 1), _rot_exact(v, 2), _rot_exact(v, 3)])
    a = np.concatenate([pts, np.zeros((len(pts), 1))], 1)
    refl = pts * [1, -1]
    b = np.concatenate([refl + eta * (pts @ _Rz(37.0)[:2, :2].T), np.zeros((len(pts), 1))], 1)
    return P4(a), P4(b), np.arange(len(pts))


def _zero_chain(seed):
    a4, b4, _ = _scene(seed, 80, outliers=0.2)
    a4[21], b4[21] = a4[20], b4[20]                        # coincident members
    clique = np.sort(np.concatenate([np.arange(0, 60), [5, 5, 17]]))   # repeated members
    return a4, b4, clique


def _degenerate_h():
    """The unit square onto its mirror image across the diagonal: H = 2 [[0, 1], [1, 0]], cc = ss = 0."""
    a = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], float)
    b = a[:, [1, 0, 2]] + [5.0, -3.0, 0.5]
    return P4(a), P4(b), np.arange(4)


def _median_cluster(k, n_iso=40, seed=0, spread=0.1):
    """z COTE inputs: k members within +-spread (every interval overlaps every other) and n_iso members 0.75 apart (> 2 range):
    the optimum is the cluster with n_card = k (k = 1: every member isolated)."""
    rng = np.random.default_rng(seed)
    cl = rng.uniform(-spread, spread, k) if k > 1 else np.zeros(0)
    iso = 1.0 + 0.75 * np.arange(n_iso if k > 1 else n_iso + 1)
    z = np.concatenate([cl, iso]).astype(np.float32).astype(float)
    perm = rng.permutation(len(z))
    return _line(len(z), z=z[perm])


def _signed_zero():
    a4, b4, cl = _line(24, t=(0.0, 0.0, 0.0))
    b4[::2, 2] = -0.0
    b4[::3, 1] = -0.0
    return a4, b4, cl


def _far(seed, off):
    return _scene(seed, 300, L=340, yaw=31.0, outliers=0.2, t=(off, -off, 30.0), extent=50.0)


RANGE025 = dict(cote_noise_bound=0.25)
LINE_OUT = [1, 1, 1, 0, 1, 1, 1, 1, 0, 0, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1]
CASES = {
    # sizes (random scenes, 30 % outliers)
    **{f"size{c}": (lambda c=c: _scene(100 + c, c, L=min(c + c // 7 + 1, 8192) if c <= 8192 else c), {}) for c in
       (2, 3, 31, 32, 33, 255, 256, 257, 4095, 4096, 4097, 32768)},
    # GNC
    "noisefree_yaw0": (lambda: _line(33), {}),
    "noisefree_yaw90": (lambda: _line(33, quarter=1), {}),
    "noisefree_yaw180": (lambda: _line(33, quarter=2), {}),
    "maxr2_below": (lambda: _line(32, [0.5, -0.5] + [0.0] * 30), dict(rot_noise_bound=math.sqrt(2 * 0.25 / (1 - 2.0 ** -20)))),
    "maxr2_above": (lambda: _line(32, [0.5, -0.5] + [0.0] * 30), dict(rot_noise_bound=math.sqrt(2 * 0.25 / (1 + 2.0 ** -20)))),
    "max_iterations0": (lambda: _line(32, _mask_resid(LINE_OUT)), dict(rotation_max_iterations=0)),
    "max_iterations1": (lambda: _line(32, _mask_resid(LINE_OUT)), dict(rotation_max_iterations=1)),
    "cost_threshold0": (lambda: _line(32, _mask_resid(LINE_OUT)), dict(rotation_cost_threshold=0.0, rotation_max_iterations=20)),
    "cost_threshold_inf": (lambda: _line(32, _mask_resid(LINE_OUT)), dict(rotation_cost_threshold=math.inf)),
    "gnc_factor1": (lambda: _line(32, _mask_resid(LINE_OUT)), dict(rotation_gnc_factor=1.0, rotation_max_iterations=12)),
    "gnc_factor1.0001": (lambda: _line(32, _mask_resid(LINE_OUT)), dict(rotation_gnc_factor=1.0001)),
    "gnc_factor100": (lambda: _line(32, _mask_resid(LINE_OUT)), dict(rotation_gnc_factor=100.0)),
    "rot_noise_bound1e-9": (lambda: _line(32, _mask_resid(LINE_OUT, big=0.25)), dict(rot_noise_bound=1e-9)),
    "outliers0": (lambda: _scene(7, 600, outliers=0.0), {}),
    "outliers50": (lambda: _scene(8, 600, outliers=0.5), {}),
    "outliers90": (lambda: _scene(9, 600, outliers=0.9), {}),
    "yaw+179.99": (lambda: _scene(10, 300, yaw=179.99, outliers=0.1), {}),
    "yaw-179.99": (lambda: _scene(11, 300, yaw=-179.99, outliers=0.1), {}),
    "near_reflection": (lambda: _near_reflection(12), {}),
    "zero_chain": (lambda: _zero_chain(13), {}),
    # COTE
    "cote_all_equal": (lambda: _line(40, t=(2.5, -1.25, 0.75)), {}),
    "cote_z_2range": (lambda: _line(33, z=0.5 * np.arange(33)), RANGE025),
    "cote_tie_at_optimum": (lambda: _line(5, z=[0.0, 0.5, 0.5, 0.5, 3.0]), RANGE025),
    "cote_x_2range": (lambda: _line(16, [0.5] * 15 + [-7.5], spacing=1.0), dict(rot_noise_bound=20.0, **RANGE025)),
    "cote_range0.3_residue": (lambda: _line(30, z=np.repeat([0.0, 0.1, 0.2, 5.0, 5.1, 5.2, 9.0, 9.05, 9.1, 9.15], 3)[:30]), {}),
    "cote_signed_zero": (_signed_zero, {}),
    "cote_far_4e5": (lambda: _far(14, 4e5), {}),
    "cote_far_5e6": (lambda: _far(15, 5e6), {}),
    "median_upper_event": (lambda: _line(4, z=[0.0, 1.9, 1.9, 1.9]), dict(cote_noise_bound=1.0)),
    **{f"median_card{k}": (lambda k=k: _median_cluster(k, seed=k), RANGE025) for k in (1, 2, 255, 256, 257, 4100)},
    # rotation-inlier COTE
    "rot_inliers_none": (lambda: _line(16, _mask_resid([1, 0] * 8)), dict(using_rot_inliers_when_estimating_cote=1)),
    "rot_inliers_one": (lambda: _line(16, _mask_resid([0] * 5 + [1, 1] + [0] * 9)), dict(using_rot_inliers_when_estimating_cote=1)),
    "rot_inliers_all": (lambda: _line(16), dict(using_rot_inliers_when_estimating_cote=1)),
    "rot_inliers_wrap": (lambda: _line(20, _mask_resid([1, 1] + [0] * 5 + [1, 1, 1] + [0] * 8 + [1, 1])),
                         dict(using_rot_inliers_when_estimating_cote=1)),
    # RyRx prior, both branches
    "ryrx20": (lambda: _scene(16, 400, outliers=0.3, prior=_Ry(20.0) @ _Rz(0)), dict(RyRx=_Ry(20.0))),
    "ryrx20_rot_inliers": (lambda: _scene(16, 400, outliers=0.3, prior=_Ry(20.0)), dict(RyRx=_Ry(20.0), using_rot_inliers_when_estimating_cote=1)),
}
ILL_CONDITIONED = {"near_reflection"}
MODES = {"median": COTE_MEDIAN, "mean": COTE_WEIGHTED_MEAN}
_cache = {}


def case(name, mode="median"):
    key = (name, mode)
    if key not in _cache:
        build, kw = CASES[name]
        a4, b4, clique = build()
        p = _prm(**kw)
        p.cote_mode = MODES[mode]
        x, y = chain_tims(a4, b4, clique)
        _cache[key] = (a4, b4, np.asarray(clique, np.int32), p, dict(dev=ref_gnc(x, y, p, "device"), ora=ref_gnc(x, y, p, "oracle")))
    return _cache[key]


CASE_IDS = list(CASES)
CPU_KEYS = [(n, m) for n in CASES for m in MODES]
CPU_IDS = [f"{n}-{m}" for n, m in CPU_KEYS]


# ==== edge assertions =========================================================================================================
def check_edges(name, a4, b4, clique, p, g, d):
    """The construction `name` hits its edge: g = the exact GNC restatement, d = the downstream restatement (median mode, given the
    oracle's R and rotation mask)."""
    c = len(clique)
    z = d["axes"][2]
    if name.startswith("size"):
        assert c == int(name[4:]) and g["iters"] >= 1 and g["eps"] <= WELL_CONDITIONED
        if c == 32768:
            assert d["axes"][0]["n_card"] > 4096
    elif name.startswith("noisefree"):
        q = {"yaw0": 0, "yaw90": 1, "yaw180": 2}[name.split("_")[1]]
        assert g["exit"] == "mu" and g["iters"] == 1 and g["cost"] == math.inf and g["mask"].all()
        want = [np.arctan2(LD(0), LD(1)), np.arctan2(LD(1), LD(0)), np.arctan2(LD(0), LD(-1))][q]
        assert yaw_gap(g["yaw"], want) == 0.0 and g["safe"]
    elif name == "maxr2_below":
        assert g["exit"] == "mu" and g["iters"] == 1 and -2.0 ** -19 < float(g["mu0"]) ** -1 < 0 and g["safe"]
    elif name == "maxr2_above":
        assert g["exit"] != "mu" and g["iters"] > 1 and 0 < float(g["mu0"]) ** -1 < 2.0 ** -19 and g["safe"]
    elif name == "max_iterations0":
        assert g["iters"] == 0 and g["mask"].all() and g["cost"] == math.inf
    elif name == "max_iterations1":
        assert g["iters"] == 1 and g["exit"] == "max_iterations"
    elif name == "cost_threshold0":
        assert g["iters"] == 20 and g["exit"] == "max_iterations"
    elif name == "cost_threshold_inf":
        assert g["iters"] == 2 and g["exit"] == "cost"            # inf - inf is not < inf at iteration 0
    elif name.startswith("gnc_factor"):
        assert g["safe"] and g["exit"] in ("cost", "max_iterations") and g["iters"] >= 2
    elif name == "rot_noise_bound1e-9":
        assert g["nb2"] == 1e-2 and list(g["mask"]) == LINE_OUT
    elif name.startswith("outliers"):
        frac = int(name[8:]) / 100
        assert g["exit"] == "mu" if frac == 0 else g["n_rot"] < (1.2 - frac) * c
    elif name.startswith("yaw"):
        assert abs(abs(float(g["yaw"])) - np.deg2rad(179.99)) < 1e-3
    elif name == "near_reflection":
        assert 0 < g["cond0"] < 1e-4                                # ||(cc, ss)|| / ||H|| at iteration 0
    elif name == "zero_chain":
        x, y = chain_tims(a4, b4, clique)
        assert (np.hypot(*x.T) == 0).sum() >= 4
    elif name == "cote_all_equal":
        assert all(len(set(X.tolist())) == 1 for X in d["X"]) and all(ax["n_card"] == c for ax in d["axes"])
    elif name == "cote_z_2range":
        assert any(z["mixed_tie"]) and 0 in z["cards"][:-1]            # consensus returns to 0 before the last event
    elif name == "cote_tie_at_optimum":
        k, ev = z["min_idx"], z["order"]
        v = z["vals"][ev[k]]
        assert any(z["vals"][e] == v and e % 2 != ev[k] % 2 for e in ev), "a lower and an upper event tie at the optimum"
        assert z["n_card"] == 3 and 0 in z["cards"][:k]
    elif name == "cote_x_2range":
        x = d["axes"][0]
        assert any(x["mixed_tie"]) and 0 in x["cards"][:-1]
    elif name == "cote_range0.3_residue":
        assert any(v != 0.0 for v in z["dwc_at_zero"][:-1]), "dot_weights_consensus leaves a residue at card 0"
    elif name == "cote_signed_zero":
        assert any(math.copysign(1, v) < 0 for v in d["X"][2]) and any(math.copysign(1, v) > 0 for v in d["X"][2])
    elif name.startswith("cote_far"):
        assert np.abs(b4[:, 0]).min() > 3e5
    elif name == "median_upper_event":
        assert z["upper_cand"] and z["n_card"] == 3
    elif name.startswith("median_card"):
        assert z["n_card"] == int(name[11:])
    elif name.startswith("rot_inliers"):
        n_rot = len(rot_inliers(g["mask"]))
        want = {"none": 0, "one": 1, "all": c, "wrap": 5}[name.split("_")[2]]
        assert n_rot == want and d["N"] == (c if want == 0 else want)
        if name.endswith("wrap"):
            assert rot_inliers(g["mask"]) == [0, 1, 8, 9, 19]
    elif name.startswith("ryrx"):
        assert d["use_rot"] == name.endswith("rot_inliers") and g["eps"] <= WELL_CONDITIONED


def check_downstream(d, T, tmask, n_final, final):
    """Bit-identical translation (== where a zero median has no defined sign), trans_mask (zeros past N), count and list."""
    t = np.array(T[12:15], np.float64)
    for ax in range(3):
        if d["axes"][ax]["ambiguous"]:
            assert t[ax] == d["t"][ax] == 0.0, ax
        else:
            assert t[ax:ax + 1].tobytes() == d["t"][ax:ax + 1].tobytes(), (ax, t[ax], d["t"][ax])
    assert np.asarray(tmask, np.uint8).tobytes() == d["tmask"].tobytes()
    assert n_final == d["n_final"]
    assert np.asarray(final, np.int32).tobytes() == d["final"].tobytes()


# ==== CPU =====================================================================================================================
@pytest.mark.parametrize("name", CASE_IDS)
def test_pose_constructions_hit_their_edges(oracle, name):
    a4, b4, clique, p, g = case(name)
    res, rm, _, st = oracle.solve_pose(a4, b4, clique, p)
    assert st == 0
    d = ref_downstream(a4, b4, clique, p, rotation_of(res), rm)
    check_edges(name, a4, b4, clique, p, g["dev"], d)


@pytest.mark.parametrize("key", CPU_KEYS, ids=CPU_IDS)
def test_oracle_matches_float64_restatement(oracle, key):
    a4, b4, clique, p, g = case(*key)
    go = g["ora"]
    res, rm, tm, st, fin = oracle.solve_pose(a4, b4, clique, p, want_final=True)
    assert st == 0 and res.valid == 1
    R = rotation_of(res)
    if go["iters"] and go["eps"] < math.inf:
        assert yaw_gap(yaw_of(R, p), go["yaw"]) <= go["eps"], (yaw_gap(yaw_of(R, p), go["yaw"]), go["eps"])
    if go["safe"]:
        assert res.gnc_iters == go["iters"]
        assert rm.tobytes() == go["mask"].tobytes()
        assert res.n_rot_inliers == go["n_rot"]
    d = ref_downstream(a4, b4, clique, p, R, rm)
    assert res.n_rot_inliers == len(d["rot_list"])
    check_downstream(d, res.T[:], tm, res.n_final_inliers, fin)


def test_restated_cote_matches_oracle_on_raw_inputs(oracle):
    """The COTE restatement against qo_test_cote directly, on inputs with ties, gaps and card-0 residues."""
    rng = np.random.default_rng(5)
    sets = [np.repeat([0.0, 0.1, 0.2, 5.0, 5.1, 5.2, 9.0, 9.05], 3), 0.5 * np.arange(40), np.zeros(17), [0.0, 1.9, 1.9, 1.9],
            rng.normal(0, 0.2, 301), np.round(rng.normal(0, 1, 500), 1), [3.0]]
    for X in sets:
        X = np.asarray(X, np.float64)
        for rng_ in (0.25, 0.3, 1.0):
            for median in (True, False):
                e, inl = oracle.cote(X, rng_, median)
                e2, inl2, _ = ref_cote(X, rng_, median)
                assert np.float64(e).tobytes() == np.float64(e2).tobytes() and np.array_equal(inl, inl2.astype(bool))


def test_degenerate_h_every_yaw_is_a_maximiser(oracle):
    """cc = ss = 0 with H != 0: trace(R H) is the same for every R.  The oracle's Jacobi SVD gives some rotation; both attain the
    maximum, and downstream of R the oracle still matches the restatement bit for bit."""
    a4, b4, clique = _degenerate_h()
    p = _prm()
    x, y = chain_tims(a4, b4, clique)
    H = x.T @ y
    assert H[0, 0] + H[1, 1] == 0 and H[0, 1] - H[1, 0] == 0 and np.abs(H).max() > 0
    res, rm, tm, st, fin = oracle.solve_pose(a4, b4, clique, p, want_final=True)
    R = rotation_of(res)
    assert st == 0 and abs(np.trace(R[:2, :2] @ H)) <= 1e-12
    D = np.array([[0.0, 1.0], [1.0, 0.0]])
    Ro = oracle.svd_rot2d(np.eye(2), D, np.ones(2))            # H = D: the Jacobi restatement picks -I, also a maximiser
    assert np.allclose(Ro, -np.eye(2), rtol=0, atol=1e-15) and abs(np.trace(Ro @ D)) <= 1e-15
    check_downstream(ref_downstream(a4, b4, clique, p, R, rm), res.T[:], tm, res.n_final_inliers, fin)


def test_stage_call_status_for_tiny_inputs(oracle):
    """Fewer than two correspondences is DEGENERATE_INPUT, a clique of <= 1 member otherwise DEGENERATE_CLIQUE: as
    solve_correspondences and the device report them."""
    a4, b4, _ = _line(3)
    assert oracle.solve_pose(a4[:1], b4[:1], [0], _prm())[3] == 2
    assert oracle.solve_pose(a4[:0], b4[:0], [], _prm())[3] == 2
    assert oracle.solve_pose(a4, b4, [1], _prm())[3] == 1
    assert oracle.solve_pose(a4, b4, [], _prm())[3] == 1


# ==== GPU =====================================================================================================================
@pytest.fixture(scope="module")
def h8k():
    with Handle(max_batch_slots=1, max_corr=8192) as h:
        yield h


@pytest.fixture(scope="module")
def h32k():
    with Handle(max_batch_slots=1, max_corr=32768) as h:     # one slot: about 256 MB
        yield h


def _device_checks(h, a4, b4, clique, p, g):
    res, rm, tm, st = h.solve_pose(a4, b4, clique, p)
    assert st == 0 and res.valid == 1
    R = rotation_of(res)
    if g["iters"] and g["eps"] < math.inf:
        assert yaw_gap(yaw_of(R, p), g["yaw"]) <= g["eps"], (yaw_gap(yaw_of(R, p), g["yaw"]), g["eps"])
    if g["safe"]:
        assert (res.gnc_iters, res.n_rot_inliers) == (g["iters"], g["n_rot"])
        assert rm.tobytes() == g["mask"].tobytes()
    d = ref_downstream(a4, b4, clique, p, R, rm)
    assert res.n_rot_inliers == len(d["rot_list"])
    check_downstream(d, res.T[:], tm, res.n_final_inliers, h.last_final_inliers())
    return res, rm, tm


@pytest.mark.gpu
@pytest.mark.parametrize("key", CPU_KEYS, ids=CPU_IDS)
def test_device_pose_matches_float64_restatement(request, oracle, key):
    a4, b4, clique, p, g = case(*key)
    h = request.getfixturevalue("h32k" if len(a4) > 8192 else "h8k")
    g = g["dev"]
    if key[0] not in ILL_CONDITIONED and g["iters"]:
        assert g["eps"] <= WELL_CONDITIONED, g["eps"]
    res, rm, tm = _device_checks(h, a4, b4, clique, p, g)
    ro, rmo, _, _ = oracle.solve_pose(a4, b4, clique, p)
    if g["safe"] and case(*key)[4]["ora"]["safe"]:
        assert (res.gnc_iters, res.n_rot_inliers) == (ro.gnc_iters, ro.n_rot_inliers) and rm.tobytes() == rmo.tobytes()


@pytest.mark.gpu
def test_device_degenerate_h_returns_the_identity(h8k):
    a4, b4, clique = _degenerate_h()
    p = _prm()
    res, rm, tm, st = h8k.solve_pose(a4, b4, clique, p)
    assert st == 0 and np.array_equal(rotation_of(res), np.eye(3))
    check_downstream(ref_downstream(a4, b4, clique, p, rotation_of(res), rm), res.T[:], tm, res.n_final_inliers, h8k.last_final_inliers())


@pytest.mark.gpu
def test_device_tiny_inputs_and_out_of_range_cliques(h8k):
    a4, b4, clique, p, g = case("size33")
    want = h8k.solve_pose(a4, b4, clique, p)
    want_fin = h8k.last_final_inliers()
    L = len(a4)
    for bad in ([0, 1, L], [-1, 2, 3], [0, 2**31 - 1]):
        with pytest.raises(QuatroB200Error) as e:
            h8k.solve_pose(a4, b4, bad, p)
        assert e.value.code == -1
    got = h8k.solve_pose(a4, b4, clique, p)
    assert bytes(got[0]) == bytes(want[0]) and got[1].tobytes() == want[1].tobytes() and got[2].tobytes() == want[2].tobytes()
    assert h8k.last_final_inliers().tobytes() == want_fin.tobytes()
    a3, b3, _ = _line(3)
    assert h8k.solve_pose(a3[:1], b3[:1], [0], p)[3] == 2
    assert h8k.solve_pose(a3, b3, [1], p)[3] == 1


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", ["1", "4"])
def test_mixed_adversarial_wave_equals_single_calls(monkeypatch, lanes):
    """Every case of at most 8192 members as one INLIER_NONE set (the clique is every correspondence) in one qb200_solve_batch_each on
    a max_corr = 8192 handle, cliques on both sides of the 4096 switch, each with its own COTE mode, rotation-inlier, RyRx and GNC
    knobs: every record and list byte-identical to qb200_solve_correspondences / qb200_solve_pose on that set alone."""
    monkeypatch.setenv("QB200_LANES", lanes)
    sets, params = [], []
    for i, name in enumerate(CASES):
        a4, b4, clique, p, _ = case(name, "median" if i % 2 else "mean")
        if len(clique) > 8192:
            continue
        q = Params.from_buffer_copy(p)
        q.inlier_selection_mode = INLIER_NONE
        sets.append((np.ascontiguousarray(a4[clique]), np.ascontiguousarray(b4[clique])))
        params.append(q)
    assert any(len(s[0]) > 4096 for s in sets) and any(len(s[0]) <= 4096 for s in sets)
    with Handle(max_batch_slots=4, max_corr=8192) as h:
        recs, lists = h.solve_batch_each(sets, params, buffers=ListBuffers(len(sets), 8192, MEM_HOST, SET_LISTS))
        for i, ((a4, b4), q) in enumerate(zip(sets, params)):
            r1, st = h.solve_correspondences(a4, b4, q)
            assert recs[i].tobytes() == bytes(r1), i
            assert lists[i]["final_inliers"].tobytes() == h.last_final_inliers().tobytes(), i
            assert lists[i]["clique"].tobytes() == np.arange(len(a4), dtype=np.int32).tobytes()
            r2, rm, tm, _ = h.solve_pose(a4, b4, np.arange(len(a4)), q)
            assert lists[i]["rot_inlier_mask"].tobytes() == rm.tobytes() and lists[i]["trans_inlier_mask"].tobytes() == tm.tobytes(), i
            assert np.array(r2.T[:]).tobytes() == recs[i]["T"].tobytes() and r2.gnc_iters == recs[i]["gnc_iters"]
