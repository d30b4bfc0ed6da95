"""NumPy restatement of rtti_kmeans_fit (csrc/kmeans.cu): the same algorithm and the same float32 / float64 roundings,
so the CPU tests can run rtti_b200.attention_utils.spectral_clustering without a GPU and compare it with scikit-learn.

The kernel's float32 fused multiply-adds are rounded once from float64 here; float64 fmas are a multiply and an add.
"""
import math

import numpy as np

f32 = np.float32
# number of Lloyd steps that relocated an empty cluster (dmax > 0), for tests that must reach that branch
RELOCATIONS = 0


def _fma32(a, b, c):
    return (a.astype(np.float64) * b + c).astype(f32)


def _upcast_sqdist(X, rows, X64):
    """[len(rows), n] float64 -2 a.b + |a|^2 + |b|^2, clipped at 0, as float32."""
    a = X64[rows]
    d = -2.0 * (a @ X64.T)
    d += (a * a).sum(1)[:, None]
    d += (X64 * X64).sum(1)[None, :]
    return np.maximum(d, 0.0).astype(f32)


def _assign(X, cen):
    k = cen.shape[0]
    cn = np.zeros(k, f32)
    for f in range(k):
        cn = (cn + cen[:, f] * cen[:, f]).astype(f32)
    acc = np.zeros((X.shape[0], k), f32)
    for f in range(X.shape[1]):
        acc = _fma32(X[:, f:f + 1], cen[None, :, f], acc)
    d = _fma32(np.full_like(acc, -2.0), acc, cn[None, :])
    return d.argmin(1).astype(np.int32)


def _rowdist(X, cen, lab):
    a = np.zeros(X.shape[0], f32)
    for f in range(X.shape[1]):
        d = (X[:, f] - cen[lab, f]).astype(f32)
        a = (a + d * d).astype(f32)
    return a


def _fit_one(X, X64, dr, T, max_iter, tol_abs):
    n, k = X.shape
    c0 = int(dr[0])
    cen = np.empty((k, k), f32)
    cen[0] = X[c0]
    closest = _upcast_sqdist(X, [c0], X64)[0]
    pot = f32(closest.astype(np.float64).sum())
    for c in range(1, k):
        rv = dr[1 + (c - 1) * T:1 + c * T] * np.float64(pot)
        cum = np.cumsum(closest, dtype=f32)
        cand = np.minimum(np.searchsorted(cum.astype(np.float64), rv, side="left"), n - 1)
        dc = np.minimum(closest[None, :], _upcast_sqdist(X, cand, X64))
        pots = dc.astype(np.float64).sum(1).astype(f32)
        b = int(np.argmin(pots))
        closest, pot = dc[b], pots[b]
        cen[c] = X[cand[b]]
    lab = np.full(n, -1, np.int32)
    strict = False
    flag = 0
    for it in range(max_iter):
        new = _assign(X, cen)
        changed = not np.array_equal(new, lab)
        lab = new
        sums = np.zeros((k, k))
        cnt = np.bincount(lab, minlength=k).astype(np.float64)
        np.add.at(sums, lab, X.astype(np.float64))
        if (cnt == 0).any():
            dist = _rowdist(X, cen, lab)
            if dist.max() > 0:
                global RELOCATIONS
                RELOCATIONS += 1
                if (cnt == 0).sum() > 1:
                    flag = 1
                for j in np.flatnonzero(cnt == 0):
                    far = int(np.argmax(dist))
                    tied = np.flatnonzero(dist == dist[far])
                    if (X[tied] != X[far]).any():
                        flag = 1
                    dist[far] = -1
                    old = lab[far]
                    sums[old] -= X[far]
                    sums[j] = X[far]
                    cnt[j] = 1
                    cnt[old] -= 1
        w = cnt.astype(f32)
        cnew = sums.astype(f32)
        amax = int(np.argmax(w))
        for j in range(k):   # one pass in cluster order, as _average_centers
            if w[j] > 0:
                cnew[j] = cnew[j] * (f32(1) / w[j])
            else:
                cnew[j] = cnew[amax]
        shift = f32(0)
        for j in range(k):
            sh = np.sqrt(_rowdist(cnew[j:j + 1], cen[j:j + 1], np.zeros(1, np.int32))[0])
            shift = f32(shift + sh * sh)
        cen = cnew
        if not changed:
            strict = True
            break
        if shift <= tol_abs:
            break
    if not strict:
        lab = _assign(X, cen)
    return lab, float(_rowdist(X, cen, lab).astype(np.float64).sum()), it + 1, flag


def kmeans_fit(x, draws, max_iter=300, tol=1e-4):
    """Same contract as rtti_b200.ops.kmeans_fit on numpy arrays: (labels [n_init, n] int32, inertia [n_init] float64,
    n_iter [n_init] int32, flags [n_init] int32)."""
    X = np.ascontiguousarray(x, dtype=f32)
    n, k = X.shape
    T = 2 + int(math.log(k))
    a = np.zeros(k, f32)
    for i in range(n):
        a = (a + X[i]).astype(f32)
    m = (a / f32(n)).astype(f32)
    v = np.zeros(k, f32)
    for i in range(n):
        d = (X[i] - m).astype(f32)
        v = (v + d * d).astype(f32)
    var = (v / f32(n)).astype(f32)
    va = f32(0)
    for f in range(k):
        va = f32(va + var[f])
    tol_abs = f32(f32(va / f32(k)) * f32(tol))
    X = (X - m).astype(f32)
    X64 = X.astype(np.float64)
    out = [_fit_one(X, X64, np.asarray(d, np.float64), T, max_iter, tol_abs) for d in draws]
    return (np.stack([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out], np.int32),
            np.array([o[3] for o in out], np.int32))
