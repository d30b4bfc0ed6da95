"""Spectral clustering of the token maps on the device (attention_utils.spectral_clustering, rtti_kmeans_fit) against
scikit-learn: bit-equal segment labels and the same NumPy RNG state afterwards.

CPU tests run the product's draws, embedding and restart selection with the NumPy restatement of the kernel
(tests/kmeans_emu.py); GPU tests run the kernel."""
import ctypes
import warnings

import numpy as np
import pytest
import torch

from tests import kmeans_emu, synth

warnings.filterwarnings("ignore", module="sklearn")

N_INIT = 100


def _blobs(n, k, seed, kind):
    g = np.random.default_rng(seed)
    c = g.normal(size=(max(k, 2), k)) * 3
    x = c[g.integers(0, len(c), n)] + g.normal(size=(n, k))
    if kind == "aniso":
        x = x @ g.normal(size=(k, k))
    if kind == "dup":   # n/8 distinct rows: exact distance ties
        x = x[g.integers(0, n // 8, n)]
    if kind == "few":   # fewer distinct rows than clusters: duplicate seeds, several clusters empty at once
        x = x[g.integers(0, k // 2 + 1, n)]
    return x.astype(np.float32)


# (n, k) pairs whose embedding fits the kernel's shared memory
KMEANS_CASES = [(n, k, kind) for n in (257, 1024, 4096) for k in (1, 2, 5, 9, 16, 32)
                for kind in ("gauss", "aniso", "dup")
                if 4 * n * (k + 2) + 18 * 1024 <= 227 * 1024]


def _same_state(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a.get_state(), b.get_state()))


def _inertia_close(got, ref, x, tol):
    """Relative to the data's total sum of squares, so clusterings whose inertia is rounding noise compare too.
    scikit-learn sums the inertia in float32 in an OpenMP-thread-dependent order (about sqrt(n) * 6e-8 relative), so
    1e-5 is the tightest tolerance that holds for its own result from run to run."""
    scale = float(((x - x.mean(0)) ** 2).sum())
    return abs(got - ref) <= tol * max(ref, scale * 1e-3)


def _kmeans_case(n, k, kind, fit):
    from sklearn.cluster import KMeans
    from rtti_b200.attention_utils import kmeans_draws, select_restart
    x = _blobs(n, k, n + k, kind)
    rs_ref, rs = np.random.RandomState(k), np.random.RandomState(k)
    km = KMeans(k, n_init=N_INIT, random_state=rs_ref).fit(x)
    labels, inertia, _, flags = fit(x, kmeans_draws(rs, n, k, N_INIT))
    assert not flags.any()
    b = select_restart(labels, inertia, k)
    return x, km, labels[b], inertia[b], _same_state(rs, rs_ref)


@pytest.mark.parametrize("n,k,kind", [c for c in KMEANS_CASES if c[0] <= 1024])
def test_kmeans_restatement_matches_sklearn(n, k, kind):
    x, km, labels, inertia, same_state = _kmeans_case(n, k, kind, kmeans_emu.kmeans_fit)
    assert np.array_equal(labels, km.labels_)
    assert same_state
    assert _inertia_close(inertia, km.inertia_, x, 1e-5)


def test_kmeans_restatement_relocates_empty_clusters_like_sklearn():
    """Blobs whose Lloyd iterations empty a cluster while samples lie off their centres (the relocation branch of
    _relocate_empty_clusters_dense, one cluster at a time): labels still equal scikit-learn's."""
    kmeans_emu.RELOCATIONS = 0
    x, km, labels, _, same_state = _kmeans_case(257, 32, "gauss", kmeans_emu.kmeans_fit)
    assert kmeans_emu.RELOCATIONS > 0
    assert np.array_equal(labels, km.labels_) and same_state


def kmeans_draws_for(n, k):
    from rtti_b200.attention_utils import kmeans_draws
    return kmeans_draws(np.random.RandomState(k), n, k, 10)


def test_ambiguous_relocation_is_flagged_and_handed_to_sklearn():
    """Two clusters emptied in one Lloyd step: scikit-learn fills them in np.argpartition's unspecified order, so the
    restart is flagged, and spectral_clustering rewinds the RNG and returns scikit-learn's labels."""
    from rtti_b200 import attention_utils as au
    # all-zero uniforms make k-means++ pick index 0 again (searchsorted(cumsum, 0) == 0): three equal seeds, so the
    # first Lloyd step leaves clusters 1 and 2 empty at once; with two equal seeds only one, which is unambiguous
    x = np.random.default_rng(0).normal(size=(64, 3)).astype(np.float32)
    assert kmeans_emu.kmeans_fit(x, np.zeros((1, 7)))[3][0] == 1
    assert kmeans_emu.kmeans_fit(x[:, :2], np.zeros((1, 3)))[3][0] == 0
    # fewer distinct rows than clusters: float32 cluster means drift off the duplicated seeds, so scikit-learn
    # relocates several clusters at once as well
    assert kmeans_emu.kmeans_fit(_blobs(257, 9, 266, "few"), kmeans_draws_for(257, 9))[3].any()
    aff = _soft_blobs(0)
    calls = []

    def flagged_fit(emb, d):
        calls.append(1)
        out = _emu_fit(emb, d)
        return out[:3] + (np.ones_like(out[3]),)
    got, ref, same_state = _spectral_case(aff, 6, kmeans_fit=flagged_fit)
    assert calls and np.array_equal(got, ref) and same_state


def test_kernel_shapes_outside_its_limits_go_to_sklearn():
    """k > 32 (e.g. --num_segments 40) keeps scikit-learn's result instead of raising."""
    aff = _soft_blobs(1)

    def no_kernel(*a):
        raise AssertionError("k-means kernel called outside its shape limits")
    got, ref, same_state = _spectral_case(aff, 40, kmeans_fit=no_kernel)
    assert np.array_equal(got, ref) and same_state


def _soft_blobs(seed, n_blobs=6, temp=0.05):
    g = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.arange(32), np.arange(32), indexing="ij")
    pts = np.stack([yy, xx], -1).reshape(-1, 2) / 32.0
    cen = g.uniform(0, 1, (n_blobs, 2))
    feat = np.exp(-((pts[:, None] - cen[None]) ** 2).sum(-1) / 0.02)
    feat = feat / feat.sum(1, keepdims=True)
    logits = feat @ feat.T / temp
    a = np.exp(logits - logits.max(1, keepdims=True))
    return torch.from_numpy((a / a.sum(1, keepdims=True)).astype(np.float32))


def _near_uniform(seed, eps, groups=4):
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, groups, (1024,), generator=g)
    a = torch.ones(1024, 1024) + eps * (lab[:, None] == lab[None, :]).float() + 1e-7 * torch.rand(1024, 1024, generator=g)
    return a / a.sum(1, keepdim=True)


def _synth_affinity(seed):
    from rtti_b200.attention_utils import self_affinity
    return self_affinity(synth.synth_maps(seed)[0])


SPECTRAL_CASES = ([("synth", s, k) for s in range(4) for k in (4, 5, 9)]
                  + [("soft", s, k) for s in (0, 1, 2) for k in range(2, 13)]
                  + [("uniform", 1e-2, 4), ("uniform", 1e-3, 4), ("uniform", 1e-4, 9)])


def _affinity(kind, arg):
    return {"synth": _synth_affinity, "soft": _soft_blobs, "uniform": lambda e: _near_uniform(0, e)}[kind](arg)


def _spectral_case(aff, k, **kw):
    from sklearn.cluster import SpectralClustering
    from rtti_b200 import attention_utils as au
    np.random.seed(6)
    ref = SpectralClustering(k, affinity="precomputed", n_init=N_INIT, assign_labels="kmeans").fit_predict(aff.cpu().numpy())
    ref_state = np.random.get_state()
    np.random.seed(6)
    got = au.spectral_clustering(aff, k, **kw)
    return got, ref, all(np.array_equal(x, y) for x, y in zip(np.random.get_state(), ref_state))


def _emu_fit(x, draws):
    return kmeans_emu.kmeans_fit(x.cpu().numpy(), draws)


# Near-uniform affinities at k = 4 whose eigengaps straddle EIGENGAP_MIN: 3.9e-6 and 2.0e-6 run on the device path,
# 1.0e-6 (just below) and 3.8e-7 are handed to scikit-learn
GAP_SWEEP = [("uniform", e, 4) for e in (1.6e-5, 8e-6, 4e-6, 1.6e-6)]


def test_gap_sweep_straddles_the_threshold():
    from rtti_b200 import attention_utils as au
    gaps = []
    for _, e, k in GAP_SWEEP:
        ev = au.spectral_embedding(_affinity("uniform", e), k)[1]
        gaps.append(float(ev[k] - ev[k - 1]))
    assert min(gaps[:2]) >= au.EIGENGAP_MIN > max(gaps[2:]) and gaps[2] > 0.9e-6


@pytest.mark.parametrize("kind,arg,k", SPECTRAL_CASES + GAP_SWEEP)
def test_spectral_clustering_matches_sklearn(kind, arg, k):
    aff = _affinity(kind, arg)
    got, ref, same_state = _spectral_case(aff, k, kmeans_fit=_emu_fit)
    assert got.dtype == np.int32 and np.array_equal(got, ref)
    assert same_state


def test_eigengap_guard_hands_ill_posed_affinities_to_sklearn():
    """Near-uniform affinity with a 9th eigenvalue that is not separated: the kernel must not run."""
    from rtti_b200 import attention_utils as au
    aff = _near_uniform(1, 1e-4)
    _, evals = au.spectral_embedding(aff, 9)
    assert float(evals[9] - evals[8]) < au.EIGENGAP_MIN

    def no_kernel(*a):
        raise AssertionError("k-means kernel called below the eigengap threshold")
    got, ref, same_state = _spectral_case(aff, 9, kmeans_fit=no_kernel)
    assert np.array_equal(got, ref) and same_state


def test_kmeans_draws_equal_sklearn_calls():
    """The bulk draw equals choice(n, p=w) followed by k-1 uniform(size=trials) per restart."""
    from rtti_b200.attention_utils import kmeans_draws
    for n, k in ((257, 5), (1024, 9), (1000, 1)):
        rs, rs2 = np.random.RandomState(3), np.random.RandomState(3)
        d = kmeans_draws(rs, n, k, 7)
        w = np.ones(n, np.float32)
        t = 2 + int(np.log(k))
        for r in range(7):
            assert d[r, 0] == rs2.choice(n, p=w / w.sum())
            for c in range(1, k):
                assert np.array_equal(d[r, 1 + (c - 1) * t:1 + c * t], rs2.uniform(size=t))
        assert _same_state(rs, rs2)


def test_kmeans_c_abi_rejects_bad_arguments_without_launching():
    from rtti_b200 import _lib
    lib = _lib.load()
    V = ctypes.c_void_p
    buf = (ctypes.c_char * 4096)()
    a = (ctypes.addressof(buf) + 15) // 16 * 16
    ARG, SHAPE = -1, -2
    fit = lambda x, n, k, n_init, max_iter, tol=1e-4: lib.rtti_kmeans_fit(V(x), V(a), n, k, n_init, max_iter, tol, V(a), V(a),
                                                                         V(a), V(a), V(0))
    assert fit(0, 1024, 4, 100, 300) == ARG            # null embedding
    assert fit(a, 1024, 4, 0, 300) == ARG              # no restart
    assert fit(a, 1024, 4, 100, 0) == ARG              # no iteration
    assert fit(a, 1024, 4, 100, 300, -1.0) == ARG      # negative tolerance
    assert fit(a, 1024, 0, 100, 300) == SHAPE          # k < 1
    assert fit(a, 1024, 33, 100, 300) == SHAPE         # k > 32
    assert fit(a, 3, 4, 100, 300) == SHAPE             # fewer samples than clusters
    assert fit(a, 4097, 4, 100, 300) == SHAPE          # n > 4096
    assert fit(a, 4096, 16, 100, 300) == SHAPE         # embedding does not fit in shared memory
    assert lib.rtti_kmeans_fit(V(a), V(0), 64, 4, 1, 1, 1e-4, V(a), V(a), V(a), V(a), V(0)) == ARG   # null draws
    assert lib.rtti_kmeans_fit(V(a), V(a), 64, 4, 1, 1, 1e-4, V(a), V(a), V(a), V(0), V(0)) == ARG   # null flags
    assert lib.rtti_kmeans_supported(1024, 32) == 0 and lib.rtti_kmeans_supported(4096, 11) == 0
    assert lib.rtti_kmeans_supported(4096, 12) == SHAPE and lib.rtti_kmeans_supported(1024, 33) == SHAPE


# ---------------------------------------------------------------- GPU

def _gpu_fit(x, draws):
    from rtti_b200 import ops
    out = ops.kmeans_fit(torch.from_numpy(np.ascontiguousarray(x)).cuda(), torch.from_numpy(draws).cuda())
    return tuple(v.cpu().numpy() for v in out)


@pytest.mark.gpu
@pytest.mark.parametrize("n,k,kind", KMEANS_CASES)
def test_kmeans_kernel_matches_sklearn(n, k, kind):
    x, km, labels, inertia, same_state = _kmeans_case(n, k, kind, _gpu_fit)
    assert np.array_equal(labels, km.labels_)
    assert same_state
    assert _inertia_close(inertia, km.inertia_, x, 1e-5)


@pytest.mark.gpu
def test_kmeans_kernel_is_deterministic_and_matches_its_restatement():
    from rtti_b200.attention_utils import kmeans_draws
    x = _blobs(1024, 9, 5, "aniso")
    draws = kmeans_draws(np.random.RandomState(0), 1024, 9, N_INIT)
    a, b = _gpu_fit(x, draws), _gpu_fit(x, draws)
    assert all(np.array_equal(u, v) for u, v in zip(a, b))
    e = kmeans_emu.kmeans_fit(x, draws)
    assert np.array_equal(a[0], e[0]) and np.array_equal(a[2], e[2]) and not a[3].any()
    x = np.random.default_rng(0).normal(size=(64, 3)).astype(np.float32)   # see test_ambiguous_relocation_is_flagged_...
    assert _gpu_fit(x, np.zeros((1, 7)))[3][0] == 1 and _gpu_fit(x[:, :2].copy(), np.zeros((1, 3)))[3][0] == 0
    assert np.allclose(a[1], e[1], rtol=1e-9, atol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,arg,k", SPECTRAL_CASES)
def test_spectral_clustering_on_device_matches_sklearn(kind, arg, k):
    aff = _affinity(kind, arg).cuda()
    got, ref, same_state = _spectral_case(aff, k)
    assert np.array_equal(got, ref)
    assert same_state


@pytest.mark.gpu
def test_spectral_clustering_on_sd15_capture_matches_sklearn():
    from tests.token_map_cluster_bench import sd15_capture
    aff, _ = sd15_capture()
    got, ref, same_state = _spectral_case(aff, 9)
    assert np.array_equal(got, ref)
    assert same_state
