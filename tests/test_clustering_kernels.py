"""GPU tests of the fp64 clustering kernels, problem by problem, against plain references (pytest -m gpu):

* batched centroid linkage (one CTA per problem, shared-memory state up to 4096 rows, global memory beyond) against
  the single-problem launch, the reversed batch and scipy's ``linkage(.., "centroid")`` / ``fcluster``;
* batched VBx (one 8-CTA cluster per problem; the D == 128 shared-memory tile path and the plain loop of any other D)
  against the oracle's VBx (utils/vbx.py) and against the single-problem launch;
* PLDA transform, VBx centroids and cosine cdist against numpy / scipy;
* the 3 x K assignment against ``linear_sum_assignment`` (ties of inactive speakers included) and ``np.argmax``.

All outputs are fp64 or integers: everything is compared bit for bit or at 1e-8 and tighter.
"""
import numpy as np
import pytest
import torch
from scipy.cluster.hierarchy import fcluster, linkage
from scipy.spatial.distance import cdist
from scipy.special import softmax

from oracle import pipeline as P
from pyannote_audio_b200 import ops
from pyannote_audio_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ctx(dev):
    from pyannote_audio_b200.models import get_context

    return get_context(dev)


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _same_partition(a, b):
    m = {}
    for x, y in zip(a, b):
        if m.setdefault(x, y) != y:
            return False
    return len(set(m.values())) == len(m)


# ---------------------------------------------------------------------------------------------------------
# batched centroid linkage
# ---------------------------------------------------------------------------------------------------------
LINK_SIZES = (0, 1, 2, 3, 31, 300, 4096, 4097, 5981)        # both sides of the 4096-row shared-memory limit


def _link_rows(rng, n, dim):
    """Clustered Gaussian rows holding float32 values, with exact duplicates (zero-distance ties) and
    near-duplicates."""
    if n == 0:
        return np.zeros((0, dim))
    centers = rng.standard_normal((7, dim))
    x = centers[rng.integers(0, 7, n)] + 0.5 * rng.standard_normal((n, dim))
    if n >= 3:
        dup = rng.choice(n, size=max(1, n // 20), replace=False)
        src = rng.integers(0, n, size=dup.size)
        x[dup] = x[src]                                                      # exact duplicates
        near = rng.choice(n, size=max(1, n // 50), replace=False)
        x[near] = x[rng.integers(0, n, size=near.size)] * (1 + 1e-6 * rng.standard_normal((near.size, 1)))
    return x.astype(np.float32).astype(np.float64)


def _normed(x, normalize):
    if normalize == "float32":
        x32 = x.astype(np.float32)
        return (x32 / np.linalg.norm(x32, axis=1, keepdims=True)).astype(np.float64)
    return x / np.linalg.norm(x, axis=1, keepdims=True)


@pytest.mark.parametrize("dim,normalize", [(256, "float32"), (256, True), (3, True), (3, "float32"),
                                           (100, "float32")])
def test_linkage_batched_per_problem(ctx, dev, dim, normalize):
    rng = np.random.default_rng(100 + dim)
    sizes = list(LINK_SIZES)
    xs = [_link_rows(rng, n, dim) for n in sizes]
    ro = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    assert (np.diff(ro) >= 0).all()
    Z = ctx.linkage_centroid_batched(_t(np.concatenate(xs), dev), ro, normalize=normalize).cpu().numpy()
    assert Z.shape == (sum(max(n - 1, 0) for n in sizes), 4)
    # the same problems in reverse order
    rev = xs[::-1]
    ro_r = np.concatenate([[0], np.cumsum([len(x) for x in rev])]).astype(np.int32)
    Zr = ctx.linkage_centroid_batched(_t(np.concatenate(rev), dev), ro_r, normalize=normalize).cpu().numpy()
    zoff = np.concatenate([[0], np.cumsum([max(n - 1, 0) for n in sizes])])
    zoff_r = np.concatenate([[0], np.cumsum([max(len(x) - 1, 0) for x in rev])])
    for f, (n, x) in enumerate(zip(sizes, xs)):
        Zf = Z[zoff[f]: zoff[f + 1]]
        fr = len(sizes) - 1 - f
        assert np.array_equal(Zf, Zr[zoff_r[fr]: zoff_r[fr + 1]]), f"n={n}: depends on the problem order"
        if n < 2:
            assert Zf.shape == (0, 4)
            continue
        alone = ctx.linkage_centroid(_t(x, dev), normalize=normalize).cpu().numpy()
        assert np.array_equal(Zf, alone), f"n={n}: batched launch differs from the single-problem launch"
        ref = linkage(_normed(x, normalize), "centroid", "euclidean")
        np.testing.assert_allclose(np.sort(Zf[:, 2]), np.sort(ref[:, 2]), rtol=1e-9, atol=1e-12, err_msg=f"n={n}")
        assert np.array_equal(Zf[:, 3].max(), float(n)) and (Zf[:, :2] < 2 * n - 1).all()
        for t in (0.0, 0.3, 0.6, 0.9, 1.2):
            assert _same_partition(fcluster(ref, t, "distance"), ops.fcluster_distance(Zf, t)), (n, t)


def test_linkage_batched_empty_problems(ctx, dev):
    """Zero-size problems are no-ops: they produce no rows of Z and do not shift their neighbours' rows."""
    rng = np.random.default_rng(7)
    a, b = _link_rows(rng, 40, 16), _link_rows(rng, 9, 16)
    ref = ctx.linkage_centroid_batched(_t(np.concatenate([a, b]), dev), [0, 40, 49]).cpu().numpy()
    got = ctx.linkage_centroid_batched(_t(np.concatenate([a, b]), dev), [0, 0, 40, 40, 40, 49, 49]).cpu().numpy()
    assert np.array_equal(got, ref)
    with pytest.raises(ValueError):
        ctx.linkage_centroid_batched(_t(np.concatenate([a, b]), dev), [0, 40, 30])        # decreasing offsets


# ---------------------------------------------------------------------------------------------------------
# batched VBx
# ---------------------------------------------------------------------------------------------------------
VBX_SHAPES = ((1, 1), (2, 2), (31, 3), (32, 8), (33, 9), (200, 16), (500, 64), (700, 65), (1000, 130))
EPS = 1e-4


def _vbx_problem(rng, n, S, D, plda, hot):
    """PLDA features of clustered embeddings (D == 128) or scaled clustered Gaussians, and an initial gamma."""
    k = max(1, min(S, 6))
    who = rng.integers(0, k, n)
    if D == 128:
        centers = rng.standard_normal((k, 256))
        fea = plda((centers[who] + 0.6 * rng.standard_normal((n, 256))).astype(np.float32).astype(np.float64))
    else:
        centers = 2.0 * rng.standard_normal((k, D))
        fea = centers[who] + rng.standard_normal((n, D))
    if hot:                                           # softmax(7 * one_hot(ahc)) as the pipeline builds it
        ahc = np.concatenate([np.arange(S), rng.integers(0, S, max(0, n - S))])[:n] if n >= S else np.arange(n) % S
        q = np.zeros((n, S))
        q[np.arange(n), ahc] = 1.0
        gamma0 = softmax(7.0 * q, axis=1)
    else:
        gamma0 = rng.dirichlet(np.ones(S), size=n)
    return np.ascontiguousarray(fea), gamma0


def _oracle_vbx(fea, phi, gamma0, Fa, Fb):
    gamma, pi, Li = P.VBx(fea, phi, Fa=Fa, Fb=Fb, pi=gamma0.shape[1], gamma=gamma0, maxIters=20, epsilon=EPS)
    L = np.array([l[0] for l in Li])
    # the stopping test must not be decided by rounding: every ELBO step is clear of epsilon
    margin = np.abs(np.diff(L) - EPS).min() if len(L) > 1 else np.inf
    assert margin > 1e-7, f"borderline ELBO stopping test (|dL - eps| = {margin:.2e}): choose another seed"
    return gamma, pi, len(Li)


@pytest.mark.parametrize("D", [128, 100])
@pytest.mark.parametrize("Fa,Fb", [(0.07, 0.8), (0.3, 0.5)])
def test_vbx_batched_per_problem(ctx, dev, D, Fa, Fb):
    rng = np.random.default_rng(D + int(100 * Fa))
    plda = P.PLDA(**syn.make_plda(2))
    phi = plda.phi.copy() if D == 128 else np.sort(np.exp(rng.uniform(np.log(0.05), np.log(20.0), D)))[::-1].copy()
    probs = []
    for hot in (True, False):
        for n, S in VBX_SHAPES:
            probs.append((n, S) + _vbx_problem(rng, n, S, D, plda, hot))
    fea = np.concatenate([p[2] for p in probs])
    g0 = np.concatenate([p[3].reshape(-1) for p in probs])
    ns, Ss = [p[0] for p in probs], [p[1] for p in probs]
    gamma, pi, iters = ctx.vbx_batched(_t(fea, dev), _t(phi, dev), _t(g0, dev), ns, Ss, Fa, Fb, max_iters=20,
                                       want_iters=True)
    gamma, pi = gamma.cpu().numpy(), pi.cpu().numpy()
    go = so = 0
    for j, (n, S, fea_j, g0_j) in enumerate(probs):
        g_j, p_j = gamma[go: go + n * S].reshape(n, S), pi[so: so + S]
        go, so = go + n * S, so + S
        rg, rp, rit = _oracle_vbx(fea_j, phi, g0_j, Fa, Fb)
        what = f"(n, S) = ({n}, {S}), {'one-hot' if j < len(VBX_SHAPES) else 'Dirichlet'} start"
        assert iters[j] == rit, f"{what}: {iters[j]} iterations, oracle {rit}"
        np.testing.assert_allclose(g_j, rg, rtol=1e-8, atol=1e-10, err_msg=what)
        np.testing.assert_allclose(p_j, rp, rtol=1e-8, atol=1e-10, err_msg=what)
        ga, pa, ia = ctx.vbx(_t(fea_j, dev), _t(phi, dev), _t(g0_j, dev), Fa, Fb, max_iters=20)
        assert ia == iters[j] and np.array_equal(ga.cpu().numpy(), g_j) and np.array_equal(pa.cpu().numpy(), p_j), \
            f"{what}: batched launch differs from the single-problem launch"


# ---------------------------------------------------------------------------------------------------------
# PLDA transform, centroids, cosine cdist
# ---------------------------------------------------------------------------------------------------------
def test_plda_transform(ctx, dev):
    from pyannote_audio_b200.clustering import PLDA

    d = syn.make_plda(2)
    dplda, oplda = PLDA(d), P.PLDA(**d)
    rng = np.random.default_rng(11)
    for n in (1, 7, 1000):
        x = rng.standard_normal((n, 256)).astype(np.float32).astype(np.float64)
        got = dplda.transform(_t(x, dev)).cpu().numpy()
        ref = oplda.plda_tf(oplda.xvec_tf(x))
        assert got.shape == (n, 128)
        np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(dplda.phi, oplda.phi, rtol=0, atol=0)


def test_weighted_centroids(ctx, dev):
    rng = np.random.default_rng(12)
    n, S, dim = 300, 9, 256
    q = rng.dirichlet(np.ones(S), size=n)
    train = rng.standard_normal((n, dim)).astype(np.float32).astype(np.float64)
    for kept in (np.array([0, 2, 3, 7]), np.array([8, 1]), np.arange(S), np.zeros(0, dtype=np.int64)):
        got = ctx.weighted_centroids(_t(q, dev), _t(kept.astype(np.int32), dev), _t(train, dev)).cpu().numpy()
        W = q[:, kept]
        ref = W.T @ train / W.sum(0)[:, None]
        assert got.shape == (len(kept), dim)
        np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-13)


def test_cdist_cosine_edges(ctx, dev):
    rng = np.random.default_rng(13)
    for m in (1, 127, 128, 129):
        for k in (1, 5):
            b = rng.standard_normal((k, 256))
            a = rng.standard_normal((m, 256))
            a[0] = b[0]                                      # identical: 0
            if m > 2:
                a[1] = -b[0]                                 # opposite: 2
                a[m - 1] = 0.0                               # all-zero row: NaN
            got = ctx.cdist_cosine(_t(a, dev), _t(b, dev)).cpu().numpy()
            ref = cdist(a, b, "cosine")
            assert np.array_equal(np.isnan(got), np.isnan(ref)), (m, k)
            np.testing.assert_allclose(got, ref, rtol=1e-10, atol=1e-12, equal_nan=True)
            assert abs(got[0, 0]) <= 4.5e-16
            if m > 2:
                assert abs(got[1, 0] - 2.0) <= 4.5e-16 and np.isnan(got[m - 1]).all()


# ---------------------------------------------------------------------------------------------------------
# assignment
# ---------------------------------------------------------------------------------------------------------
def _assign_inputs(rng, K, C=240):
    """2 - cosine-distance-like scores; chunk c has (c % 4) speakers set to the reference's `const` (inactive), so
    their rows tie exactly."""
    soft = 2 - rng.uniform(0, 2, size=(C, 3, K))
    const = soft.min() - 1.0
    for c in range(C):
        soft[c, rng.permutation(3)[: c % 4]] = const
    return soft


@pytest.mark.parametrize("K", [1, 2, 3, 4, 7, 20])
def test_assign_against_linear_sum_assignment(ctx, dev, K):
    rng = np.random.default_rng(20 + K)
    soft = _assign_inputs(rng, K)
    hard = ctx.assign(_t(soft, dev), constrained=True).cpu().numpy()
    ref = P.constrained_argmax(soft)
    bad = np.flatnonzero((hard != ref).any(axis=1))
    assert bad.size == 0, f"K={K}: chunks {bad[:10].tolist()} (inactive rows {[c % 4 for c in bad[:10]]})"
    # exact ties everywhere (quantised scores)
    q = rng.integers(0, 3, size=(60, 3, K)).astype(np.float64) * 0.25
    assert np.array_equal(ctx.assign(_t(q, dev), constrained=True).cpu().numpy(), P.constrained_argmax(q))
    assert np.array_equal(ctx.assign(_t(soft, dev), constrained=False).cpu().numpy(), np.argmax(soft, axis=2))
    assert np.array_equal(ctx.assign(_t(q, dev), constrained=False).cpu().numpy(), np.argmax(q, axis=2))


def test_assign_nan_semantics(ctx, dev):
    """NaN scores: ``constrained_argmax`` replaces them by the nan-minimum before the solver (clustering.py:128-132),
    the unconstrained path is ``np.argmax`` (a NaN counts as the maximum)."""
    from pyannote_audio_b200.clustering import VBxClustering

    rng = np.random.default_rng(30)
    for K in (1, 2, 3, 5):
        soft = _assign_inputs(rng, K, C=80)
        soft[rng.uniform(size=(80, 3)) < 0.15] = np.nan               # whole rows (NaN embeddings)
        part = soft.copy()
        part[rng.uniform(size=part.shape) < 0.1] = np.nan              # and single entries
        clus = VBxClustering(P.PLDA(**syn.make_plda(2)), device=dev)
        assert np.array_equal(clus.constrained_argmax(soft), P.constrained_argmax(soft)), K
        assert np.array_equal(clus.constrained_argmax(part), P.constrained_argmax(part)), K
        assert np.array_equal(ctx.assign(_t(part, dev), constrained=False).cpu().numpy(), np.argmax(part, axis=2)), K
    with pytest.raises(ValueError):
        ctx.assign(_t(np.zeros((2, 3, 128)), dev), constrained=True)          # cluster ids are int8
