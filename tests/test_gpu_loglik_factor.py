"""The float64 log-likelihood factorisation (smk_potrf_loglik_f64, csrc/potrf_ll.cu, DESIGN section 7) at the block counts
the slice sampler runs it at, against LAPACK and the float64 oracle.

LogLik pads to Npad = ceil128(N + 1), so the factorisation runs over nblk = Npad / 128 block columns.  enqueue() takes
the columns in pairs and branches on how many block rows are left below each of them: the look-ahead hand-offs carried
into the next pair start at nblk >= 4, the background update on the side stream (and the next pair's wait for it) at
nblk >= 5, and the steady state, where the background update of pair j runs next to the look-ahead of pair j+2, at
nblk >= 7.  The tests cover nblk = 1 ... 10 with the augmented row N both as the last row of the last block (N = 127
mod 128) and alone in a fresh block (N = 0 mod 128), the headline size (N = 4096, nblk = 33) and N = 8192 (nblk = 65);
batch sizes S = 1, 2, 3, 6 and 8, which change the number of CTAs the background update leaves to the spine.

What a stale or missing block update looks like: a backward error some 1e10 times LAPACK's or more, not a factor of a
few.  What a race or a dependency between batch items looks like: the bitwise invariants below fail.  Each output tile is
produced by one CTA in a fixed k order, so a batch item equals the same matrix factored alone, a graph replay equals the
direct launch sequence, and the strict upper triangle (never read) cannot change the lower one.
"""
import functools

import numpy as np
import pytest
import scipy.linalg as spla

from oracle import gp_oracle as O
from tests.helpers import check_rows, ratio, sym

gpu = pytest.mark.gpu

U = 2.0 ** -53          # unit roundoff of float64
NB = 128                # block size of potrf_ll.cu


def _npad(N):
    return (N + 1 + NB - 1) // NB * NB


# ---------------------------------------------------------------------------------------------------- device plumbing
@pytest.fixture(scope="module")
def eng():
    import torch
    from spearmint_b200.engine import GPEIEngine
    return GPEIEngine(dtype=torch.float64)


@pytest.fixture(scope="module")
def backend():
    from spearmint_b200.backend import DeviceBackend
    return DeviceBackend()


def _lib():
    from spearmint_b200 import _lib as L
    return L.lib()


def _data(N, D, seed):
    rs = np.random.RandomState(seed)
    X = rs.rand(N, D)
    y = np.sin(3 * X).sum(1) + 0.01 * rs.randn(N)
    return X, (y - y.mean()) / y.std(), rs


def _hypers(rs, S, D, noise):
    return [(0.1 * rs.randn(), noise, float(np.exp(0.25 * rs.randn())), rs.uniform(0.3, 2.0, D)) for _ in range(S)]


def _inputs(eng, kind, X, y, hs, Npad):
    """[S][Npad][Npad] as LogLik.batch builds it: smk_cov_build_lower into zeros, then the augmented row N."""
    import torch
    from spearmint_b200.engine import KINDS, check, fn, ptr
    N, D = X.shape
    S, f64 = len(hs), torch.float64
    hb = eng.hypers(hs, kind)
    Xd, yd = eng.to_dev(X), eng.to_dev(y)
    A = torch.zeros((S, Npad, Npad), dtype=f64, device=eng.device)
    st = eng.stream()
    check(fn("smk_cov_build_lower", f64)(KINDS[kind], N, D, S, ptr(Xd), ptr(hb.inv_ls), ptr(hb.amp2), ptr(hb.noise),
                                         ptr(A), Npad, st), "cov_build_lower")
    check(fn("smk_loglik_set_rhs", f64)(N, Npad, S, ptr(yd), ptr(hb.mean), ptr(A), st), "loglik_set_rhs")
    return A


def _workspace(eng, Npad, S):
    """(workspace, info) of one call site: the graph cache keys on (A, workspace, info, Npad, S)."""
    import torch
    ws = torch.empty((_lib().smk_potrf_loglik_workspace_bytes(Npad, S),), dtype=torch.uint8, device=eng.device)
    return ws, torch.full((S,), -1, dtype=torch.int32, device=eng.device)


def _potrf(eng, A, use_graph=0, ws=None):
    """Factors A [S][Npad][Npad] in place; returns info[S] read back to the host (so nothing is in flight after it)."""
    from spearmint_b200.engine import check, ptr
    S, Npad = A.shape[0], A.shape[-1]
    ws, info = ws if ws is not None else _workspace(eng, Npad, S)
    check(_lib().smk_potrf_loglik_f64(Npad, S, ptr(A), ptr(ws), ws.numel(), ptr(info), use_graph, eng.stream()),
          "potrf_loglik")
    return info[:S].cpu().numpy()


def _finish(eng, L, N):
    """(sum_{i<N} log L_ii, |L[N, :N]|^2) per matrix, by smk_loglik_finish_f64."""
    import torch
    from spearmint_b200.engine import check, fn, ptr
    S, Npad = L.shape[0], L.shape[-1]
    out = torch.empty((2, S), dtype=torch.float64, device=eng.device)
    check(fn("smk_loglik_finish", torch.float64)(N, Npad, S, ptr(L), ptr(out[0]), ptr(out[1]), eng.stream()),
          "loglik_finish")
    return out.cpu().numpy()


def _same_lower(a, b):
    import torch
    return torch.equal(torch.tril(a), torch.tril(b))


# ---------------------------------------------------------------------------------------------------- host references
def _kappa(K, N, Lk=None):
    """Spectral condition number of the N x N covariance K (lower triangle read).  At N > 4096 the eigen-decomposition
    costs too much on the host: LAPACK's 1-norm estimate from the factor Lk (kappa_1 >= kappa_2 for a symmetric matrix)."""
    if N <= 4096:
        w = np.linalg.eigvalsh(K[:N, :N])
        return float(w[-1] / w[0])
    anorm = np.abs(sym(K[:N, :N])).sum(axis=0).max()
    rcond, info = spla.lapack.dpocon(Lk[:N, :N], anorm, uplo="L")
    assert info == 0
    return float(1.0 / rcond)


# ---------------------------------------------------------------------------------------------------- 1. the factorisation
def _small_cases():
    """nblk = 1 ... 10, row N last in its block (N = 127 mod 128) and alone in a fresh block (N = 0 mod 128), kernel / D /
    noise / S rotating through Matern52 and SE, D in {3, 8, 32}, noise 1e-2 ... 1e-6 and S in {1, 2, 3, 8}."""
    kinds, Ds, noises, Ss = ("Matern52", "SE"), (3, 8, 32), (1e-2, 1e-3, 1e-4, 1e-5, 1e-6), (1, 2, 3, 8)
    out, i = [], 0
    for nblk in range(1, 11):
        for res in (127, 0):
            N = NB * nblk - 1 if res == 127 else NB * (nblk - 1)
            if N <= 0:
                continue
            assert _npad(N) // NB == nblk
            out.append(pytest.param(N, kinds[i % 2], Ds[i % 3], noises[i % 5], Ss[i % 4],
                                    id="nblk%02d-N%d-%s-D%d-noise%g-S%d" % (nblk, N, kinds[i % 2], Ds[i % 3],
                                                                         noises[i % 5], Ss[i % 4])))
            i += 1
    return out


def _factor_case(eng, record_property, N, kind, D, noise, S, seed, dense):
    import torch
    Npad = _npad(N)
    X, y, rs = _data(N, D, seed)
    hs = _hypers(rs, S, D, noise)
    A_in = _inputs(eng, kind, X, y, hs, Npad)                       # the exact input, kept
    A = A_in.clone()
    info = _potrf(eng, A, 0)                                        # checked after the backward error (more telling)
    sld, quad = _finish(eng, A, N)

    # against LAPACK and the oracle, on the host
    rows = np.arange(Npad) if dense else check_rows(N, Npad, rs)
    for s, h in enumerate(hs):
        Ah, L = A_in[s].cpu().numpy(), np.tril(A[s].cpu().numpy())
        Lref = spla.cholesky(sym(Ah), lower=True, check_finite=False)
        r_gpu, r_lap = ratio(L, Ah, rows, U), ratio(Lref, Ah, rows, U)
        bound = max(32.0 * r_lap, 2.0 * N)
        record_property("s%d_backward_ratio_gpu" % s, r_gpu)
        record_property("s%d_backward_ratio_lapack" % s, r_lap)
        assert r_gpu <= bound, "item %d: backward error %.3g u|L||L^T| (LAPACK %.3g, bound %.3g)" % (s, r_gpu, r_lap, bound)
        assert info[s] == 0
        # rows N+1 .. Npad-1 of L are the identity
        pad = L[N + 1:]
        ref_pad = np.zeros_like(pad)
        ref_pad[:, N + 1:] = np.eye(Npad - N - 1)
        assert np.array_equal(pad, ref_pad)
        # the two pieces of the log-likelihood, against LAPACK's factor of the same matrix and the oracle
        kappa = _kappa(Ah, N, Lref)
        rtol = 50.0 * kappa * U
        record_property("s%d_kappa" % s, kappa)
        ld = np.log(np.diag(Lref)[:N])
        sld_ref, quad_ref = ld.sum(), Lref[N, :N].dot(Lref[N, :N])
        msg = "item %d, kappa %.3g, rtol %.3g" % (s, kappa, rtol)
        assert abs(sld[s] - sld_ref) <= rtol * np.abs(ld).sum(), (sld[s], sld_ref, msg)
        assert abs(quad[s] - quad_ref) <= rtol * quad_ref, (quad[s], quad_ref, msg)
        if dense or s == 0:           # the oracle rebuilds and refactors K: once per case at N >= 4096
            lp_ref = O.gp_logprob(kind, h[0], h[1], h[2], h[3], X, y)
            assert abs(-sld[s] - 0.5 * quad[s] - lp_ref) <= rtol * (np.abs(ld).sum() + 0.5 * quad_ref), (lp_ref, msg)

    # bitwise invariants, on the device
    ws = _workspace(eng, Npad, S)
    G = A_in.clone()
    _potrf(eng, G, 1, ws)                                           # new key: direct launch + capture (or a replay)
    assert _same_lower(G, A), "use_graph=1 (first call) differs from use_graph=0"
    G.copy_(A_in)
    _potrf(eng, G, 1, ws)                                           # same key: a replay of the captured graph
    assert _same_lower(G, A), "graph replay differs from use_graph=0"
    del G
    upper = torch.triu(torch.ones((Npad, Npad), dtype=torch.bool, device=eng.device), 1)
    Z = torch.tril(A_in)
    _potrf(eng, Z, 0)
    assert _same_lower(Z, A), "the strict upper triangle of the input changed the factor"
    Z = A_in.masked_fill(upper, float("nan"))
    _potrf(eng, Z, 0)
    assert _same_lower(Z, A), "a NaN strict upper triangle changed the factor: it is read"
    del Z, upper
    if S > 1:
        for s in range(S):
            one = A_in[s:s + 1].clone()
            assert _potrf(eng, one, 0)[0] == info[s]
            assert _same_lower(one[0], A[s]), "batch item %d differs from the same matrix factored alone" % s


@gpu
@pytest.mark.parametrize("N,kind,D,noise,S", _small_cases())
def test_factor_block_counts_1_to_10(eng, record_property, N, kind, D, noise, S):
    """Every branch of enqueue() (nblk = 1 ... 10) against LAPACK on the same input, dense over the whole matrix.

    Bound: the componentwise backward error may be at most max(32 x LAPACK's, 2 N).  The panels multiply by explicit
    inverses of the 32 x 32 diagonal pieces, which can cost more than LAPACK's substitution on ill-conditioned pieces.
    Worst ratio measured on an H100 80 GB HBM3 (SXM, 700 W) over all items of these cases, in units of u, with the largest
    GPU / LAPACK quotient of one item in brackets:
      noise 1e-2: 36.6 against LAPACK's 20.2 (1.8x)      noise 1e-3: 37.3 against 16.0 (2.3x)
      noise 1e-4: 30.3 against 22.9 (1.8x)               noise 1e-5: 61.9 against 18.8 (3.4x)
      noise 1e-6: 63.6 against 16.6 (3.8x)
    A skipped block update in enqueue() measures 6e11 - 5e15, or leaves non-finite entries.  When row N sits alone in the last block (N = 0 mod 128), an update
    that only that block misses changes nothing but the augmented pivot 1e30, which no output reads: such a case passes
    with or without it.
    """
    _factor_case(eng, record_property, N, kind, D, noise, S, seed=N + 7 * S, dense=True)


@gpu
@pytest.mark.parametrize("N,kind,D,noise,S", [
    pytest.param(4096, "Matern52", 32, 1e-3, 1, id="nblk33-N4096-Matern52-D32-noise1e-3-S1"),
    pytest.param(4096, "SE", 8, 1e-6, 2, id="nblk33-N4096-SE-D8-noise1e-6-S2"),
    pytest.param(4096, "Matern52", 3, 1e-5, 6, id="nblk33-N4096-Matern52-D3-noise1e-5-S6"),
    pytest.param(8192, "Matern52", 32, 1e-4, 1, id="nblk65-N8192-Matern52-D32-noise1e-4-S1"),
])
def test_factor_at_size(eng, record_property, N, kind, D, noise, S):
    """The headline (N = 4096, nblk = 33) and c5 (N = 8192, nblk = 65) sizes, where the steady state runs for many pairs.
    The backward error is evaluated on a row subset (block edges, 32-piece edges of five blocks, the last 200 rows, row N,
    300 random rows) for both factors.  Same bound as at nblk <= 10.  Worst ratio measured on an H100 80 GB HBM3 (SXM,
    700 W), in units of u:
      noise 1e-3 (N = 4096): 19.2 against LAPACK's 8.1     noise 1e-4 (N = 8192): 23.4 against 12.6
      noise 1e-5 (N = 4096): 31.7 against 15.7             noise 1e-6 (N = 4096): 30.1 against 11.0
    """
    _factor_case(eng, record_property, N, kind, D, noise, S, seed=N + S, dense=False)


# ---------------------------------------------------------------------------------------------------- 2. graph replay and the cache
@gpu
def test_graph_replay_new_contents_then_smaller_batch(eng):
    """A captured graph replayed on the same buffers with new contents factors the new contents; the same A with a
    smaller S is a new key, factors only its S matrices and leaves the rest of the buffer alone."""
    N, D, S, kind = 1100, 8, 3, "Matern52"                           # nblk = 9: steady state
    Npad = _npad(N)
    X, y, rs = _data(N, D, 31)
    A1 = _inputs(eng, kind, X, y, _hypers(rs, S, D, 1e-4), Npad)
    X2, y2, rs2 = _data(N, D, 32)
    A2 = _inputs(eng, kind, X2, y2, _hypers(rs2, S, D, 1e-6), Npad)
    ref1, ref2 = A1.clone(), A2.clone()
    assert np.all(_potrf(eng, ref1, 0) == 0) and np.all(_potrf(eng, ref2, 0) == 0)

    ws = _workspace(eng, Npad, S)
    buf = A1.clone()
    assert np.all(_potrf(eng, buf, 1, ws) == 0)
    assert _same_lower(buf, ref1)
    buf.copy_(A2)
    assert np.all(_potrf(eng, buf, 1, ws) == 0)                      # replay
    assert _same_lower(buf, ref2)
    buf[:2].copy_(A1[:2])
    assert np.all(_potrf(eng, buf[:2], 1, ws) == 0)                  # same A pointer, S = 2: a new key
    assert _same_lower(buf[:2], ref1[:2])
    assert _same_lower(buf[2], ref2[2])                              # item 2 untouched
    buf[:2].copy_(A2[:2])
    assert np.all(_potrf(eng, buf[:2], 1, ws) == 0)                  # ... and its replay
    assert _same_lower(buf[:2], ref2[:2])


def _spd_batch(rs, S, n):
    mats = []
    for _ in range(S):
        X = rs.rand(n, 4)
        mats.append(O.cov("Matern52", float(np.exp(0.3 * rs.randn())), rs.uniform(0.3, 2.0, 4), X)
                    + 10.0 ** rs.uniform(-6, -2) * np.eye(n))
    return np.stack(mats)


@gpu
def test_graph_cache_rollover(eng):
    """More than 64 distinct (A, workspace, info, Npad, S) keys: the cache is emptied and refilled on the way.  Every call
    is checked against a direct launch of the same input; keys from before and after the rollover are used again with
    new contents.  Every result is read back before the next call, as LogLik.batch does, so no graph is in flight when
    the cache destroys it."""
    import torch
    keys, step = 80, 256                                             # A pointers 2 KB apart: one key each
    pool = torch.zeros((keys * step + 3 * 256 * 256,), dtype=torch.float64, device=eng.device)
    ws = _workspace(eng, 256, 3)
    rs = np.random.RandomState(77)

    def run(k):
        Npad, S = (128, 256)[k % 2], 1 + (k // 2) % 3
        A = pool[k * step:k * step + S * Npad * Npad].view(S, Npad, Npad)
        inp = torch.from_numpy(_spd_batch(rs, S, Npad)).to(eng.device)
        A.copy_(inp)
        assert np.all(_potrf(eng, A, 1, ws) == 0)
        got = A.clone()
        ref = inp.clone()
        assert np.all(_potrf(eng, ref, 0) == 0)
        assert _same_lower(got, ref), "key %d (Npad %d, S %d)" % (k, Npad, S)
        L = np.tril(got[0].cpu().numpy())
        h = inp[0].cpu().numpy()
        assert ratio(L, h, np.arange(Npad), U) <= max(32.0 * ratio(spla.cholesky(h, lower=True), h, np.arange(Npad), U),
                                                      2.0 * Npad)

    for k in range(keys):
        run(k)
    run(0)                           # evicted by the rollover: captured again
    run(keys - 1)                    # still cached: a replay
    run(1)


# ---------------------------------------------------------------------------------------------------- 3. info, non-PD matrices
PIVOTS = ("block0_mid_piece", "at_128", "piece_edge_later_block", "last_block")


def _pivot_index(nblk, where):
    Npad = NB * nblk
    return {"block0_mid_piece": 45, "at_128": 128, "piece_edge_later_block": NB * (nblk // 2) + 64,
            "last_block": Npad - 20}[where]


@functools.lru_cache(maxsize=1)
def _planted_base(nblk):
    """(A0 = B B^T, diag(B), two other positive-definite matrices) for Npad = 128 nblk: B lower triangular with a
    positive diagonal, so every leading block of A0 is positive definite."""
    Npad = NB * nblk
    mats, diags = [], []
    for seed in range(3):
        rs = np.random.RandomState(100 * nblk + seed)
        B = np.tril(rs.randn(Npad, Npad), -1) * (0.5 / np.sqrt(Npad)) + np.diag(1.0 + rs.rand(Npad))
        mats.append(B.dot(B.T))
        diags.append(np.diag(B).copy())
    return mats[0], diags[0], mats[1], mats[2]


def _planted(nblk, where):
    """A0 with pivot i0 made negative: A0[i0, i0] -= 1.5 B[i0, i0]^2 turns the i0-th pivot into -0.5 B[i0, i0]^2 and
    leaves everything before it as it was.  Returns (bad, i0, good1, good2)."""
    A0, d, g1, g2 = _planted_base(nblk)
    i0 = _pivot_index(nblk, where)
    bad = A0.copy()
    bad[i0, i0] -= 1.5 * d[i0] ** 2
    return bad, i0, g1, g2


PLANTED = [(nblk, where) for nblk in (2, 5, 8, 33) for where in PIVOTS]


@pytest.mark.parametrize("nblk,where", PLANTED)
def test_planted_pivot_fixture_lapack(nblk, where):
    """The fixture of test_info_names_planted_pivot: LAPACK's dpotrf stops at exactly the planted pivot, and the other
    matrices of the batch factor."""
    bad, i0, g1, g2 = _planted(nblk, where)
    assert spla.lapack.dpotrf(bad, lower=1)[1] == i0 + 1
    if where == PIVOTS[0]:
        assert spla.lapack.dpotrf(g1, lower=1)[1] == 0 and spla.lapack.dpotrf(g2, lower=1)[1] == 0


@gpu
@pytest.mark.parametrize("nblk,where", PLANTED)
def test_info_names_planted_pivot(eng, nblk, where):
    """info[s] is exactly the 1-based index of the first non-positive pivot of item s, and a non-PD item changes
    nothing else of the batch: the other items have info 0 and equal their solo factorisations bit for bit."""
    import torch
    bad, i0, g1, g2 = _planted(nblk, where)
    host = np.stack([g1, bad, g2])
    for use_graph in (0, 1):
        A = torch.from_numpy(host).to(eng.device)
        info = _potrf(eng, A, use_graph)
        assert info.tolist() == [0, i0 + 1, 0], (use_graph, info, i0)
        for s in (0, 2):
            one = torch.from_numpy(host[s:s + 1]).to(eng.device)
            assert _potrf(eng, one, 0)[0] == 0
            assert _same_lower(one[0], A[s]), (use_graph, s)


@gpu
def test_loglik_batch_isolates_a_non_pd_item(backend):
    """LogLik.batch([good, bad, good]) at N = 1000: NaN for the indefinite item (negative noise), the other two equal
    their solo evaluations bit for bit."""
    N, D, kind = 1000, 5, "Matern52"
    X, y, rs = _data(N, D, 41)
    ll = backend.loglik(kind, X, y)
    good = _hypers(rs, 2, D, 1e-3)
    bad = (0.0, -5.0, 1.0, np.ones(D))
    out = ll.batch([good[0], bad, good[1]])
    assert np.isfinite(out[0]) and np.isnan(out[1]) and np.isfinite(out[2]), out
    assert ll.batch([good[0]])[0] == out[0]
    assert ll.batch([good[1]])[0] == out[2]
    with pytest.raises(np.linalg.LinAlgError):
        ll(*bad)


# ---------------------------------------------------------------------------------------------------- 4. the callers at size
def _loglik_tol(K, N, lp_ref):
    """50 kappa u of the value's scale 0.5 sum |log lambda_i| + 0.5 quad, from the eigenvalues of K."""
    w = np.linalg.eigvalsh(K)
    kappa = float(w[-1] / w[0])
    sld = 0.5 * np.log(w).sum()
    quad = -2.0 * (lp_ref + sld)
    return 50.0 * kappa * U * (0.5 * np.abs(np.log(w)).sum() + 0.5 * abs(quad)), kappa


@gpu
@pytest.mark.parametrize("N", [127, 128, 1023, 1600, 4096])
def test_loglik_at_size(backend, monkeypatch, N):
    """LogLik (the dedicated factorisation) against the oracle's log-likelihood, and against LogLik on the generic
    float64 factorisation (SMK_LOGLIK_IMPL=simt), within 50 kappa u."""
    D, kind = (3, "Matern52") if N != 1023 else (8, "SE")
    X, y, rs = _data(N, D, 51 + N)
    hs = [(0.1 * rs.randn(), noise, float(np.exp(0.25 * rs.randn())), rs.uniform(0.3, 2.0, D))
          for noise in ((1e-2, 1e-6, 1e-3) if N >= 4096 else (1e-2, 1e-4, 1e-6, 1e-3))]
    ll = backend.loglik(kind, X, y)
    assert ll.fast and ll.Npad == _npad(N)
    got = ll.batch(hs)
    monkeypatch.setenv("SMK_LOGLIK_IMPL", "simt")
    ll2 = backend.loglik(kind, X, y)
    assert not ll2.fast
    got2 = ll2.batch(hs)
    for s, h in enumerate(hs):
        ref = O.gp_logprob(kind, h[0], h[1], h[2], h[3], X, y)
        tol, kappa = _loglik_tol(O.cov(kind, h[2], h[3], X) + h[1] * np.eye(N), N, ref)
        assert abs(got[s] - ref) <= tol, (s, got[s], ref, "kappa %.3g" % kappa)
        assert abs(got[s] - got2[s]) <= tol, (s, got[s], got2[s], "kappa %.3g" % kappa)


@gpu
def test_latent_loglik_at_size(backend):
    """LatentLogLik at N = 1600 with six batch items, each with its own ff in its augmented row
    (smk_loglik_set_rhs_batched with ldy = N), against the classification-GP oracle within 50 kappa u."""
    from tests import constrained_oracle as CO
    N, D, kind, noise = 1600, 4, "Matern52", 1e-3
    rs = np.random.RandomState(61)
    comp = rs.rand(N, D)
    labels = (comp[:, 0] + comp[:, 1] < 1.1).astype(float)
    ls = rs.uniform(0.3, 1.5, D)
    ll = backend.latent_loglik(kind, comp, ls, noise)
    assert ll.fast and ll.max_batch == 6
    items = [(rs.uniform(0.3, 3.0), np.where(labels > 0, 1.0, -1.0) + rs.randn(N)) for _ in range(6)]
    got = ll.batch(items)
    for s, (a, f) in enumerate(items):
        ref = CO.latent_loglik(kind, a, ls, f, comp, noise)
        tol, kappa = _loglik_tol(O.cov(kind, a, ls, comp) + noise * np.eye(N), N, ref)
        assert abs(got[s] - ref) <= tol, (s, got[s], ref, "kappa %.3g" % kappa)
    assert ll(*items[4]) == got[4]


@gpu
def test_sampler_chain_two_phase_speculation(backend, tmp_path):
    """At N = 1600 LogLik batches a slice move in two phases (speculate = (0, 2)).  Two sample_hypers calls of
    GPEIOptChooserB200 on the device give the hyper-samples of the sequential oracle chain from the same seed (rtol 1e-6,
    the rule of the next() tests) and leave the RNG where the oracle chain leaves it."""
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    from tests.oracle_backend import OracleBackend
    N, D = 1600, 3
    rs = np.random.RandomState(71)
    comp = rs.rand(N, D)
    vals = np.sin(3 * comp).sum(1) + 0.1 * rs.randn(N)
    runs = []
    for name, be in (("device", backend), ("oracle", OracleBackend())):
        d = tmp_path / name
        d.mkdir()
        ch = mod.init(str(d), "covar=Matern52,mcmc_iters=2,use_multiprocessing=0")
        ch._backend = be
        np.random.seed(5)
        ch._real_init(D, vals)
        ch.sample_hypers(comp, vals)
        ch.sample_hypers(comp, vals)
        runs.append((ch, np.random.rand()))
    (dev, u_dev), (ora, u_ora) = runs
    assert dev._loglik.speculate == (0, 2)
    assert dev._loglik.launch_batches < dev._loglik.calls           # the batched path was taken
    assert len(dev.hyper_samples) == len(ora.hyper_samples) == 3
    for a, b in zip(dev.hyper_samples, ora.hyper_samples):
        np.testing.assert_allclose(np.hstack(a), np.hstack(b), rtol=1e-6, atol=1e-9)
    assert u_dev == u_ora
