"""Device engine for the GP-EI hot path: owns HBM buffers (torch tensors) and drives the C-ABI kernels.

Mirrors, per batch of hyper-samples, what the reference does one sample at a time in
``GPEIOptChooser.compute_ei`` (chooser/GPEIOptChooser.py:527-619) and
``GPEIperSecChooser.compute_ei_per_s`` (chooser/GPEIperSecChooser.py:437-548):

    cov_build -> potrf -> chol_solve (alpha) -> predict (mu, var) -> ei_sweep

HBM layout (T = float32 on the grid path, float64 for log-likelihoods / refinement / logic tests):
    X        [N][D]            observed (or observed+pending) inputs, row-major
    C        [M][D]            candidates
    hypers   inv_ls[S][D], amp2[S], noise[S], mean[S]
    factor   [S][Npad][Npad]   K, overwritten by its lower Cholesky factor; Npad = ceil128(N)
    winv     [S][Npad/NB][NB][NB]  inverses of the diagonal blocks of L
    alpha    [S][F][Npad]
    mu       [S][F][ldm], var [S][ldm], ei [S][ldm], ei_sum [ldm];  ldm = ceil128(M)

torch provides the allocator and the stream only.  Nothing here falls back to the CPU.
"""
import ctypes as C
import os

import numpy as np
import scipy.stats as sps
import torch

from . import _lib
from ._lib import KINDS, check, fn, ptr

JITTER = 1e-6   # OPT:209-210
CONSTRAINT_NOISE = 1e-3   # noise of the classification GP of the constrained chooser (CONS:184)


def _ceil(x, m):
    return ((x + m - 1) // m) * m


class HyperBatch(object):
    """S hyper-samples (the reference's list of (mean, noise, amp2, ls) tuples, OPT:628) on the device."""

    def __init__(self, hyper_samples, kind, device, dtype):
        S = len(hyper_samples)
        D = len(np.atleast_1d(hyper_samples[0][3]))
        mean = np.array([h[0] for h in hyper_samples], dtype=np.float64)
        noise = np.array([h[1] for h in hyper_samples], dtype=np.float64)
        amp2 = np.array([h[2] for h in hyper_samples], dtype=np.float64)
        ls = np.vstack([np.atleast_1d(h[3]) for h in hyper_samples]).astype(np.float64)
        if kind == "SE":            # gp.SE overwrites ls with ones (gp.py:88)
            ls = np.ones_like(ls)
        host = np.concatenate([mean, noise, amp2, (1.0 / ls).ravel()])
        dev = torch.from_numpy(host).to(device=device, dtype=dtype, non_blocking=False)
        self.S, self.D = S, D
        self.mean, self.noise, self.amp2 = dev[:S], dev[S:2 * S], dev[2 * S:3 * S]
        self.inv_ls = dev[3 * S:].view(S, D)
        self.host_mean, self.host_noise, self.host_amp2, self.host_ls = mean, noise, amp2, ls
        self.nbytes = host.size * (8 if dtype == torch.float64 else 4)

    def slice(self, a, b):
        """Samples a..b-1 as a HyperBatch of their own (views of the same device memory)."""
        o = object.__new__(HyperBatch)
        o.S, o.D = b - a, self.D
        o.mean, o.noise, o.amp2, o.inv_ls = self.mean[a:b], self.noise[a:b], self.amp2[a:b], self.inv_ls[a:b]
        o.host_mean, o.host_noise = self.host_mean[a:b], self.host_noise[a:b]
        o.host_amp2, o.host_ls = self.host_amp2[a:b], self.host_ls[a:b]
        o.nbytes = 0
        return o


class Factor(object):
    """Batched Cholesky factors of K_s = amp2_s (k + 1e-6 I) + noise_s I for S hyper-samples."""

    def __init__(self, eng, kind, X, hb, L=None, winv=None, info=None, factor_impl=None):
        self.eng, self.kind, self.hb = eng, kind, hb
        self.factor_impl = factor_impl or eng.factor_impl
        self.X = X
        self.N, self.D = X.shape
        self.Npad = _ceil(self.N, 128)
        S, dt, dev = hb.S, eng.dtype, eng.device
        NB = eng.NB
        self._owned = []
        self.L = L if L is not None else self._take((S, self.Npad, self.Npad))
        self.winv = winv if winv is not None else self._take((S, self.Npad // NB, NB, NB))
        self.info = info if info is not None else torch.zeros((S,), dtype=torch.int32, device=dev)
        st = eng.stream()
        check(fn("smk_cov_build", dt)(KINDS[kind], self.N, self.N, self.D, S, ptr(X), None, ptr(hb.inv_ls),
                                      ptr(hb.amp2), ptr(hb.noise), ptr(self.L), self.Npad, st), "cov_build")
        if self.factor_impl == "tc" and dt == torch.float32 and self.Npad >= 256:
            L = _lib.lib()
            nb = 2 * S * self.Npad * self.Npad * 4
            ws = eng.take((nb,), torch.uint8)
            if eng.fused_inverse:
                # factor and explicit inverse in one pipelined call (the inverse runs one block step behind on a second
                # stream): every consumer of a tensor-core factor needs the inverse anyway
                Np = L.smk_tc_np(self.N)
                hi = self._take((S, Np, Np), torch.float32)
                lo = self._take((S, Np, Np), torch.float32)
                nt = L.smk_trtri_tc_workspace_bytes(self.Npad, Np, S)
                wt = eng.take((nt,), torch.uint8)
                check(L.smk_potrf_trtri_tc_f32(self.Npad, Np, S, ptr(self.L), ptr(self.winv), ptr(self.info), ptr(ws), nb,
                                               ptr(hi), ptr(lo), ptr(wt), nt, st), "potrf_trtri_tc")
                eng.give(ws, wt)              # scratch of this call only (the call joins back into st: stream-ordered reuse)
                self._linv = (hi, lo, Np)
            else:
                eng.give(ws)                  # scratch of this call only (stream-ordered reuse)
                check(L.smk_potrf_lower_batched_tc_f32(self.Npad, S, ptr(self.L), ptr(self.winv), ptr(self.info),
                                                       ptr(ws), nb, st), "potrf_tc")
        else:
            check(fn("smk_potrf_lower_batched", dt)(self.Npad, S, ptr(self.L), ptr(self.winv), ptr(self.info), st),
                  "potrf")

    def _take(self, shape, dtype=None):
        t = self.eng.take(shape, dtype)
        self._owned.append(t)
        return t

    def __del__(self):
        try:
            self.eng.give(*self._owned)      # back to the engine's free list; later work is stream-ordered behind ours
        except Exception:
            pass

    def linv(self):
        """(hi, lo, Np): explicit inverse of the factor as a tf32 hi/lo pair of float32 arrays; computed once."""
        if getattr(self, "_linv", None) is None:
            eng, L = self.eng, _lib.lib()
            S = self.hb.S
            Np = L.smk_tc_np(self.N)
            hi = self._take((S, Np, Np), torch.float32)
            lo = self._take((S, Np, Np), torch.float32)
            if self.factor_impl == "tc" and self.Npad >= 256:
                nb = L.smk_trtri_tc_workspace_bytes(self.Npad, Np, S)
                ws = eng.take((nb,), torch.uint8)
                eng.give(ws)
                check(L.smk_trtri_split_tc_f32(self.Npad, Np, S, ptr(self.L), ptr(self.winv), ptr(hi), ptr(lo), ptr(ws),
                                               nb, eng.stream()), "trtri_split_tc")
            else:
                nb = L.smk_trtri_workspace_bytes(Np, S)
                ws = eng.take((nb,), torch.uint8)
                eng.give(ws)
                check(L.smk_trtri_split_f32(self.Npad, Np, S, ptr(self.L), ptr(self.winv), ptr(hi), ptr(lo), ptr(ws),
                                            nb, eng.stream()), "trtri_split")
            self._linv = (hi, lo, Np)
        return self._linv

    def linv16(self):
        """(h16, l16, exps, Np): the GEMM operand copy of the inverse -- per-sample power-of-two scale 2^exps[s] and the
        fp16 (hi, lo) pair consumed by the 3xFP16 tensor-core predict; computed once."""
        if getattr(self, "_linv16", None) is None:
            eng, L = self.eng, _lib.lib()
            hi, lo, Np = self.linv()
            S = self.hb.S
            h16 = self._take((S, Np, Np), torch.float16)
            l16 = self._take((S, Np, Np), torch.float16)
            exps = torch.empty((2 * S,), dtype=torch.int32, device=eng.device)
            check(L.smk_linv_pack_f16(Np, S, ptr(hi), ptr(lo), ptr(h16), ptr(l16), ptr(exps), eng.stream()),
                  "linv_pack_f16")
            self._linv16 = (h16, l16, exps, Np)
        return self._linv16

    def alpha_via_linv(self, y):
        """alpha = Linv^T Linv (y - mean), [S][1][Npad]; needs the explicit inverse (tensor-core predict path)."""
        eng, L = self.eng, _lib.lib()
        hi, lo, Np = self.linv()
        S = self.hb.S
        alpha = torch.empty((S, 1, self.Npad), dtype=torch.float32, device=eng.device)
        tmp = torch.empty((S, Np), dtype=torch.float32, device=eng.device)
        check(L.smk_linv_alpha_f32(self.N, Np, S, ptr(hi), ptr(lo), ptr(y), ptr(self.hb.mean), ptr(alpha), self.Npad,
                                   ptr(tmp), eng.stream()), "linv_alpha")
        self._z = tmp          # z = Linv (y - mean): the predict GEMM reduces the mean from it (mu - mean = z . beta)
        return alpha

    def guard(self, rows):
        """[S] float32 on the device: estimated relative error of the predictive variance at a candidate sitting on one of
        the observed points ``rows`` (4 indices: the incumbents) if the explicit inverse is used (csrc/guard.cu)."""
        eng, L = self.eng, _lib.lib()
        hi, lo, Np = self.linv()
        S = self.hb.S
        g = torch.empty((S,), dtype=torch.float32, device=eng.device)
        rows = torch.as_tensor(np.resize(np.asarray(rows, dtype=np.int32), 4), device=eng.device)
        nb = L.smk_tc_guard_workspace_bytes(Np, S)
        ws = eng.take((nb,), torch.uint8)
        eng.give(ws)
        check(L.smk_tc_guard_f32(self.N, self.Npad, Np, S, ptr(self.L), ptr(hi), ptr(lo), ptr(self.hb.amp2),
                                 ptr(self.hb.noise), ptr(rows), ptr(g), ptr(ws), nb, eng.stream()), "tc_guard")
        return g

    def check_pd(self):
        """The reference lets spla.cholesky raise LinAlgError (SURVEY 8b 'Errors'); so do we."""
        info = self.info.cpu().numpy()
        if np.any(info != 0):
            s = int(np.nonzero(info)[0][0])
            raise np.linalg.LinAlgError("%d-th leading minor of the array is not positive definite "
                                        "(hyper-sample %d)" % (int(info[s]), s))

    def solve(self, y, F=1, y_stride=0, ldy=None, n_lead=None, want_alpha=True, want_logdet=False,
              want_quad=False, subtract_mean=True):
        """alpha = K^-1 (y - mean) for F right-hand sides; optionally sum log diag(L) and the quadratic form.

        ``n_lead`` < N solves against the leading n_lead x n_lead block of the factor (OPT:574)."""
        eng, hb = self.eng, self.hb
        S, dt, dev = hb.S, eng.dtype, eng.device
        n = self.N if n_lead is None else n_lead
        rb, nb_ = (4, 128) if dt == torch.float32 else (2, 64)
        if eng.esize * (rb * self.Npad + rb * nb_ + (256 // nb_) * rb * nb_) > 227 * 1024:
            raise _lib.SmkError("chol_solve keeps its right-hand sides in shared memory: N = %d exceeds its limit (about "
                                "%d for this element type); use the explicit-inverse path" % (self.N, 227 * 1024 // (eng.esize * rb)))
        alpha = torch.empty((S, F, self.Npad), dtype=dt, device=dev) if want_alpha else None
        sld = torch.empty((S,), dtype=dt, device=dev) if want_logdet else None
        quad = torch.empty((S, F), dtype=dt, device=dev) if want_quad else None
        check(fn("smk_chol_solve", dt)(n, self.Npad, S, F, ptr(self.L), ptr(self.winv), ptr(y), y_stride,
                                       ldy if ldy is not None else n, ptr(hb.mean) if subtract_mean else None,
                                       ptr(alpha), ptr(sld), ptr(quad), eng.stream()), "chol_solve")
        return alpha, sld, quad


class _LeadingView(object):
    """A Factor-like view exposing only the first N rows of a joint factor's inputs (for cross_mean)."""

    def __init__(self, fac, X, N):
        self.hb, self.X, self.N, self.D, self.Npad = fac.hb, X, N, fac.D, fac.Npad
        self.L, self.winv = fac.L, fac.winv


class Prepared(object):
    """Everything about one chunk of hyper-samples that does not depend on the candidate set:
    factors, alpha (one column, or F fantasy columns), bests, optional time-GP factor and alpha."""
    pass


class GPEIEngine(object):
    """One engine per process / GPU and element type.  float32 is the grid path."""

    def __init__(self, device=None, dtype=torch.float32):
        if not torch.cuda.is_available():
            raise _lib.SmkError("spearmint_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        _lib.lib()
        self.device = torch.device(device if device is not None else "cuda:%d" % torch.cuda.current_device())
        torch.cuda.set_device(self.device)
        self.dtype = dtype
        self.esize = 8 if dtype == torch.float64 else 4
        self.NB = _lib.lib().smk_block(self.esize)
        self._ws = None
        self._ws_tc = None
        # fused-predict implementation: "tc" = wgmma/TMA 3xFP16 kernel (float32 in/out), "simt" = register-tiled FMA
        self.predict_impl = os.environ.get("SMK_PREDICT_IMPL", "tc" if dtype == torch.float32 else "simt")
        if dtype != torch.float32:
            self.predict_impl = "simt"
        # N^3 steps (Cholesky trailing update, triangular inverse): "tc" = wgmma 3xTF32 left-looking variants
        self.factor_impl = os.environ.get("SMK_FACTOR_IMPL", "tc" if self.predict_impl == "tc" else "simt")
        # The explicit-inverse tensor-core chain is the path for LARGE factors.  Below tc_min_n observations the float32
        # blocked-substitution chain (SIMT Cholesky + SIMT predict) is used: it is 3-8x more accurate on the smooth,
        # ill-conditioned problems small N goes with (C2 / C4: 1.5e-3 against 8e-3 ... 1.2e-2 of max EI, DESIGN.md section 6)
        # and at that size it costs milliseconds.
        self.tc_min_n = int(os.environ.get("SMK_TC_MIN_N", "2048"))
        # opt-in accuracy guard of the tensor-core chain (csrc/guard.cu, _guarded_impl): a hyper-sample whose ESTIMATED EI
        # error exceeds this fraction of its EI scale is re-evaluated in float64.  The estimate is conservative (it
        # over-predicts the actual error), so it is off by default (0) and meant for users whose problems are both large
        # and badly conditioned.
        self.guard_threshold = float(os.environ.get("SMK_TC_GUARD", "0"))
        self.last = {}
        self._deferred_info = []
        self._chunk_cache = {}
        self.last_guard = None
        self.timers = None   # set to {} to record (start, end) CUDA events per stage on the launch stream
        self._pool = {}      # (stream, shape, dtype) -> free tensors: the big per-call buffers are recycled, never re-allocated
        self._home = {}      # data_ptr -> stream the buffer belongs to
        self._side = None    # second stream: the factor chain of one half of the samples runs under the other half's GEMM
        # the persistent GEMM and the generator leave no SM for the side stream's kernels to run on, and two groups double the
        # launches.  Off unless asked for.
        self.overlap = os.environ.get("SMK_FACTOR_OVERLAP", "0") == "1"
        # tensor-core chain: factorisation and explicit inverse as one pipelined call (csrc/predict_tc.cu: potrf_trtri_tc);
        # SMK_FUSED_INVERSE=0 runs them one after the other (the two separate entry points)
        self.fused_inverse = os.environ.get("SMK_FUSED_INVERSE", "1") == "1"
        # Opt-in (SMK_MEAN_FROM_GEMM=1, SMK_PREGEN=1): predictive mean reduced in the GEMM epilogue (mu - mean = z . beta,
        # z = Linv (y - mean)) instead of in the generator (alpha . kx) -- the generator then depends on nothing the
        # factorisation produces, and the first candidate chunk is generated on a second stream WHILE K is factored and
        # inverted.  The generator then competes with the factorisation's small kernels, and the mean inherits the
        # tensor-core accumulation error of beta: accuracy first, so both stay off.
        self.mean_from_gemm = os.environ.get("SMK_MEAN_FROM_GEMM", "0") == "1"
        self.pregen_enabled = self.mean_from_gemm and os.environ.get("SMK_PREGEN", "0") == "1"
        self._helper64 = None

    # ------------------------------------------------------------------ buffers
    def take(self, shape, dtype=None):
        """A device buffer of exactly this shape from the engine's free list (allocated on first use only).  The C library
        never allocates; this is the host-side mirror of that rule: steady-state calls reuse the same HBM."""
        # one free list per stream: a buffer given back right after its last launch may be taken again at once, which is
        # only ordered correctly among launches of the SAME stream
        key = (torch.cuda.current_stream(self.device).cuda_stream, tuple(int(x) for x in shape), dtype or self.dtype)
        free = self._pool.get(key)
        if free:
            return free.pop()
        try:
            t = torch.empty(key[1], dtype=key[2], device=self.device)
        except torch.cuda.OutOfMemoryError:
            self.trim()                       # buffers of other shapes are the only thing the pool can be blamed for
            t = torch.empty(key[1], dtype=key[2], device=self.device)
        self._home[t.data_ptr()] = key[0]
        return t

    def trim(self):
        self._pool.clear()
        self._home.clear()
        torch.cuda.empty_cache()

    def pooled_bytes(self):
        return sum(t.numel() * t.element_size() for v in self._pool.values() for t in v)

    def give(self, *tensors):
        for t in tensors:
            if t is not None:          # back to the free list of the stream it was taken on
                home = self._home.get(t.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)
                self._pool.setdefault((home, tuple(t.shape), t.dtype), []).append(t)

    def helper64(self):
        """The float64 engine on the same device (pending-point conditionals, deep-tail re-evaluation)."""
        if self.dtype == torch.float64:
            return self
        if self._helper64 is None:
            self._helper64 = GPEIEngine(device=self.device, dtype=torch.float64)
        return self._helper64

    # ------------------------------------------------------------------ timing helpers
    def _t0(self):
        if self.timers is None:
            return None
        e = torch.cuda.Event(enable_timing=True)
        e.record(torch.cuda.current_stream(self.device))
        return e

    def _t1(self, name, e0):
        if e0 is None:
            return
        e1 = torch.cuda.Event(enable_timing=True)
        e1.record(torch.cuda.current_stream(self.device))
        self.timers.setdefault(name, []).append((e0, e1))

    def stage_ms(self):
        """Sum of recorded stage durations in ms (call after a synchronize)."""
        return {k: sum(a.elapsed_time(b) for a, b in v) for k, v in (self.timers or {}).items()}

    # ------------------------------------------------------------------ plumbing
    def stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def to_dev(self, a):
        a = np.ascontiguousarray(a, dtype=np.float64)
        return torch.from_numpy(a).to(device=self.device, dtype=self.dtype)

    def workspace(self, nbytes):
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = torch.empty((nbytes,), dtype=torch.uint8, device=self.device)
        return self._ws

    def max_samples_per_chunk(self, Npad, ldm, F=1):
        """How many hyper-samples fit at once in ~70% of free HBM: factor + winv + alpha + mu/var/ei per sample, plus --
        on the tensor-core path -- the explicit inverse (tf32 pair, fp16 pair, the transposed pair of the inversion
        workspace: 20 B per element of Np^2) and the cross-covariance chunk (4 B per (candidate, observation) and
        sample, capped by the library's 20 GB chunk budget)."""
        # cudaMemGetInfo is a driver call that can take milliseconds next to a busy GPU (and it is on the path of every
        # sweep): asked again only when the allocator's own counter moved by more than 1 GB since the last answer
        alloc = torch.cuda.memory_allocated(self.device)
        key = (Npad, ldm, F)
        hit = self._chunk_cache.get(key)
        if hit is not None and abs(alloc - hit[0]) < (1 << 30):
            return hit[1]
        ans = self._max_samples_per_chunk(Npad, ldm, F)
        self._chunk_cache[key] = (alloc, ans)
        return ans

    def _max_samples_per_chunk(self, Npad, ldm, F):
        free, _ = torch.cuda.mem_get_info(self.device)
        free += torch.cuda.memory_reserved(self.device) - torch.cuda.memory_allocated(self.device)
        free += self.pooled_bytes()           # recycled (or dropped by take() on demand)
        budget = 0.7 * free
        per = self.esize * (Npad * Npad + Npad * self.NB + F * Npad + (F + 3) * ldm)
        if self.predict_impl == "tc" and self.dtype == torch.float32:
            Np = _ceil(Npad, 256)
            per += 20 * Np * Np + (8 * Npad * Npad if self.fused_inverse else 0)   # + the factorisation's tf32 panel copies, live next to the inversion's workspace
            per_kxt = 4.0 * ldm * Np + 4.0 * (Np // 512 + 1) * ldm      # operand chunk + row-group-pair partials
            cap = float(21 << 30)
            s1 = budget / (per + per_kxt)
            if s1 * per_kxt <= cap:
                return max(1, int(s1))
            return max(1, int((budget - cap) // per))
        fixed = _lib.lib().smk_predict_workspace_bytes(self.esize, Npad)
        return max(1, int((budget - fixed) // per))

    # ------------------------------------------------------------------ building blocks
    def hypers(self, hyper_samples, kind):
        return HyperBatch(hyper_samples, kind, self.device, self.dtype)

    def factor(self, kind, X, hb, **kw):
        return Factor(self, kind, X, hb, **kw)

    def chain_for(self, n):
        """("tc" | "simt") for a factor of n observations: the tensor-core chain from tc_min_n on, else blocked substitution."""
        if self.predict_impl == "tc" and self.dtype == torch.float32 and n >= self.tc_min_n:
            return "tc"
        return "simt"

    def cov(self, kind, hb, X, Y=None):
        """Batched chooser.cov (OPT:207-212): returns [S][N][N] (self, jitter included, no noise) or [S][N][M]."""
        N, D = X.shape
        dt = self.dtype
        if Y is None:
            out = torch.empty((hb.S, N, N), dtype=dt, device=self.device)
            check(fn("smk_cov_build", dt)(KINDS[kind], N, N, D, hb.S, ptr(X), None, ptr(hb.inv_ls), ptr(hb.amp2),
                                          None, ptr(out), N, self.stream()), "cov_build")
        else:
            M = Y.shape[0]
            out = torch.empty((hb.S, N, M), dtype=dt, device=self.device)
            check(fn("smk_cov_build", dt)(KINDS[kind], N, M, D, hb.S, ptr(X), ptr(Y), ptr(hb.inv_ls),
                                          ptr(hb.amp2), None, ptr(out), M, self.stream()), "cov_build")
        return out

    def pregen(self, kind, X_dev, C_dev, hb, F=1):
        """Queues the cross-covariance operand of the first candidate chunk on the library's generator stream (forked from
        ours) and returns C_dev as the token ei_prepared() hands back to predict(); None if this shape is not pre-generated
        (two-buffer chunking)."""
        L = _lib.lib()
        N, D = X_dev.shape
        M = C_dev.shape[0]
        Np = L.smk_tc_np(N)
        nb = L.smk_predict_tc_workspace_bytes(Np, M, hb.S, F)
        if self._ws_tc is None or self._ws_tc.numel() < nb:
            self._ws_tc = None
            self._ws_tc = torch.empty((nb,), dtype=torch.uint8, device=self.device)
        rc = L.smk_predict_tc_pregen_f32(KINDS[kind], N, Np, M, D, hb.S, ptr(X_dev), ptr(C_dev), ptr(hb.inv_ls), ptr(hb.amp2),
                                         ptr(self._ws_tc), self._ws_tc.numel(), F, self.stream())
        if rc == -22:
            return None
        check(rc, "predict_tc_pregen")
        return C_dev

    def predict(self, kind, fac, C_dev, alpha, impl=None, dbg_beta=None, alpha_f=None, F=1, pregenerated=False):
        """Predictive mean / variance at the candidates for every sample of the factor batch.  With ``alpha_f``
        ([S][F][Npad], tensor-core path) also the F fantasy means, returned as a third tensor [S][F][ldm].
        ``pregenerated``: the first candidate chunk's cross-covariance was queued by pregen() for exactly these inputs."""
        hb, dt = fac.hb, self.dtype
        M = C_dev.shape[0]
        ldm = _ceil(M, 128)
        mu = torch.empty((hb.S, ldm), dtype=dt, device=self.device)
        var = torch.empty((hb.S, ldm), dtype=dt, device=self.device)
        if (impl or self.predict_impl) == "tc" and isinstance(fac, Factor):
            L = _lib.lib()
            h16, l16, lexp, Np = fac.linv16()
            nb = L.smk_predict_tc_workspace_bytes(Np, M, hb.S, F if alpha_f is not None else 1)
            if self._ws_tc is None or self._ws_tc.numel() < nb:
                self._ws_tc = None
                self._ws_tc = torch.empty((nb,), dtype=torch.uint8, device=self.device)
            mu_f = torch.empty((hb.S, F, ldm), dtype=dt, device=self.device) if alpha_f is not None else None
            z = getattr(fac, "_z", None) if self.mean_from_gemm else None
            check(L.smk_predict_tc_f32(KINDS[kind], fac.N, Np, M, fac.D, hb.S, ptr(fac.X), ptr(C_dev), ptr(hb.inv_ls),
                                       ptr(hb.amp2), ptr(hb.mean), ptr(h16), ptr(l16), ptr(lexp), ptr(alpha), fac.Npad,
                                       ptr(mu), ptr(var), ldm, ptr(self._ws_tc), nb, ptr(dbg_beta),
                                       F if alpha_f is not None else 1, ptr(alpha_f), ptr(mu_f), ptr(z),
                                       1 if (pregenerated and z is not None) else 0, self.stream()),
                  "predict_tc")
            if alpha_f is not None:
                return mu, var, ldm, mu_f
            return mu, var, ldm
        nb = _lib.lib().smk_predict_workspace_bytes(self.esize, fac.Npad)
        ws = self.workspace(nb)
        check(fn("smk_predict", dt)(KINDS[kind], fac.N, fac.Npad, M, fac.D, hb.S, ptr(fac.X), ptr(C_dev),
                                    ptr(hb.inv_ls), ptr(hb.amp2), ptr(hb.mean), ptr(fac.L), ptr(fac.winv),
                                    ptr(alpha), ptr(mu), ptr(var), ldm, ptr(ws), nb, self.stream()), "predict")
        return mu, var, ldm

    def cross_mean(self, kind, fac, C_dev, alpha, F):
        hb, dt = fac.hb, self.dtype
        M = C_dev.shape[0]
        ldm = _ceil(M, 128)
        mu = torch.empty((hb.S, F, ldm), dtype=dt, device=self.device)
        check(fn("smk_cross_mean", dt)(KINDS[kind], fac.N, fac.Npad, M, fac.D, hb.S, F, ptr(fac.X), ptr(C_dev),
                                       ptr(hb.inv_ls), ptr(hb.amp2), ptr(hb.mean), ptr(alpha), ptr(mu), ldm,
                                       self.stream()), "cross_mean")
        return mu

    def ei_sweep(self, M, S, F, mu, var, ldm, best, log_time=None, want_ei=True, ei_sum=None, ei_max=None, accumulate=True):
        dt = self.dtype
        ei = torch.empty((S, ldm), dtype=torch.float64, device=self.device) if want_ei else None   # EI is always double
        if ei_sum is None and accumulate:
            ei_sum = torch.zeros((ldm,), dtype=torch.float64, device=self.device)
        check(fn("smk_ei_sweep", dt)(M, S, F, ptr(mu), ptr(var), ldm, ptr(best), ptr(log_time), ptr(ei),
                                     ptr(ei_sum) if accumulate else None, ptr(ei_max), self.stream()), "ei_sweep")
        return ei, ei_sum

    def ei_sweep_weighted(self, M, S, F, mu, var, ldm, best, w, want_ei=True, ei_sum=None):
        """ei_sweep with each per-sample EI multiplied by w[s][j] (double [S][ldm]), CONS:878 / 940."""
        ei = torch.empty((S, ldm), dtype=torch.float64, device=self.device) if want_ei else None
        if ei_sum is None:
            ei_sum = torch.zeros((ldm,), dtype=torch.float64, device=self.device)
        check(fn("smk_ei_sweep_weighted", self.dtype)(M, S, F, ptr(mu), ptr(var), ldm, ptr(best), ptr(w), ptr(ei),
                                                      ptr(ei_sum), None, self.stream()), "ei_sweep_weighted")
        return ei, ei_sum

    def topk(self, score, M, k):
        """Indices of the k largest scores, ascending (argsort(score)[-k:], OPT:270; [-1] is the argmax, OPT:294).
        The device selection handles k <= 256 per call; larger k (the reference accepts any grid_subset) takes several
        rounds, each masking what the previous ones took."""
        dt = score.dtype                      # EI scores are float64 (see ei_sweep)
        K = 256
        if k <= K:
            idx, val = self._topk_once(score, M, k)
        else:
            work = score[:M].clone()
            parts_i, parts_v = [], []
            left = k
            while left > 0:
                kk = min(K, left)
                i, v = self._topk_once(work, M, kk)           # ascending
                parts_i.append(i)
                parts_v.append(v)
                work[i.long()] = float("-inf")
                left -= kk
            idx = torch.cat(parts_i[::-1])                   # later rounds hold smaller scores
            val = torch.cat(parts_v[::-1])
        return idx, val

    def _topk_once(self, score, M, k):
        dt = score.dtype
        nb = _lib.lib().smk_topk_workspace_bytes(M, k)
        ws = torch.empty((nb,), dtype=torch.uint8, device=self.device)
        idx = torch.empty((k,), dtype=torch.int32, device=self.device)
        val = torch.empty((k,), dtype=dt, device=self.device)
        check(fn("smk_topk", dt)(M, k, ptr(score), ptr(idx), ptr(val), ptr(ws), nb, self.stream()), "topk")
        return idx, val

    # ------------------------------------------------------------------ candidate-independent state
    def prepare(self, kind, hyper_samples, comp, pend, vals, normals=None, time_hyper_samples=None, durs_log=None,
                resident=None, cand_dev=None):
        """Factor + alpha (+ fantasies, + time GP) for one chunk of hyper-samples.  ``resident`` = dict(X, y, best,
        hb) of tensors already in HBM (the bench's `value` leg).  ``cand_dev``: the candidates the first sweep will be
        over, if known -- their cross-covariance is then generated while the factorisation runs."""
        p = Prepared()
        p.pregen = None
        p.kind = kind
        p.host = dict(hyper_samples=hyper_samples, comp=comp, pend=pend, vals=vals, normals=normals,
                      time_hyper_samples=time_hyper_samples, durs_log=durs_log)
        p.gbound, p.flagged, p.prep64 = None, None, None
        P = 0 if pend is None else int(pend.shape[0])
        if resident is not None:
            Xo, yd, best_val = resident["X"], resident["y"], resident["best"]
            hb = resident.get("hb") or self.hypers(hyper_samples, kind)
        else:
            Xo, yd, best_val = self.to_dev(comp), self.to_dev(vals), float(np.min(vals))
            hb = self.hypers(hyper_samples, kind)
        p.hb, p.N, p.P, p.S = hb, Xo.shape[0], P, hb.S
        p.time = None
        if time_hyper_samples is not None:          # PSEC:442-459
            thb = self.hypers(time_hyper_samples, kind)
            tfac = self.factor(kind, Xo, thb)
            ta, _, _ = tfac.solve(self.to_dev(durs_log), F=1)
            p.time = (tfac, ta)
        if P == 0:
            t = self._t0()
            chain = self.chain_for(Xo.shape[0])
            if (cand_dev is not None and chain == "tc" and self.factor_impl == "tc" and self.pregen_enabled
                    and self.guard_threshold <= 0):
                p.pregen = self.pregen(kind, Xo, cand_dev, hb)
            fac = self.factor(kind, Xo, hb, factor_impl=chain if self.factor_impl == "tc" else "simt")
            self._t1("cov_potrf", t)
            t = self._t0()
            p.impl = self._guarded_impl(fac, p) if chain == "tc" else "simt"
            if p.impl == "tc":
                alpha = fac.alpha_via_linv(yd)       # explicit inverse (trtri, once per factor batch) + two mat-vecs
            else:
                alpha, _, _ = fac.solve(yd, F=1)
            self._t1("linv_alpha" if p.impl == "tc" else "chol_solve", t)
            p.fac, p.alpha, p.F = fac, alpha, 1
            p.bests = torch.full((hb.S, 1), best_val, dtype=self.dtype, device=self.device)
            p.bests_host = np.full((hb.S, 1), best_val)
            p.pred_alpha = alpha.view(hb.S, fac.Npad)
        else:
            if comp is None:
                raise _lib.SmkError("pending points need the host arrays (comp, pend, vals), not resident tensors")
            self._prepare_pending(p, kind, hb, hyper_samples, Xo, self.to_dev(pend), yd, np.asarray(comp, float),
                                  np.asarray(pend, float), np.asarray(vals, float), np.asarray(normals, float))
        return p

    def _guarded_impl(self, fac, p):
        """Arms the accuracy guard of the explicit-inverse (tensor-core) predict for this factor batch.

        csrc/guard.cu measures g_s = relative variance error the path makes for a candidate sitting on the data.  The EI
        of such a candidate (s^2 ~ noise + jitter, u ~ 0) then moves by about  0.5 phi(0) g sqrt(noise + 1e-6 amp2), which
        is kept per sample as the absolute bound p.gbound[s].  After every sweep the bound is compared with the largest EI
        of the sample (ei_prepared): a sample whose bound exceeds guard_threshold * max EI is re-evaluated on the float64
        engine.  Well-conditioned problems (the headline) do not trip it; smooth low-dimensional ones (C2, C4) do."""
        p.gbound, p.flagged, p.prep64 = None, None, None
        if self.guard_threshold > 0:
            # probes: the observed points with the lowest values -- the incumbent (the chooser's jitter cloud sits on it) and
            # its runners-up, where EI concentrates
            vals = p.host.get("vals")
            rows = np.argsort(vals)[:4] if vals is not None else [fac.N - 1]
            rows = [int(r) for r in rows if r < fac.N]
            g = fac.guard(rows).double().cpu().numpy()                   # one small read per factor batch
            hb = fac.hb
            p.gbound = 0.2 * g * np.sqrt(hb.host_noise + JITTER * hb.host_amp2)
            self.last_guard = dict(g_max=float(g.max()), bound_max=float(p.gbound.max()))
        return "tc"

    def _prepare_pending(self, p, kind, hb, hyper_samples, Xo, Pd, yd, comp, pend, vals, normals):
        """Pending-fantasy prologue (OPT:558-603) for one chunk of hyper-samples.

        The P x P conditional of the pending points (pend_m, pend_K, OPT:577-585) is formed from a FLOAT64 joint
        factor: pend_K = Lpp Lpp' - noise I cancels down to the 1e-6 amp2 jitter when a pending point sits next to an
        observation (the 1e-3 jitter cloud next() itself proposes) or duplicates another pending point, and float32
        rounding of the joint factor is of that order -- the reference's float64 succeeds there, so must we.  The
        fantasy draw uses the host with the caller's normals (the host RNG order is the reference's).  The float32
        joint factor of the grid path and the F fantasy right-hand sides stay on the float32 engine."""
        N, P, F = Xo.shape[0], Pd.shape[0], normals.shape[-1]
        S = hb.S
        per_sample = (normals.ndim == 3)     # (S,P,F): GPEIChooser draws fresh normals per hyper-sample (GPEI:237)
        h64 = self.helper64()
        hb64 = hb if h64 is self else h64.hypers(hyper_samples, kind)
        Xo64, Pd64 = h64.to_dev(comp), h64.to_dev(pend)
        Xj64 = torch.cat([Xo64, Pd64], dim=0).contiguous()
        fac64 = h64.factor(kind, Xj64, hb64)
        fac64.check_pd()                                       # LinAlgError like OPT:567
        # alpha of the observed-only system from the leading N x N block of the joint factor (OPT:574-577)
        a_obs, _, _ = fac64.solve(h64.to_dev(vals), F=1, n_lead=N)
        # pend_m = pend_cross' alpha + mean (OPT:581): cross mean of the observed set at the P pending points
        pend_m = h64.cross_mean(kind, _LeadingView(fac64, Xo64, N), Pd64, a_obs, 1)[:, 0, :P].cpu().numpy()   # (S,P)
        # pend_K = Schur complement - noise I, from the trailing P x P block of the joint factor (OPT:582)
        Lpp = fac64.L[:, N:N + P, N:N + P].cpu().numpy()
        fant = np.empty((S, F, N + P))
        bests = np.empty((S, F))
        for s in range(S):
            Lp = np.tril(Lpp[s])
            pend_K = Lp.dot(Lp.T) - hb.host_noise[s] * np.eye(P)
            pend_chol = np.linalg.cholesky(pend_K)                                # LinAlgError like OPT:585
            pf = pend_chol.dot(normals[s] if per_sample else normals) + pend_m[s][:, None]   # (P,F)  OPT:589
            fant[s, :, :N] = vals[None, :]
            fant[s, :, N:] = pf.T
            bests[s] = np.minimum(vals.min(), pf.min(axis=0))                     # OPT:597
        chain = self.chain_for(N + P)
        if h64 is self:
            fac = fac64
        else:
            del fac64
            fac = self.factor(kind, torch.cat([Xo, Pd], dim=0).contiguous(), hb,
                              factor_impl=chain if self.factor_impl == "tc" else "simt")
            fac.check_pd()
        fant_d = self.to_dev(fant)                                                # [S][F][N+P]
        alpha_f, _, _ = fac.solve(fant_d, F=F, y_stride=F * (N + P), ldy=N + P)   # OPT:603
        p.fac, p.alpha, p.F = fac, alpha_f, F
        p.impl = self._guarded_impl(fac, p) if chain == "tc" else "simt"
        p.bests, p.bests_host = self.to_dev(bests), bests
        p.pred_alpha = torch.zeros((S, fac.Npad), dtype=self.dtype, device=self.device)

    def ei_prepared(self, p, Cd, want_matrix=True, ei_sum=None, cand_host=None, weight=None):
        """EI of every candidate in Cd for every sample of a Prepared chunk.  Returns (ei [S][ldm] | None, ei_sum).
        ``cand_host``: the float64 candidates behind Cd (used only if the accuracy guard re-evaluates a sample).
        ``weight``: double [S][ldm] that multiplies each sample's EI (the constrained pass's probability of feasibility)."""
        kind, fac, hb = p.kind, p.fac, p.hb
        M = Cd.shape[0]
        ldm = _ceil(M, 128)
        log_time = None
        if p.time is not None:
            tfac, ta = p.time
            log_time = self.cross_mean(kind, tfac, Cd, ta, 1).view(tfac.hb.S, ldm)
        t = self._t0()
        impl = getattr(p, "impl", None) or self.predict_impl
        if p.P > 0 and impl == "tc" and p.F > 1:
            _, var, _, mu = self.predict(kind, fac, Cd, p.pred_alpha, impl=impl, alpha_f=p.alpha, F=p.F)   # OPT:605-610
        else:
            pre = getattr(p, "pregen", None)
            p.pregen = None
            pre = pre is not None and pre.data_ptr() == Cd.data_ptr() and impl == "tc"
            mu, var, _ = self.predict(kind, fac, Cd, p.pred_alpha, impl=impl, pregenerated=pre)   # OPT:544-548 / 605-610
            if p.P > 0:
                mu = self.cross_mean(kind, fac, Cd, p.alpha, p.F)                  # OPT:609
            else:
                mu = mu.view(hb.S, 1, ldm)
        self._t1("predict", t)
        t = self._t0()
        guarded = p.gbound is not None and p.host.get("comp") is not None
        if weight is not None:
            if guarded or log_time is not None:
                raise _lib.SmkError("the probability-weighted sweep has no accuracy guard and no per-second variant")
            out = self.ei_sweep_weighted(M, hb.S, p.F, mu, var, ldm, p.bests, weight, want_matrix, ei_sum)
            self._t1("ei_sweep", t)
            return out
        if not guarded:
            out = self.ei_sweep(M, hb.S, p.F, mu, var, ldm, p.bests, log_time, want_matrix, ei_sum)
            self._t1("ei_sweep", t)
            return out
        # ---- guarded sweep: per-sample EI and its maximum first, the sum over samples after the check
        if ei_sum is None:
            ei_sum = torch.zeros((ldm,), dtype=torch.float64, device=self.device)
        ei_max = torch.empty((hb.S,), dtype=torch.int64, device=self.device)
        ei, _ = self.ei_sweep(M, hb.S, p.F, mu, var, ldm, p.bests, log_time, True, None, ei_max=ei_max, accumulate=False)
        self._t1("ei_sweep", t)
        if p.flagged is None:                                             # decided on the first sweep of this factor batch
            # scale of each sample's EI: its own maximum, but not below the largest MEAN EI of the batch -- a sample whose EI
            # is negligible everywhere cannot move the proposal and is not worth a float64 pass
            tmp = torch.zeros((ldm,), dtype=torch.float64, device=self.device)
            check(_lib.lib().smk_ei_colsum(M, hb.S, ptr(ei), ldm, ptr(tmp), self.stream()), "ei_colsum")
            _, top = self._topk_once(tmp, M, 1)
            both = torch.cat([ei_max.view(torch.float64), top / float(hb.S)]).cpu().numpy()   # the one host read
            scale = np.maximum(both[:hb.S], both[hb.S])
            ratio = p.gbound / np.maximum(scale, 1e-300)
            p.flagged = [int(s) for s in np.nonzero(ratio > self.guard_threshold)[0]]
            self.last_guard = dict(self.last_guard or {}, flagged=len(p.flagged), S=hb.S, worst_ratio=float(ratio.max()))
        if p.flagged:
            self._reevaluate_f64(p, Cd, cand_host, ei)
        check(_lib.lib().smk_ei_colsum(M, hb.S, ptr(ei), ldm, ptr(ei_sum), self.stream()), "ei_colsum")
        return (ei if want_matrix else None), ei_sum

    def _reevaluate_f64(self, p, Cd, cand_host, ei):
        """Rows p.flagged of ei (per-sample EI of this candidate set) recomputed by the float64 build of the same kernels
        (blocked-substitution predict): what the tensor-core path cannot deliver for these samples, the reference's own
        precision can.  The float64 factors are built once per Prepared and reused by later sweeps."""
        h64 = self.helper64()
        H = p.host
        sel = p.flagged
        if cand_host is None:
            cand_host = Cd.double().cpu().numpy()
        if p.prep64 is None:
            hs = [H["hyper_samples"][s] for s in sel]
            ths = None if H["time_hyper_samples"] is None else [H["time_hyper_samples"][s] for s in sel]
            nrm = H["normals"]
            if nrm is not None and np.ndim(nrm) == 3:
                nrm = np.asarray(nrm)[sel]
            p.prep64 = h64.prepare(p.kind, hs, H["comp"], H["pend"], H["vals"], nrm, ths, H["durs_log"])
            p.prep64.fac.check_pd()
        e64, _ = h64.ei_prepared(p.prep64, h64.to_dev(cand_host), True, None)
        ei[torch.as_tensor(sel, device=self.device)] = e64

    # ------------------------------------------------------------------ whole path
    def ei_over_hypers_device(self, kind, hyper_samples, comp, pend, cand, vals, normals=None,
                              time_hyper_samples=None, durs_log=None, want_matrix=True, inputs_on_device=None,
                              defer_pd_check=False):
        """Runs the batched path; returns (ei [S][ldm] or None, ei_sum [ldm], M) as device tensors.

        ``defer_pd_check``: do not read the factorisations' status words back here (one host synchronisation per chunk);
        the caller calls check_deferred() before it uses the results -- back-to-back calls then queue without draining the GPU.

        ``normals`` (P,F): the fantasy standard normals the reference draws on the host (OPT:588-589).
        ``time_hyper_samples`` + ``durs_log``: EI per second (PSEC:437-548).
        ``inputs_on_device``: optional dict(X=, C=, y=, best=, hb=) of resident tensors (bench `value` leg)."""
        P = 0 if pend is None else int(pend.shape[0])
        S = len(hyper_samples)
        res = inputs_on_device
        Cd = res["C"] if res is not None else self.to_dev(cand)
        N = res["X"].shape[0] if res is not None else comp.shape[0]
        M = Cd.shape[0]
        ldm = _ceil(M, 128)
        Fn = 1 if P == 0 else int(normals.shape[-1])
        chunk = self.max_samples_per_chunk(_ceil(N + P, 128), ldm, Fn)
        ei_sum = torch.zeros((ldm,), dtype=torch.float64, device=self.device)
        ei_all = torch.empty((S, ldm), dtype=torch.float64, device=self.device) if want_matrix else None
        if chunk >= S and self.can_overlap(N, S, P, time_hyper_samples):
            self._two_group_pass(kind, hyper_samples, comp, cand, vals, res, Cd, want_matrix, ei_sum, ei_all)
            self.last = dict(N=N, M=M, S=S, P=P, chunk=chunk, groups=2)
            return ei_all, ei_sum, M
        for s0 in range(0, S, chunk):
            r = res if (res is not None and chunk >= S) else (dict(res, hb=None) if res is not None else None)
            nrm = normals[s0:s0 + chunk] if (normals is not None and np.ndim(normals) == 3) else normals
            prep = self.prepare(kind, hyper_samples[s0:s0 + chunk], comp, pend, vals, nrm,
                                None if time_hyper_samples is None else time_hyper_samples[s0:s0 + chunk],
                                durs_log, resident=r, cand_dev=Cd)
            ei, _ = self.ei_prepared(prep, Cd, want_matrix, ei_sum, cand_host=cand)
            if defer_pd_check:
                self._deferred_info.append(prep.fac.info)
            else:
                prep.fac.check_pd()     # one host sync per chunk, after everything is queued
            if want_matrix:
                ei_all[s0:s0 + prep.S] = ei
            del prep
        self.last = dict(N=N, M=M, S=S, P=P, chunk=chunk)
        return ei_all, ei_sum, M

    def check_deferred(self):
        """Raises numpy.linalg.LinAlgError (like spla.cholesky) if any factorisation queued with defer_pd_check failed."""
        infos, self._deferred_info = self._deferred_info, []
        for info in infos:
            bad = np.nonzero(info.cpu().numpy())[0]
            if bad.size:
                raise np.linalg.LinAlgError("%d-th leading minor of the array is not positive definite (hyper-sample %d)"
                                            % (int(info[int(bad[0])]), int(bad[0])))

    def can_overlap(self, N, S, P, time_hyper_samples):
        return (self.overlap and S >= 4 and P == 0 and time_hyper_samples is None and self.chain_for(N) == "tc")

    def prepare_two_groups(self, kind, hyper_samples, comp, vals, res=None):
        """[prep of the first half, prep of the second half]: the factor chain (K build, Cholesky, inverse, operand pack:
        ~18 % of the headline step, latency-bound, a handful of SMs busy) of the SECOND half is queued on a side stream, so
        that it runs underneath the cross-covariance generator and predict GEMM of the FIRST half (ei_groups).  The chain is
        low-power work, so unlike overlapping the generator with the GEMM (both at the power cap: slower, DESIGN.md section
        5) this does not cost the GEMM its clock.  On 8 GPUs (5 samples per rank) it hides most of the latency floor that
        round 1's scaling run ran into."""
        S = len(hyper_samples)
        h = (S + 1) // 2
        main = torch.cuda.current_stream(self.device)
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.device)
        side = self._side
        if res is not None:                       # inputs already resident: group views of the caller's tensors
            hb = res.get("hb")
            r0 = dict(res, hb=hb.slice(0, h) if hb is not None else None)
            r1 = dict(res, hb=hb.slice(h, S) if hb is not None else None)
        else:                                     # upload once, share between the groups
            shared = dict(X=self.to_dev(comp), y=self.to_dev(vals), best=float(np.min(vals)))
            r0, r1 = dict(shared, hb=None), dict(shared, hb=None)
        prep0 = self.prepare(kind, hyper_samples[:h], comp, None, vals, None, None, None, resident=r0)
        side.wait_stream(main)                    # inputs uploaded; everything of the previous call is behind us
        with torch.cuda.stream(side):
            prep1 = self.prepare(kind, hyper_samples[h:], comp, None, vals, None, None, None, resident=r1)
            prep1.ready = side.record_event()
        prep0.ready = None
        return [prep0, prep1]

    def ei_groups(self, preps, Cd, want_matrix, ei_sum, cand_host=None):
        """EI of every candidate for the samples of all groups, in order; waits for a group's factor chain only when its turn
        comes.  Returns (ei [S][ldm] | None, ei_sum)."""
        main = torch.cuda.current_stream(self.device)
        parts = []
        for p in preps:
            if getattr(p, "ready", None) is not None:
                main.wait_event(p.ready)
            ei, ei_sum = self.ei_prepared(p, Cd, want_matrix, ei_sum, cand_host=cand_host)
            parts.append(ei)
        return (torch.cat(parts, dim=0) if want_matrix else None), ei_sum

    def _two_group_pass(self, kind, hyper_samples, comp, cand, vals, res, Cd, want_matrix, ei_sum, ei_all):
        preps = self.prepare_two_groups(kind, hyper_samples, comp, vals, res)
        ei, _ = self.ei_groups(preps, Cd, want_matrix, ei_sum, cand_host=cand)
        for p in preps:
            p.fac.check_pd()                      # host syncs after everything is queued
        if want_matrix:
            ei_all[:] = ei

    def ei_over_hypers(self, kind, hyper_samples, comp, pend, cand, vals, normals=None,
                       time_hyper_samples=None, durs_log=None):
        """Host-facing: numpy in, (M,S) float64 numpy out -- the reference's ei_over_hypers contract (OPT:331-341)."""
        ei, ei_sum, M = self.ei_over_hypers_device(kind, hyper_samples, comp, pend, cand, vals, normals,
                                                   time_hyper_samples, durs_log, want_matrix=True)
        self.tail_fix(kind, hyper_samples, len(hyper_samples), comp, pend, cand, vals, normals, time_hyper_samples,
                      durs_log, ei, ei_sum, M)
        return ei[:, :M].t().contiguous().double().cpu().numpy()

    # ------------------------------------------------------------------ deep-tail regime: exact ranking of the short-list
    TAIL_MEAN_EI = 1e-6      # below this max mean-EI the float32 moments no longer rank candidates like the reference
    TAIL_SHORTLIST = 256

    def tail_fix(self, kind, hs_local, S_total, comp, pend, cand, vals, normals, ths_local, durs_log, ei, ei_sum, M,
                 reduce_fn=None, rescore=None):
        """Late in a run max EI is 1e-8 ... 1e-60: EI = s (u Phi(u) + phi(u)) depends exponentially on u = (best - mu) / s,
        and float32 predictive moments then carry tens of percent of relative error -- enough to reorder the top of the
        ranking, while the reference (float64) proposes its exact argmax (OPT:294).  When the largest mean EI of a pass is
        below TAIL_MEAN_EI, the TAIL_SHORTLIST best candidates of the float32 ranking are re-evaluated with the float64
        build of the same kernels and their EI (per sample and summed) replaces the float32 values, so the argmax / top-k
        are decided in float64 exactly like the reference's.  ``ei_sum`` must already be the global (all-reduced) sum;
        ``reduce_fn`` all-reduces the short-list sums in place when hyper-samples are sharded over ranks.
        ``rescore(h64, cand_sub)`` -> (ei, ei_sum) replaces the plain EI pass of the short-list (constrained EI)."""
        if self.dtype != torch.float32:
            return False
        top = float(ei_sum[:M].max())                       # one scalar read; the caller synchronises right after anyway
        if not (top < self.TAIL_MEAN_EI * S_total):
            return False
        k = min(self.TAIL_SHORTLIST, M)
        idx, _ = self.topk(ei_sum, M, k)
        idx_h = idx.cpu().numpy().astype(np.int64)
        sub = torch.zeros((k,), dtype=torch.float64, device=self.device)
        if hs_local:
            h64 = self.helper64()
            sub_cand = np.ascontiguousarray(cand[idx_h])
            if rescore is not None:
                e64, s64 = rescore(h64, sub_cand)
            else:
                e64, s64, _ = h64.ei_over_hypers_device(kind, hs_local, comp, pend, sub_cand, vals, normals, ths_local,
                                                        durs_log, want_matrix=True)
            sub += s64[:k]
            if ei is not None:
                ei[:, idx.long()] = e64[:, :k]
        if reduce_fn is not None:
            reduce_fn(sub)
        ei_sum[idx.long()] = sub
        return True

    # ------------------------------------------------------------------ constrained EI (CONS = GPConstrainedEIChooser.py)
    def constraint_prob_device(self, kind, chyper_samples, ff, comp, labels, Cd, noise=CONSTRAINT_NOISE, want_mean=False):
        """P(feasible) = Phi(gain_s m_c(x)) at the candidates Cd, double [S][ldm] (CONS:816-842); with ``want_mean`` also
        m_c (double [S][ldm], None in the vanilla case).

        ``chyper_samples``: the reference's (constraint_mean, gain, amp2, ls) tuples; ``ff``: the one latent vector over
        every complete input ``comp`` (violations included) that the reference uses for every sample (CONS:293, 819-839).
        Without both feasible and violating points the reference skips the classification GP and weights every candidate
        by Phi(gain_s * 1) (CONS:816-817, 842); ``labels=None`` always evaluates the classification GP
        (pred_constraint_voilation, CONS:425-447, has no such branch).  Otherwise t_alpha = K_c^-1 ff comes from a FLOAT64
        factor of amp2 (k + 1e-6 I) + noise I: with noise 1e-3 its entries are large and of both signs, so float32 would lose
        m_c.  That solve keeps its right-hand side in shared memory (Factor.solve), which limits N to about 14 000
        complete observations; larger N raises SmkError."""
        S, M = len(chyper_samples), Cd.shape[0]
        ldm = _ceil(M, 128)
        gain = np.array([float(c[1]) for c in chyper_samples])
        if labels is not None and (np.all(np.asarray(labels) > 0) or np.all(np.asarray(labels) <= 0)):
            p = torch.as_tensor(sps.norm.cdf(gain), dtype=torch.float64, device=self.device)
            return p.view(S, 1).expand(S, ldm).contiguous(), None
        N, D = comp.shape
        h64 = self.helper64()
        X64, ff64 = h64.to_dev(comp), h64.to_dev(np.ravel(ff))
        X = X64 if h64 is self else self.to_dev(comp)
        gain_d = torch.as_tensor(gain, dtype=torch.float64, device=self.device)
        p = torch.empty((S, ldm), dtype=torch.float64, device=self.device)
        m = torch.empty((S, ldm), dtype=torch.float64, device=self.device) if want_mean else None
        hs = [(0.0, noise, float(c[2]), np.atleast_1d(np.asarray(c[3], dtype=float))) for c in chyper_samples]
        chunk = h64.max_samples_per_chunk(_ceil(N, 128), ldm)
        for s0 in range(0, S, chunk):
            t = self._t0()
            hb64 = h64.hypers(hs[s0:s0 + chunk], kind)
            fac = h64.factor(kind, X64, hb64, factor_impl="simt")
            t_alpha, _, _ = fac.solve(ff64, F=1, subtract_mean=False)           # CONS:834, one ff for every sample
            self._t1("constraint_factor", t)
            fac.check_pd()                                                      # LinAlgError like CONS:830
            hb = hb64 if h64 is self else self.hypers(hs[s0:s0 + chunk], kind)
            t = self._t0()
            check(fn("smk_constraint_prob", self.dtype)(KINDS[kind], N, fac.Npad, M, D, hb.S, ptr(X), ptr(Cd),
                                                        ptr(hb.inv_ls), ptr(hb.amp2), ptr(t_alpha), ptr(gain_d[s0:]),
                                                        ptr(p[s0:]), ptr(m[s0:]) if want_mean else None, ldm,
                                                        self.stream()), "constraint_prob")
            self._t1("constraint_prob", t)
            del fac
        return p, m

    def constrained_ei_over_hypers_device(self, kind, hyper_samples, chyper_samples, ff, comp, labels, pend, cand, vals,
                                          normals=None, noise=CONSTRAINT_NOISE):
        """The constrained grid pass (CONS:450-468, 806-940) as device tensors: (ei [S][ldm], ei_sum [ldm], M).

        The objective EI is the plain pass on the feasible points only (``labels > 0``), each sample's EI -- mean over the
        fantasies first -- multiplied by P(feasible) of the paired constraint sample in the same sweep.  ``normals``
        (S,P,F): the reference draws a fresh fantasy block per sample (CONS:910)."""
        if self.guard_threshold > 0:
            raise _lib.SmkError("the constrained pass does not run the tensor-core accuracy guard (SMK_TC_GUARD)")
        labels = np.asarray(labels)
        good = labels > 0
        if not np.any(good):
            raise ValueError("constrained EI needs at least one feasible observation")
        comp_g, vals_g = np.ascontiguousarray(comp[good]), np.asarray(vals, dtype=float)[good]
        S = len(hyper_samples)
        P = 0 if pend is None else int(pend.shape[0])
        if len(chyper_samples) != S:
            raise ValueError("%d objective but %d constraint hyper-samples" % (S, len(chyper_samples)))
        if np.size(ff) != comp.shape[0]:
            raise ValueError("ff has %d entries for %d complete observations" % (np.size(ff), comp.shape[0]))
        if P and (normals is None or np.ndim(normals) != 3 or np.shape(normals)[:2] != (S, P)):
            raise ValueError("pending points need fantasy normals of shape (S, P, F) = (%d, %d, F), got %s"
                             % (S, P, None if normals is None else np.shape(normals)))
        Cd = self.to_dev(cand)
        M = Cd.shape[0]
        ldm = _ceil(M, 128)
        w, _ = self.constraint_prob_device(kind, chyper_samples, ff, comp, labels, Cd, noise)
        chunk = self.max_samples_per_chunk(_ceil(comp_g.shape[0] + P, 128), ldm, 1 if P == 0 else int(normals.shape[-1]))
        ei_sum = torch.zeros((ldm,), dtype=torch.float64, device=self.device)
        ei_all = torch.empty((S, ldm), dtype=torch.float64, device=self.device)
        for s0 in range(0, S, chunk):
            nrm = None if normals is None else normals[s0:s0 + chunk]
            prep = self.prepare(kind, hyper_samples[s0:s0 + chunk], comp_g, pend, vals_g, nrm, cand_dev=Cd)
            ei, _ = self.ei_prepared(prep, Cd, True, ei_sum, weight=w[s0:s0 + prep.S])
            prep.fac.check_pd()
            ei_all[s0:s0 + prep.S] = ei
            del prep
        self.last = dict(N=comp.shape[0], N_good=comp_g.shape[0], M=M, S=S, P=P, chunk=chunk)
        return ei_all, ei_sum, M

    def constrained_ei_over_hypers(self, kind, hyper_samples, chyper_samples, ff, comp, labels, pend, cand, vals,
                                   normals=None, noise=CONSTRAINT_NOISE):
        """Host-facing: numpy in, (M,S) float64 numpy out -- GPConstrainedEIChooser.ei_over_hypers (CONS:450-468).
        In the deep-tail regime the short-list is re-scored by the float64 build (tail_fix)."""
        ei, ei_sum, M = self.constrained_ei_over_hypers_device(kind, hyper_samples, chyper_samples, ff, comp, labels,
                                                               pend, cand, vals, normals, noise)

        def rescore(h64, sub):
            e, s, _ = h64.constrained_ei_over_hypers_device(kind, hyper_samples, chyper_samples, ff, comp, labels, pend,
                                                            sub, vals, normals, noise)
            return e, s
        self.tail_fix(kind, hyper_samples, len(hyper_samples), comp, pend, cand, vals, normals, None, None, ei, ei_sum, M,
                      rescore=rescore)
        return ei[:, :M].t().contiguous().cpu().numpy()

    # ------------------------------------------------------------------ f2: GP log marginal likelihood
    def loglik(self, kind, comp, vals):
        return LogLik(self, kind, comp, vals)

    # ------------------------------------------------------------------ classification GP of the constrained chooser
    def latent_loglik(self, kind, comp, ls, noise=CONSTRAINT_NOISE):
        return LatentLogLik(self, kind, comp, ls, noise)

    def latent_factor(self, kind, comp, amp2, ls, noise):
        return LatentFactor(self, kind, comp, amp2, ls, noise)

    def constrained_refine_context(self, kind, hyper_samples, chyper_samples, ff, comp, labels, pend, vals, normals=None,
                                   noise=CONSTRAINT_NOISE):
        return ConstrainedRefineContext(self, kind, hyper_samples, chyper_samples, ff, comp, labels, pend, vals, normals,
                                        noise)

    # ------------------------------------------------------------------ f1: cached-factor EI value + gradient
    def refine_context(self, kind, hyper_samples, comp, pend, vals, normals=None, time_hyper_samples=None,
                       durs_log=None):
        return RefineContext(self, kind, hyper_samples, comp, pend, vals, normals, time_hyper_samples, durs_log)


class LogLik(object):
    """-sum(log diag chol K) - 0.5 (y-mu)' K^-1 (y-mu): the data term of every slice-sampler log-probability
    (OPT:635-640, 658-661, 689-692).  ``batch`` evaluates several hyper-parameter settings in ONE batched
    cov_build + potrf (same latency as one) and one small device->host read.  The residual rides along as an extra
    row of the covariance (csrc/solve.cu: augmentation), so the factorisation itself performs the forward
    substitution -- no serial triangular solve.  Buffers for ``max_batch`` matrices are allocated once."""

    def __init__(self, eng, kind, comp, vals, max_batch=None):
        self.eng, self.kind = eng, kind
        self.X = eng.to_dev(comp)
        self.y = eng.to_dev(vals)
        self.N, self.D = self.X.shape
        self.Npad = _ceil(self.N + 1, 128)          # room for the augmented row
        if max_batch is None:      # one slice move = 3 + SPECULATE points (util.py); small N is pure launch latency
            max_batch = 8 if self.N <= 1024 else 6
        self.max_batch = max_batch
        # slice-sampler speculation (util._slice_along): small matrices are pure launch latency -- evaluate everything a move
        # may need at once; from N ~ 1500 on a batch costs what its flops cost, so only the always-needed points go first
        # and shrink proposals follow in pairs once the interval is final
        self.speculate = (3, 0) if self.N <= 1536 else (0, 2)
        dt, dev = eng.dtype, eng.device
        # zeros once: the covariance is rebuilt in the lower triangle only (smk_cov_build_lower), the rest is never read
        self.L = torch.zeros((max_batch, self.Npad, self.Npad), dtype=dt, device=dev)
        # float64: dedicated look-ahead / DMMA factorisation (csrc/potrf_ll.cu); its workspace holds the inverse diagonal
        # blocks.  float32 (tests only): the generic blocked factorisation.
        self.fast = (dt == torch.float64) and os.environ.get("SMK_LOGLIK_IMPL", "ll") == "ll"
        self.use_graph = 1 if os.environ.get("SMK_LOGLIK_GRAPH", "1") == "1" else 0
        if self.fast:
            self.ws_bytes = _lib.lib().smk_potrf_loglik_workspace_bytes(self.Npad, max_batch)
            self.winv = torch.empty((self.ws_bytes,), dtype=torch.uint8, device=dev)
        else:
            self.winv = torch.empty((max_batch, self.Npad // eng.NB, eng.NB, eng.NB), dtype=dt, device=dev)
        self.info = torch.zeros((max_batch,), dtype=torch.int32, device=dev)
        self.out = torch.empty((2, max_batch), dtype=dt, device=dev)
        self.calls = 0
        self.launch_batches = 0

    def batch(self, hypers):
        """hypers: list of (mean, noise, amp2, ls).  Returns a float64 array; NaN marks a non-PD matrix."""
        out = np.empty(len(hypers))
        eng, dt, N, Npad = self.eng, self.eng.dtype, self.N, self.Npad
        for b0 in range(0, len(hypers), self.max_batch):
            hs = hypers[b0:b0 + self.max_batch]
            B = len(hs)
            hb = eng.hypers([(h[0], h[1], h[2], np.asarray(h[3], dtype=float)) for h in hs], self.kind)
            st = eng.stream()
            check(fn("smk_cov_build_lower", dt)(KINDS[self.kind], N, self.D, B, ptr(self.X), ptr(hb.inv_ls),
                                                ptr(hb.amp2), ptr(hb.noise), ptr(self.L), Npad, st), "cov_build")
            check(fn("smk_loglik_set_rhs", dt)(N, Npad, B, ptr(self.y), ptr(hb.mean), ptr(self.L), st), "loglik_set_rhs")
            if self.fast:
                check(_lib.lib().smk_potrf_loglik_f64(Npad, B, ptr(self.L), ptr(self.winv), self.ws_bytes, ptr(self.info),
                                                      self.use_graph, st), "potrf_loglik")
            else:
                check(fn("smk_potrf_lower_batched", dt)(Npad, B, ptr(self.L), ptr(self.winv), ptr(self.info), st), "potrf")
            check(fn("smk_loglik_finish", dt)(N, Npad, B, ptr(self.L), ptr(self.out[0]), ptr(self.out[1]), st),
                  "loglik_finish")
            r = torch.cat([self.out[0, :B].double(), self.out[1, :B].double(), self.info[:B].double()]).cpu().numpy()
            lp = -r[:B] - 0.5 * r[B:2 * B]
            lp[r[2 * B:] != 0] = np.nan
            out[b0:b0 + B] = lp
            self.calls += B
            self.launch_batches += 1
        return out

    def __call__(self, mean, noise, amp2, ls):
        v = self.batch([(mean, noise, amp2, ls)])[0]
        if np.isnan(v):
            raise np.linalg.LinAlgError("leading minor of the array is not positive definite")
        return v


class RefineContext(object):
    """(f, g) of GPEIOptChooser.grad_optimize_ei_over_hypers (OPT:360-525) / GPEIperSecChooser's (PSEC:321-435) at
    one point, with the S factors cached (the reference re-factors K for every sample on every evaluation)."""

    def __init__(self, eng, kind, hyper_samples, comp, pend, vals, normals=None, time_hyper_samples=None,
                 durs_log=None):
        if kind == "SE":
            raise AttributeError("module 'spearmint.gp' has no attribute 'grad_SE'")   # what the reference does, OPT:404
        self.eng, self.kind = eng, kind
        self.prep = eng.prepare(kind, hyper_samples, comp, pend, vals, normals, time_hyper_samples, durs_log)
        self.prep.fac.check_pd()
        self.pending = self.prep.P > 0
        self.hb = self.prep.hb
        self.evals = 0

    def _terms(self, fac, alpha, F, x):
        """out[S][F+1][D+1] of smk_ei_grad_terms for a single query point."""
        eng, dt = self.eng, self.eng.dtype
        hb = fac.hb
        S, N, D = hb.S, fac.N, fac.D
        xq = eng.to_dev(np.reshape(x, (1, D)))
        # kx as right-hand sides: cov(xq, X) -> [S][1][N]
        kx = torch.empty((S, 1, N), dtype=dt, device=eng.device)
        check(fn("smk_cov_build", dt)(KINDS[self.kind], 1, N, D, S, ptr(xq), ptr(fac.X), ptr(hb.inv_ls),
                                      ptr(hb.amp2), None, ptr(kx), N, eng.stream()), "cov_build")
        gamma, _, _ = fac.solve(kx, F=1, y_stride=N, ldy=N, subtract_mean=False)
        out = torch.empty((S, 1, F + 1, D + 1), dtype=dt, device=eng.device)
        check(fn("smk_ei_grad_terms", dt)(KINDS[self.kind], N, fac.Npad, D, S, 1, F, ptr(fac.X), ptr(xq),
                                          ptr(hb.inv_ls), ptr(hb.amp2), ptr(alpha), ptr(gamma), ptr(out),
                                          eng.stream()), "ei_grad_terms")
        return out.double().cpu().numpy()[:, 0]

    def per_sample(self, x):
        """Per hyper-sample (f_s, g_s) exactly as grad_optimize_ei returns them (OPT:391-525), incl. the 0.5*amp2."""
        p, hb = self.prep, self.hb
        F, D = p.F, p.fac.D
        out = self._terms(p.fac, p.alpha, F, x)                        # (S, F+1, D+1)
        amp2, mean = hb.host_amp2, hb.host_mean
        m = out[:, :F, D] + mean[:, None]                              # func_m (S,F)         OPT:417 / 508
        v = amp2 * (1 + JITTER) - out[:, F, D]                         # func_v (S,)          OPT:418 / 509
        s = np.sqrt(v)[:, None]
        u = (p.bests_host - m) / s
        cdf, pdf = sps.norm.cdf(u), sps.norm.pdf(u)
        ei = s * (u * cdf + pdf)                                       # (S,F)
        g_m, g_s2 = -cdf, 0.5 * pdf / s
        gx_m = out[:, :F, :D]                                          # (S,F,D)
        gx_v = -2.0 * out[:, F, :D]                                    # (S,D)
        g = 0.5 * amp2[:, None, None] * (gx_m * g_m[:, :, None] + gx_v[:, None, :] * g_s2[:, :, None])
        self.evals += 1
        if not self.pending:
            f_s, g_s, ei_s = -ei.sum(axis=1), g[:, 0, :], ei[:, 0]
        else:
            f_s, g_s, ei_s = -ei.mean(axis=1), g.mean(axis=1), ei.mean(axis=1)
        if p.time is not None:                                         # PSEC:351-435
            tfac, ta = p.time
            tout = self._terms(tfac, ta, 1, x)                         # (S, 2, D+1)
            thb = tfac.hb
            ftm = np.exp(tout[:, 0, D] + thb.host_mean)                # func_time_m
            gt = 0.5 * thb.host_amp2[:, None] * tout[:, 0, :D] * ftm[:, None]
            g_s = (ftm[:, None] * g_s - ei_s[:, None] * gt) / (ftm[:, None] ** 2)
            f_s = -(ei_s / ftm)
        return f_s, g_s

    def value_grad(self, x):
        """Sum over hyper-samples (OPT:360-388)."""
        f_s, g_s = self.per_sample(np.asarray(x, dtype=float))
        return float(f_s.sum()), g_s.sum(axis=0).flatten()


# ---------------------------------------------------------------------------------------------- classification GP
class LatentLogLik(LogLik):
    """-sum(log diag chol K_c) - 0.5 ff' K_c^-1 ff with K_c = amp2 (k(ls) + 1e-6 I) + noise I: the data term of the joint
    [amp2, ff] slice move of the constrained chooser (CONS:1169-1180).  ``batch([(amp2, ff), ...])`` evaluates every item
    with its OWN ff in one batched build + factorisation (smk_loglik_set_rhs_batched puts each ff in its augmented row)."""

    def __init__(self, eng, kind, comp, ls, noise=CONSTRAINT_NOISE, max_batch=None):
        LogLik.__init__(self, eng, kind, comp, np.zeros(comp.shape[0]), max_batch)
        self.ls, self.noise = np.atleast_1d(np.asarray(ls, dtype=float)), float(noise)

    def batch(self, items):
        """items: list of (amp2, ff).  Returns a float64 array; NaN marks a non-PD matrix."""
        out = np.empty(len(items))
        eng, dt, N, Npad = self.eng, self.eng.dtype, self.N, self.Npad
        for b0 in range(0, len(items), self.max_batch):
            its = items[b0:b0 + self.max_batch]
            B = len(its)
            hb = eng.hypers([(0.0, self.noise, float(a), self.ls) for a, _ in its], self.kind)
            y = eng.to_dev(np.vstack([np.ravel(f) for _, f in its]))
            st = eng.stream()
            check(fn("smk_cov_build_lower", dt)(KINDS[self.kind], N, self.D, B, ptr(self.X), ptr(hb.inv_ls),
                                                ptr(hb.amp2), ptr(hb.noise), ptr(self.L), Npad, st), "cov_build")
            check(fn("smk_loglik_set_rhs_batched", dt)(N, Npad, B, ptr(y), N, ptr(self.L), st), "loglik_set_rhs_batched")
            if self.fast:
                check(_lib.lib().smk_potrf_loglik_f64(Npad, B, ptr(self.L), ptr(self.winv), self.ws_bytes, ptr(self.info),
                                                      self.use_graph, st), "potrf_loglik")
            else:
                check(fn("smk_potrf_lower_batched", dt)(Npad, B, ptr(self.L), ptr(self.winv), ptr(self.info), st), "potrf")
            check(fn("smk_loglik_finish", dt)(N, Npad, B, ptr(self.L), ptr(self.out[0]), ptr(self.out[1]), st),
                  "loglik_finish")
            r = torch.cat([self.out[0, :B].double(), self.out[1, :B].double(), self.info[:B].double()]).cpu().numpy()
            lp = -r[:B] - 0.5 * r[B:2 * B]
            lp[r[2 * B:] != 0] = np.nan
            out[b0:b0 + B] = lp
            self.calls += B
            self.launch_batches += 1
        return out

    def __call__(self, amp2, ff):
        v = self.batch([(amp2, ff)])[0]
        if np.isnan(v):
            raise np.linalg.LinAlgError("leading minor of the array is not positive definite")
        return v


class LatentFactor(object):
    """The float64 lower Cholesky factor L of amp2 (k(ls) + 1e-6 I) + noise I over the complete inputs; ``draw(z)`` = L z
    on the device (smk_lower_matvec_f64).  The elliptical-slice direction nu = chol' randn (CONS:1241, chol the upper
    factor) and the prior draw of a fresh latent (CONS:1019-1022, noise 1e-6) are such products."""

    def __init__(self, eng, kind, comp, amp2, ls, noise):
        if eng.dtype != torch.float64:
            raise _lib.SmkError("LatentFactor needs the float64 engine")
        self.eng = eng
        hb = eng.hypers([(0.0, float(noise), float(amp2), np.atleast_1d(np.asarray(ls, dtype=float)))], kind)
        self.fac = eng.factor(kind, eng.to_dev(comp), hb, factor_impl="simt")
        self.fac.check_pd()                                  # LinAlgError like spla.cholesky (CONS:1021, 1197)
        self.N = comp.shape[0]
        self.out = torch.empty((self.N,), dtype=torch.float64, device=eng.device)

    def draw(self, z):
        zd = self.eng.to_dev(np.ravel(z))
        check(_lib.lib().smk_lower_matvec_f64(self.N, self.fac.Npad, ptr(self.fac.L), ptr(zd), ptr(self.out),
                                              self.eng.stream()), "lower_matvec")
        return self.out.cpu().numpy()


class ConstrainedRefineContext(RefineContext):
    """(f, g) of GPConstrainedEIChooser.grad_optimize_ei_over_hypers (CONS:471-501, 521-803) at one point, summed over the
    (objective, constraint) sample pairs, with every factor cached:
      * objective mean from the feasible points (CONS:750 / 607-641); variance from ALL complete points without pending
        points (CONS:751, 782-784) or from feasible + pending with them (CONS:637, 672);
      * with pending points EI and gradient are SUMMED over the fantasies and u uses best = min(feasible values), not the
        fantasy bests (CONS:655, 660, 677); the fantasies come from the normals the caller drew after
        npr.set_state(randomstate) (CONS:618);
      * P(feasible) = Phi(gain m_c) from the one latent ``ff``; both gradients carry the reference's 1/2 factor
        (CONS:675, 786, 683, 796); without a mix of labels the objective EI alone (CONS:679-680, 788-789)."""

    def __init__(self, eng, kind, hyper_samples, chyper_samples, ff, comp, labels, pend, vals, normals=None,
                 noise=CONSTRAINT_NOISE):
        if kind == "SE":
            raise AttributeError("module 'spearmint.gp' has no attribute 'grad_SE'")   # getattr(gp, 'grad_SE')
        self.eng, self.kind, self.evals = eng, kind, 0
        labels = np.asarray(labels)
        good = labels > 0
        comp_g, vals_g = np.ascontiguousarray(comp[good]), np.asarray(vals, dtype=float)[good]
        self.best = float(np.min(vals_g))
        self.pending = pend is not None and pend.shape[0] > 0
        self.vanilla = bool(np.all(labels > 0) or np.all(labels <= 0))
        self.prep = eng.prepare(kind, hyper_samples, comp_g, pend if self.pending else None, vals_g,
                                normals if self.pending else None)
        self.prep.fac.check_pd()
        self.hb = self.prep.hb
        if not self.pending:                 # variance from the factor of ALL complete points (CONS:745-746, 782-784)
            Xf = eng.to_dev(comp)
            self.fac_full = eng.factor(kind, Xf, self.hb)
            self.fac_full.check_pd()
            self.zero_alpha = torch.zeros((self.hb.S, 1, self.fac_full.Npad), dtype=eng.dtype, device=eng.device)
        if not self.vanilla:
            hs = [(0.0, noise, float(c[2]), np.atleast_1d(np.asarray(c[3], dtype=float))) for c in chyper_samples]
            self.gain = np.array([float(c[1]) for c in chyper_samples])
            self.camp2 = np.array([float(c[2]) for c in chyper_samples])
            self.fac_c = eng.factor(kind, eng.to_dev(comp), eng.hypers(hs, kind))
            self.fac_c.check_pd()                                                # CONS:561, 724
            self.t_alpha, _, _ = self.fac_c.solve(eng.to_dev(np.ravel(ff)), F=1, subtract_mean=False)

    def per_sample(self, x):
        p, hb = self.prep, self.hb
        F, D = p.F, p.fac.D
        amp2, mean = hb.host_amp2, hb.host_mean
        out = self._terms(p.fac, p.alpha, F, x)                        # (S, F+1, D+1)
        m = out[:, :F, D] + mean[:, None]                              # func_m (S,F)
        gx_m = out[:, :F, :D]
        if self.pending:
            v, gx_v = amp2 * (1 + JITTER) - out[:, F, D], -2.0 * out[:, F, :D]
        else:
            full = self._terms(self.fac_full, self.zero_alpha, 1, x)
            v, gx_v = amp2 * (1 + JITTER) - full[:, 1, D], -2.0 * full[:, 1, :D]
        s = np.sqrt(v)[:, None]
        u = (self.best - m) / s
        cdf, pdf = sps.norm.cdf(u), sps.norm.pdf(u)
        ei = s * (u * cdf + pdf)                                       # (S,F)
        g_m, g_s2 = -cdf, 0.5 * pdf / s
        g = 0.5 * amp2[:, None] * (gx_m * g_m[:, :, None] + gx_v[:, None, :] * g_s2[:, :, None]).sum(axis=1)   # (S,D)
        ei_tot = ei.sum(axis=1)
        self.evals += 1
        if self.vanilla:
            return -ei_tot, g
        c = self._terms(self.fac_c, self.t_alpha, 1, x)                # (S, 2, D+1)
        mc = c[:, 0, D]
        pc = sps.norm.cdf(self.gain * mc)
        gc = 0.5 * self.camp2[:, None] * self.gain[:, None] * c[:, 0, :D] * sps.norm.pdf(self.gain * mc)[:, None]
        return -ei_tot * pc, pc[:, None] * g + ei_tot[:, None] * gc
