"""Compute backend of the chooser plugins: everything numerical that ``next()`` needs, on the GPU.

    loglik(kind, comp, vals, chains=1)            -> callable(mean, noise, amp2, ls) -> float   (float64, f2)
                                                     with .batch(items); chains > 1: one round of lockstep chains
    optimize_hypers(kind, comp, vals)             -> (mean, noise, amp2, ls)  ML-II, GP.optimize_hypers   (f3)
    grid_state(kind, hyper_samples, comp, pend, vals, normals, time_hs, durs_log) -> state
    ei_matrix(state, cand)                        -> (M, S) float64 numpy                        (OPT:331-341)
    top_mean_ei(state, cand, k)                   -> indices of the k largest mean-EI candidates, ascending (OPT:270, 294)
    refine_context(...)                           -> object with value_grad(x)                   (f1, OPT:360-525)
    constrained_ei_matrix(kind, hs, constraint_hs, ff, comp, labels, pend, cand, vals, normals)
                                                  -> (M, S) float64 numpy, constrained EI        (CONS:450-468)
    forest_fit(X, y, weights, rand_r_states, max_features, max_depth, min_samples_split)
                                                  -> forest grown on the GPU                     (RF:64, 72)
    forest_predict(forest, X)                     -> (mean, var) float64 numpy                   (RF:16-26)
    forest_argmax_ei(forest, cand, best)          -> index of the largest RF EI                  (RF:75-87)

The chooser classes only talk to this interface, so the host logic (RNG order, state files, return protocol)
can be unit-tested on a CPU-only box with a stand-in backend supplied by the test; the product always constructs
``DeviceBackend`` and raises if CUDA / the shared library is missing.

Multi-GPU: when torch.distributed is initialised (one process per GPU, NCCL), the hyper-samples of the grid pass are
sharded round-robin over ranks and combined with ONE all-reduce of the per-candidate EI sum (parallel.py); the MCMC
chain and the L-BFGS refinement are replicated (same seeds -> identical on every rank).  With mcmc_chains=K > 1, chain c
runs on rank c mod W and the finished chains are exchanged in one all-gather (chains.py).
"""
import numpy as np
import torch

from . import parallel
from .engine import GPEIEngine, _ceil


class _GridState(object):
    pass


class DeviceBackend(object):
    name = "b200"

    def __init__(self, device=None, refine_dtype="float64", grid_dtype="float32"):
        """``grid_dtype``: precision of the grid pass (grid_state, ei_matrix, top_mean_ei, constrained_ei_matrix,
        constraint_predict).  "float32" is the production chain; "float64" runs it on the float64 engine (the reference's
        precision, with the prediction on the fp64 tensor cores from f64_mma_min_n on) and needs no deep-tail re-scoring."""
        if grid_dtype not in ("float32", "float64"):
            raise ValueError("grid_dtype must be float32 or float64, got %r" % (grid_dtype,))
        if device is None and torch.cuda.is_available():
            rank, world = parallel.world()
            device = "cuda:%d" % (torch.cuda.current_device() if world == 1 else rank % torch.cuda.device_count())
        self.eng32 = GPEIEngine(device=device, dtype=torch.float32)
        self.eng64 = GPEIEngine(device=device, dtype=torch.float64)
        self.refine_eng = self.eng64 if refine_dtype == "float64" else self.eng32
        self.grid_dtype = grid_dtype

    @property
    def grid_eng(self):
        """The engine of the grid pass: the float64 one with grid_dtype="float64", else the float32 one."""
        return self.eng64 if getattr(self, "grid_dtype", "float32") == "float64" else self.eng32

    # ---- f2
    def loglik(self, kind, comp, vals, chains=1):
        """chains > 1: the handle of that many lockstep chains (engine.ChainLogLik); 1: the single chain's."""
        return self.eng64.loglik(kind, comp, vals, chains)

    # ---- f3: ML-II hyper-parameters (gp.GP.optimize_hypers, GP:181-292)
    def optimize_hypers(self, kind, comp, vals):
        """-> (mean, noise, amp2, ls): L-BFGS-B on the host, likelihood value and gradient terms on the GPU in float64."""
        from .gp import GP
        g = GP(kind, engine=self.eng64)
        g.real_init(comp.shape[1], vals)
        g.optimize_hypers(comp, vals)
        return g.mean, g.noise, g.amp2, g.ls

    # ---- grid pass
    def grid_state(self, kind, hyper_samples, comp, pend, vals, normals=None, time_hyper_samples=None,
                   durs_log=None):
        """Factors all (local) hyper-samples once; reused by both grid passes of next() (OPT:269, OPT:293)."""
        eng = self.grid_eng
        rank, world = parallel.world()
        S = len(hyper_samples)
        mine = parallel.shard(S, rank, world)
        st = _GridState()
        st.kind, st.S, st.mine = kind, S, mine
        st.args = (comp, pend, vals, normals, durs_log)
        st.hs = [hyper_samples[s] for s in mine]
        st.ths = None if time_hyper_samples is None else [time_hyper_samples[s] for s in mine]
        P = 0 if pend is None else pend.shape[0]
        F = 1 if P == 0 else normals.shape[-1]
        if normals is not None and np.ndim(normals) == 3:      # per-sample normals follow their samples to the owning rank
            normals = normals[mine]
            st.args = (comp, pend, vals, normals, durs_log)
        chunk = eng.max_samples_per_chunk(_ceil(comp.shape[0] + P, 128), _ceil(200000, 128), F)
        st.preps, st.pd_checked = None, True
        err = None
        try:
            if st.hs and len(st.hs) <= chunk:        # everything resident: prepare once, sweep many
                if eng.can_overlap(comp.shape[0], len(st.hs), P, st.ths):
                    st.preps = eng.prepare_two_groups(kind, st.hs, comp, vals)   # 2nd half's factor chain on a side stream
                else:
                    st.preps = [eng.prepare(kind, st.hs, comp, pend, vals, normals, st.ths, durs_log)]
                    st.preps[0].fac.check_pd()
                st.pd_checked = len(st.preps) == 1
        except np.linalg.LinAlgError as e:           # the reference lets spla.cholesky raise (SURVEY 8b); so do we --
            err = e                                  # on every rank, or the others would hang in the all-reduce
        parallel.agree_on_error(err, eng.device)
        return st

    def _local(self, st, cand, want_matrix):
        """This rank's EI (matrix and sum over its hyper-samples).  Every rank ends with the same single
        agree_on_error() collective, whatever path it took (resident factors, chunked, empty shard)."""
        eng = self.grid_eng
        ldm = _ceil(cand.shape[0], 128)
        err, ei, ei_sum = None, None, None
        if not st.hs:
            ei_sum = torch.zeros((ldm,), dtype=torch.float64, device=eng.device)
        elif st.preps is not None:
            ei, ei_sum = eng.ei_groups(st.preps, eng.to_dev(cand), want_matrix, None, cand_host=cand)
            if not st.pd_checked:                    # deferred until the first sweep is queued: the check synchronises
                try:
                    for p in st.preps:
                        p.fac.check_pd()
                except np.linalg.LinAlgError as e:
                    err = e
                st.pd_checked = True
        else:
            comp, pend, vals, normals, durs_log = st.args
            try:                                     # chunked path: factors are (re)built per pass and may raise here
                ei, ei_sum, _ = eng.ei_over_hypers_device(st.kind, st.hs, comp, pend, cand, vals, normals, st.ths,
                                                          durs_log, want_matrix=want_matrix)
            except np.linalg.LinAlgError as e:
                err = e
        parallel.agree_on_error(err, eng.device)
        return ei, ei_sum

    def _tail_fix(self, st, cand, ei, ei_sum, M):
        """float64 re-evaluation of the short-list when the pass is in the deep-tail regime (engine.tail_fix); a float64
        pass has nothing to re-evaluate (the float64 engine's tail_fix returns at once)."""
        comp, pend, vals, normals, durs_log = st.args
        return self.grid_eng.tail_fix(st.kind, st.hs, st.S, comp, pend, cand, vals, normals, st.ths, durs_log, ei, ei_sum, M,
                                   reduce_fn=parallel.allreduce_sum_)

    def ei_matrix(self, st, cand):
        M = cand.shape[0]
        ei, ei_sum = self._local(st, cand, True)
        rank, world = parallel.world()
        if world == 1:
            self._tail_fix(st, cand, ei, ei_sum, M)
            return ei[:, :M].t().contiguous().double().cpu().numpy()
        parallel.allreduce_sum_(ei_sum)
        self._tail_fix(st, cand, ei, ei_sum, M)      # the same decision on every rank (global sum); local columns fixed
        full = torch.zeros((st.S, _ceil(M, 128)), dtype=torch.float64, device=self.grid_eng.device)
        if ei is not None:
            full[st.mine] = ei
        parallel.allreduce_sum_(full)                # columns are disjoint across ranks
        return full[:, :M].t().contiguous().double().cpu().numpy()

    def top_mean_ei(self, st, cand, k):
        M = cand.shape[0]
        _, ei_sum = self._local(st, cand, False)
        parallel.allreduce_sum_(ei_sum)              # the single exchange of the path (SURVEY 8e)
        self._tail_fix(st, cand, None, ei_sum, M)    # deep-tail passes: exact float64 ranking of the short-list
        idx, _ = self.grid_eng.topk(ei_sum, M, k)    # argsort / argmax of the mean == of the sum
        out = idx.cpu().numpy().astype(int)
        if np.any(out < 0):                          # fewer than k non-NaN scores (the reference would rank NaNs)
            raise FloatingPointError("EI is NaN for more than %d of %d candidates (non-finite hyper-parameters or "
                                     "inputs)" % (M - k, M))
        return out

    # ---- constrained EI (CONS = chooser/GPConstrainedEIChooser.py)
    def constrained_ei_matrix(self, kind, hyper_samples, chyper_samples, ff, comp, labels, pend, cand, vals,
                              normals=None):
        """(M, S) float64 numpy: GPConstrainedEIChooser.ei_over_hypers (CONS:450-468).  Sample PAIRS -- objective sample s
        with constraint sample s -- are sharded round-robin over ranks, per-sample fantasy normals (S,P,F) with them; the
        per-candidate sum is all-reduced once (it decides the deep-tail re-evaluation), the disjoint columns once."""
        eng = self.grid_eng
        rank, world = parallel.world()
        S, M = len(hyper_samples), cand.shape[0]
        ldm = _ceil(M, 128)
        mine = parallel.shard(S, rank, world)
        hs, chs = [hyper_samples[s] for s in mine], [chyper_samples[s] for s in mine]
        nrm = None if normals is None else np.asarray(normals)[mine]
        err, ei = None, None
        ei_sum = torch.zeros((ldm,), dtype=torch.float64, device=eng.device)
        if hs:
            try:
                ei, ei_sum, _ = eng.constrained_ei_over_hypers_device(kind, hs, chs, ff, comp, labels, pend, cand, vals,
                                                                      nrm)
            except np.linalg.LinAlgError as e:       # every rank raises, or the others would hang in the all-reduce
                err = e
        parallel.agree_on_error(err, eng.device)
        parallel.allreduce_sum_(ei_sum)

        def rescore(h64, sub):
            e, s, _ = h64.constrained_ei_over_hypers_device(kind, hs, chs, ff, comp, labels, pend, sub, vals, nrm)
            return e, s
        eng.tail_fix(kind, hs, S, comp, pend, cand, vals, nrm, None, None, ei, ei_sum, M,
                     reduce_fn=parallel.allreduce_sum_, rescore=rescore)
        if world == 1:
            return ei[:, :M].t().contiguous().cpu().numpy()
        full = torch.zeros((S, ldm), dtype=torch.float64, device=eng.device)
        if ei is not None:
            full[mine] = ei
        parallel.allreduce_sum_(full)                # columns are disjoint across ranks
        return full[:, :M].t().contiguous().cpu().numpy()

    def constraint_predict(self, kind, chyper, ff, comp, cand):
        """Phi(gain m_c) at ``cand`` for ONE constraint sample (pred_constraint_voilation, CONS:425-447), (M,) numpy."""
        eng = self.grid_eng
        p, _ = eng.constraint_prob_device(kind, [chyper], ff, comp, None, eng.to_dev(cand))
        return p[0, :cand.shape[0]].cpu().numpy()

    # ---- classification-GP sampler (float64)
    def latent_loglik(self, kind, comp, ls, noise):
        """callable(amp2, ff) and .batch([(amp2, ff), ...]): the data term of the joint [amp2, ff] move (CONS:1169-1180)."""
        return self.eng64.latent_loglik(kind, comp, ls, noise)

    def latent_factor(self, kind, comp, amp2, ls, noise):
        """.draw(z) = L z, L the lower Cholesky factor of amp2 (k + 1e-6 I) + noise I (CONS:1019-1022, 1193-1200)."""
        return self.eng64.latent_factor(kind, comp, amp2, ls, noise)

    def constrained_refine_context(self, kind, hyper_samples, chyper_samples, ff, comp, labels, pend, vals,
                                   normals=None, noise=1e-3):
        """object with value_grad(x): CONS:471-803 summed over the sample pairs, factors cached."""
        return self.refine_eng.constrained_refine_context(kind, hyper_samples, chyper_samples, ff, comp, labels, pend,
                                                          vals, normals, noise)

    # ---- random forest (RF = chooser/RandomForestEIChooser.py); every rank grows the same forest
    def forest_fit(self, X, y, weights, rand_r_states, max_features, max_depth=None, min_samples_split=2):
        """T regression trees grown on the GPU from the host draws of forest.draws (RF:64, 72)."""
        from .forest import DeviceForest
        eng = self.eng64
        return DeviceForest(eng.device, eng.stream(), X, y, weights, rand_r_states, max_features, max_depth,
                            min_samples_split)

    def forest_predict(self, forest, X):
        """(mean, var) float64 numpy at X (RF:16-26)."""
        out = forest.predict(X, want=("mean", "var"))
        return out["mean"].cpu().numpy(), out["var"].cpu().numpy()

    def forest_argmax_ei(self, forest, cand, best):
        """argmax of the RF EI (RF:80-87) over the candidates, numpy's first-max rule: the device top-k."""
        M = cand.shape[0]
        ei = forest.predict(cand, best, want=("ei",))["ei"]
        idx, _ = self.eng64.topk(ei, M, 1)
        i = int(idx[0].item())
        return 0 if i < 0 else i         # every EI NaN (a single tree: var is NaN): np.argmax returns 0

    # ---- f1
    def refine_context(self, kind, hyper_samples, comp, pend, vals, normals=None, time_hyper_samples=None,
                       durs_log=None):
        return self.refine_eng.refine_context(kind, hyper_samples, comp, pend, vals, normals, time_hyper_samples,
                                              durs_log)
