// forest.cu -- the random-forest regressor of RandomForestEIChooser (RF = chooser/RandomForestEIChooser.py), grown and
// evaluated on the GPU.
//
// Reference spans replaced:
//   self.rf.fit(comp, vals)            (RF:64, 72)   scikit-learn's RandomForestRegressor: T bootstrap-weighted trees,
//                                                    DepthFirstTreeBuilder + BestSplitter + MSE criterion
//   func_m, func_v = self.rf.predict() (RF:16-26)    per-tree predict, mean in tree order, np.var(ddof=1)
//   ei = func_s*(u*ncdf + npdf)        (RF:80-85)
//
// The trees are structurally those scikit-learn grows from the same bootstrap counts and splitter rand_r states (the
// host draws both from numpy's RNG, as sklearn does): every value that decides a split -- the sums of the MSE criterion,
// the proxy sl^2/wl + sr^2/wr, the children's impurities -- is formed by the same sequence of double operations, with
// explicit round-to-nearest intrinsics so that nvcc contracts nothing into an FMA.  Split candidates of one node often tie
// exactly (every split of a 2-sample node does, across all features), so the summation order is part of the result.
//
// fit: one CTA per tree walks its nodes in sklearn's order (depth-first, pop, push right then left).
//   * each feature keeps a list of the tree's in-bag samples sorted by (value, index); a node owns the segment
//     [start, end) of every list.  All lists are sorted once (a rank sort shared by the trees) and compacted per tree;
//     a split partitions every segment stably into its children.  So a node's sort is free and its constant test O(1).
//   * thread 0 runs the Fisher-Yates feature draw (it interleaves rand_r draws with the constant tests, so it is serial);
//     the drawn non-constant features are then scanned in parallel, one thread per feature, each forming its sum_left
//     sequentially as RegressionCriterion.update does; thread 0 picks the first strictly greater proxy in draw order.
//   * samples[start:end] is rewritten in the order of the last feature sorted and swap-partitioned by thread 0, as
//     BestSplitter leaves it: the children's sums run over that order.
// predict + EI: one thread per candidate walks all T trees twice (mean, then the two-pass variance).
#include <float.h>
#include <stdint.h>

#include "common.cuh"

namespace smk {

constexpr int kForestThreads = 256;
constexpr int kTreeLeaf = -1, kTreeUndefined = -2;
constexpr unsigned kRandRMax = 0x7FFFFFFFu;
constexpr float kFeatureThreshold = 1e-7f;

struct StackRec {
  int start, end, depth, parent, is_left, n_const;
  double impurity;
};

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// sklearn's our_rand_r / rand_int (xorshift on a uint32, modulo RAND_R_MAX + 1, then modulo the range)
__device__ __forceinline__ int rand_int(int low, int high, unsigned* st) {
  unsigned s = *st ? *st : 1u;
  s ^= s << 13;
  s ^= s >> 17;
  s ^= s << 5;
  *st = s;
  return low + (int)((s % (kRandRMax + 1u)) % (unsigned)(high - low));
}

// Xt[d][n] = float32 X[n][d]
__global__ void forest_transpose_kernel(int N, int D, const float* __restrict__ X, float* __restrict__ Xt) {
  const long e = (long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long)N * D) return;
  const int n = (int)(e / D), d = (int)(e % D);
  Xt[(long)d * N + n] = X[e];
}

// order[d][rank] = n, rank = #{j : (x_j, j) < (x_n, n)}: every feature sorted once by (value, index), for all trees
__global__ void __launch_bounds__(256) forest_rank_sort_kernel(int N, const float* __restrict__ Xt, int* __restrict__ order) {
  __shared__ float xs[256];
  const int d = blockIdx.y, n = blockIdx.x * 256 + threadIdx.x;
  const float* x = Xt + (long)d * N;
  const float xn = n < N ? x[n] : 0.0f;
  int rank = 0;
  for (int j0 = 0; j0 < N; j0 += 256) {
    __syncthreads();
    if (j0 + threadIdx.x < N) xs[threadIdx.x] = x[j0 + threadIdx.x];
    __syncthreads();
    const int jn = min(256, N - j0);
    for (int j = 0; j < jn; ++j) {
      const float xj = xs[j];
      rank += (xj < xn) || (xj == xn && j0 + j < n);
    }
  }
  if (n < N) order[(long)d * N + rank] = n;
}

struct FitArgs {
  int N, D, max_features, max_depth, min_samples_split, ldn;
  const float* Xt;           // [D][N]
  const double* y;           // [N]
  const double* w;           // [T][N]
  const unsigned* rand_r;    // [T]
  const int* order;          // [D][N]
  int* lists;                // [T][D][N]
  int* tmp;                  // [T][D][N]
  int* samples;              // [T][N]
  StackRec* stack;           // [T][N + 1]
  int *feature, *left, *right, *n_node_samples, *node_count;
  double *threshold, *value;
};

__global__ void __launch_bounds__(kForestThreads) forest_fit_kernel(FitArgs a) {
  extern __shared__ __align__(8) unsigned char smem[];
  const int N = a.N, D = a.D, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nwarps = kForestThreads / 32;
  double* ev_proxy = reinterpret_cast<double*>(smem);              // [D] best proxy of the e-th evaluated feature
  double* ev_thr = ev_proxy + D;                                   // [D] its threshold
  int* ev_pos = reinterpret_cast<int*>(ev_thr + D);                // [D] its position (-1: no valid position)
  int* features = ev_pos + D;                                      // [D] BestSplitter.features
  int* const_features = features + D;                              // [D] BestSplitter.constant_features
  int* ev_feat = const_features + D;                               // [D] evaluated features in draw order

  __shared__ StackRec rec;
  __shared__ int s_leaf, s_n_eval, s_last_sorted, s_best_feat, s_best_pos, s_node_id, s_sp, s_n_total, s_n_found;
  __shared__ int s_n_samples;
  __shared__ double s_best_thr, s_sum_total, s_wn, s_sq_total;

  const int t = blockIdx.x;
  const long tN = (long)t * N, tDN = (long)t * D * N;
  const double* w = a.w + tN;
  int* samples = a.samples + tN;
  int* lists = a.lists + tDN;
  int* tmp = a.tmp + tDN;
  StackRec* stack = a.stack + (long)t * (N + 1);
  const long ldn = a.ldn;
  int* feature = a.feature + t * ldn;
  int* left = a.left + t * ldn;
  int* right = a.right + t * ldn;
  int* nns = a.n_node_samples + t * ldn;
  double* threshold = a.threshold + t * ldn;
  double* value = a.value + t * ldn;

  // in-bag samples in index order (Splitter.init), weighted_n_samples over all samples
  __shared__ double s_wn_samples;
  __shared__ unsigned s_rng;
  if (tid == 0) {
    int j = 0;
    double wsum = 0.0;
    for (int i = 0; i < N; ++i) {
      if (w[i] != 0.0) samples[j++] = i;
      wsum = dadd(wsum, w[i]);
    }
    s_n_samples = j;
    s_wn_samples = wsum;
    s_rng = a.rand_r[t];
  }
  for (int d = tid; d < D; d += kForestThreads) features[d] = d;
  // per-feature sorted lists of the in-bag samples: stable compaction of the shared order, one warp per feature
  for (int d = warp; d < D; d += nwarps) {
    const int* od = a.order + (long)d * N;
    int* ld = lists + (long)d * N;
    int base = 0;
    for (int i0 = 0; i0 < N; i0 += 32) {
      const int i = i0 + lane;
      const int n = i < N ? od[i] : 0;
      const bool keep = i < N && w[n] != 0.0;
      const unsigned m = __ballot_sync(0xffffffffu, keep);
      if (keep) ld[base + __popc(m & ((1u << lane) - 1u))] = n;
      base += __popc(m);
    }
  }
  if (tid == 0) {
    StackRec r;
    r.start = 0; r.end = s_n_samples; r.depth = 0; r.parent = kTreeUndefined; r.is_left = 0; r.n_const = 0;
    r.impurity = INFINITY;
    stack[0] = r;
    s_sp = 1;
    s_node_id = 0;
  }
  bool first = true;
  __syncthreads();

  for (;;) {
    const int sp = s_sp;
    __syncthreads();                                   // everyone has read s_sp before thread 0 pops
    if (sp == 0) break;
    // ---- pop, node_reset, leaf test, feature draw (thread 0)
    if (tid == 0) {
      rec = stack[--s_sp];
      const int start = rec.start, end = rec.end, n_node = end - start;
      double st = 0.0, sq = 0.0, wn = 0.0;
      for (int p = start; p < end; ++p) {
        const int i = samples[p];
        const double wi = w[i], yi = a.y[i], wy = dmul(wi, yi);
        st = dadd(st, wy);
        sq = dadd(sq, dmul(wy, yi));
        wn = dadd(wn, wi);
      }
      s_sum_total = st; s_sq_total = sq; s_wn = wn;
      bool leaf = rec.depth >= a.max_depth || n_node < a.min_samples_split || n_node < 2;
      if (first) {
        const double mu = ddiv(st, wn);
        rec.impurity = dsub(ddiv(sq, wn), dmul(mu, mu));
      }
      leaf = leaf || rec.impurity <= DBL_EPSILON;
      s_leaf = leaf;
      s_n_eval = 0;
      s_last_sorted = -1;
      s_n_found = 0;
      s_n_total = rec.n_const;
      if (!leaf) {
        const int n_known = rec.n_const;
        int f_i = D, n_found = 0, n_drawn = 0, n_total = n_known, n_visited = 0, n_eval = 0;
        unsigned rng = s_rng;
        while (f_i > n_total && (n_visited < a.max_features || n_visited <= n_found + n_drawn)) {
          ++n_visited;
          int f_j = rand_int(n_drawn, f_i - n_found, &rng);
          if (f_j < n_known) {
            const int tq = features[n_drawn]; features[n_drawn] = features[f_j]; features[f_j] = tq;
            ++n_drawn;
            continue;
          }
          f_j += n_found;
          const int f = features[f_j];
          s_last_sorted = f;
          const int* lf = lists + (long)f * N;
          const float* xf = a.Xt + (long)f * N;
          if (xf[lf[end - 1]] <= xf[lf[start]] + kFeatureThreshold) {     // constant in this node (float32 sum)
            features[f_j] = features[n_total]; features[n_total] = f;
            ++n_found; ++n_total;
            continue;
          }
          --f_i;
          features[f_j] = features[f_i]; features[f_i] = f;
          ev_feat[n_eval++] = f;
        }
        s_rng = rng;
        s_n_eval = n_eval;
        s_n_found = n_found;
        s_n_total = n_total;
      }
    }
    __syncthreads();

    const int start = rec.start, end = rec.end;
    if (!s_leaf) {
      // ---- best split of each evaluated feature: one thread per feature, sums in sorted order
      const double sum_total = s_sum_total, wn = s_wn;
      for (int e = tid; e < s_n_eval; e += kForestThreads) {
        const int f = ev_feat[e];
        const int* lf = lists + (long)f * N;
        const float* xf = a.Xt + (long)f * N;
        double sl = 0.0, wl = 0.0, tsl = 0.0, twl = 0.0, best = -INFINITY, bthr = 0.0;
        int pos = start, bpos = -1;
        int i = lf[start];
        float xprev = xf[i];
        for (int q = start + 1; q < end; ++q) {
          const double wi = w[i];
          tsl = dadd(tsl, dmul(wi, a.y[i]));           // sample q-1 moves left if the update runs forwards
          twl = dadd(twl, wi);
          i = lf[q];
          const float xq = xf[i];
          if (xq <= xprev + kFeatureThreshold) { xprev = xq; continue; }
          if (q - pos <= end - q) {
            sl = tsl; wl = twl;
          } else {                                        // RegressionCriterion.update from the end
            sl = sum_total; wl = wn;
            for (int r = end - 1; r >= q; --r) {
              const int k = lf[r];
              sl = dsub(sl, dmul(w[k], a.y[k]));
              wl = dsub(wl, w[k]);
            }
            tsl = sl; twl = wl;
          }
          pos = q;
          const double sr = dsub(sum_total, sl), wr = dsub(wn, wl);
          const double proxy = dadd(ddiv(dmul(sl, sl), wl), ddiv(dmul(sr, sr), wr));
          if (proxy > best) {
            best = proxy;
            bpos = q;
            bthr = dadd((double)xprev / 2.0, (double)xq / 2.0);
          }
          xprev = xq;
        }
        ev_proxy[e] = best;
        ev_pos[e] = bpos;
        ev_thr[e] = bthr;
      }
      __syncthreads();
      if (tid == 0) {
        double best = -INFINITY;
        int bf = -1, bp = end;
        double bt = 0.0;
        for (int e = 0; e < s_n_eval; ++e)
          if (ev_pos[e] >= 0 && ev_proxy[e] > best) { best = ev_proxy[e]; bf = ev_feat[e]; bp = ev_pos[e]; bt = ev_thr[e]; }
        s_best_feat = bf; s_best_pos = bp; s_best_thr = bt;
      }
      // the splitter leaves samples[start:end] sorted by the last feature it sorted
      if (s_last_sorted >= 0) {
        const int* lf = lists + (long)s_last_sorted * N;
        for (int p = start + tid; p < end; p += kForestThreads) samples[p] = lf[p];
      }
      __syncthreads();
      const int bf = s_best_feat, pos = s_best_pos;
      const double thr = s_best_thr;
      if (pos < end) {
        const float* xb = a.Xt + (long)bf * N;
        if (tid == 0) {
          // partition_samples_final, then reset + update(pos) + children_impurity over the partitioned order
          int ps = start, pe = end;
          while (ps < pe) {
            const int i = samples[ps];
            if ((double)xb[i] <= thr) { ++ps; }
            else { --pe; samples[ps] = samples[pe]; samples[pe] = i; }
          }
          const double sum_total = s_sum_total, wn = s_wn;
          double sl = 0.0, wl = 0.0, sq_l = 0.0;
          if (pos - start <= end - pos) {
            for (int p = start; p < pos; ++p) {
              const int i = samples[p];
              sl = dadd(sl, dmul(w[i], a.y[i]));
              wl = dadd(wl, w[i]);
            }
          } else {
            sl = sum_total; wl = wn;
            for (int p = end - 1; p >= pos; --p) {
              const int i = samples[p];
              sl = dsub(sl, dmul(w[i], a.y[i]));
              wl = dsub(wl, w[i]);
            }
          }
          for (int p = start; p < pos; ++p) {
            const int i = samples[p];
            sq_l = dadd(sq_l, dmul(dmul(w[i], a.y[i]), a.y[i]));
          }
          const double sr = dsub(sum_total, sl), wr = dsub(wn, wl);
          const double ml = ddiv(sl, wl), mr = ddiv(sr, wr);
          const double imp_l = dsub(ddiv(sq_l, wl), dmul(ml, ml));
          const double imp_r = dsub(ddiv(dsub(s_sq_total, sq_l), wr), dmul(mr, mr));
          const double improvement =
              dmul(ddiv(wn, s_wn_samples),
                   dsub(dsub(rec.impurity, dmul(ddiv(wr, wn), imp_r)), dmul(ddiv(wl, wn), imp_l)));
          s_leaf = dadd(improvement, DBL_EPSILON) < 0.0;
          if (!s_leaf) {
            StackRec r;
            r.start = pos; r.end = end; r.depth = rec.depth + 1; r.parent = s_node_id; r.is_left = 0;
            r.n_const = s_n_total; r.impurity = imp_r;
            stack[s_sp++] = r;
            r.start = start; r.end = pos; r.is_left = 1; r.impurity = imp_l;
            stack[s_sp++] = r;
          }
        } else if (warp > 0) {
          // meanwhile warps 1.. partition every feature's segment stably into [start, pos) and [pos, end)
          for (int d = warp - 1; d < D; d += nwarps - 1) {
            int* ld = lists + (long)d * N;
            int* td = tmp + (long)d * N;
            int nl = 0, nr = 0;
            for (int p0 = start; p0 < end; p0 += 32) {
              const int p = p0 + lane;
              const bool in = p < end;
              const int i = in ? ld[p] : 0;
              const bool gl = in && (double)xb[i] <= thr;
              const unsigned ml = __ballot_sync(0xffffffffu, gl), mr = __ballot_sync(0xffffffffu, in && !gl);
              const unsigned below = (1u << lane) - 1u;
              if (gl) td[start + nl + __popc(ml & below)] = i;
              else if (in) td[pos + nr + __popc(mr & below)] = i;
              nl += __popc(ml);
              nr += __popc(mr);
            }
            __syncwarp();
            for (int p = start + lane; p < end; p += 32) ld[p] = td[p];
            __syncwarp();
          }
        }
      } else if (tid == 0) {
        s_leaf = 1;
      }
      // the constant-feature bookkeeping of node_split_best (runs whether or not a split was found)
      __syncthreads();
      if (tid == 0) {
        const int n_known = rec.n_const;
        for (int k = 0; k < n_known; ++k) features[k] = const_features[k];
        for (int k = 0; k < s_n_found; ++k) const_features[n_known + k] = features[n_known + k];
      }
    }
    // ---- the node itself (Tree._add_node) and the parent's child pointer
    if (tid == 0) {
      const int nid = s_node_id++;
      if (rec.parent != kTreeUndefined) {
        if (rec.is_left) left[rec.parent] = nid;
        else right[rec.parent] = nid;
      }
      const bool leaf = s_leaf;
      feature[nid] = leaf ? kTreeUndefined : s_best_feat;
      threshold[nid] = leaf ? (double)kTreeUndefined : s_best_thr;
      left[nid] = kTreeLeaf;
      right[nid] = kTreeLeaf;
      nns[nid] = end - start;
      value[nid] = ddiv(s_sum_total, s_wn);
      // children were pushed with the id this node has now
    }
    first = false;
    __syncthreads();
  }
  if (tid == 0) a.node_count[t] = s_node_id;
}

// mean / var / EI of every candidate over the T trees (RF:16-26, 80-85)
__global__ void forest_predict_ei_kernel(int M, int D, int T, int ldn, const float* __restrict__ C,
                                         const int* __restrict__ feature, const double* __restrict__ threshold,
                                         const int* __restrict__ left, const int* __restrict__ right,
                                         const double* __restrict__ value, double best, double* __restrict__ mean_out,
                                         double* __restrict__ var_out, double* __restrict__ ei_out) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float* c = C + (long)m * D;
  auto leaf_value = [&](int t) {
    const long o = (long)t * ldn;
    int node = 0;
    while (left[o + node] != kTreeLeaf) {
      const int f = feature[o + node];
      node = ((double)c[f] <= threshold[o + node]) ? left[o + node] : right[o + node];
    }
    return value[o + node];
  };
  double s = 0.0;
  for (int t = 0; t < T; ++t) s = dadd(s, leaf_value(t));
  const double mu = ddiv(s, (double)T);
  double acc = 0.0;
  for (int t = 0; t < T; ++t) {
    const double d = dsub(leaf_value(t), mu);
    acc = dadd(acc, dmul(d, d));
  }
  const double var = ddiv(acc, (double)(T - 1));     // T == 1: 0 / 0 = NaN, as np.var(ddof=1)
  if (mean_out) mean_out[m] = mu;
  if (var_out) var_out[m] = var;
  if (ei_out) {
    const double sd = sqrt(var) + 0.0001;
    const double u = (best - mu) / sd;
    const double cdf = 0.5 * erfc(-u * 0.7071067811865476);
    const double pdf = 0.3989422804014327 * exp(-0.5 * u * u);
    ei_out[m] = sd * (u * cdf + pdf);
  }
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static void forest_layout(int N, int D, int T, size_t* off) {
  size_t o = 0;
  off[0] = o; o += align256(sizeof(float) * (size_t)D * N);              // Xt
  off[1] = o; o += align256(sizeof(int) * (size_t)D * N);                // order
  off[2] = o; o += align256(sizeof(int) * (size_t)T * D * N);            // lists
  off[3] = o; o += align256(sizeof(int) * (size_t)T * D * N);            // tmp
  off[4] = o; o += align256(sizeof(int) * (size_t)T * N);                // samples
  off[5] = o; o += align256(sizeof(StackRec) * (size_t)T * (N + 1));     // stack
  off[6] = o;
}

size_t forest_workspace_bytes(int N, int D, int T) {
  if (N < 1 || D < 1 || T < 1) return 0;
  size_t off[7];
  forest_layout(N, D, T, off);
  return off[6];
}

static size_t forest_smem(int D) { return (size_t)D * (2 * sizeof(double) + 4 * sizeof(int)); }

int forest_fit(int N, int D, int T, const float* X, const double* y, const double* w, const uint32_t* rand_r_state,
               int max_features, int max_depth, int min_samples_split, int ldn, int* feature, double* threshold,
               int* left, int* right, int* n_node_samples, double* value, int* node_count, void* ws, size_t ws_bytes,
               cudaStream_t st) {
  if (N < 1) return -1;
  if (D < 1) return -2;
  if (T < 1) return -3;
  if (!X) return -4;
  if (!y) return -5;
  if (!w) return -6;
  if (!rand_r_state) return -7;
  if (max_features < 1) return -8;
  if (max_depth < 0) return -9;
  if (min_samples_split < 2) return -10;
  if (ldn < 2 * N - 1) return -11;
  if (!feature) return -12;
  if (!threshold) return -13;
  if (!left) return -14;
  if (!right) return -15;
  if (!n_node_samples) return -16;
  if (!value) return -17;
  if (!node_count) return -18;
  if (!ws || ws_bytes < forest_workspace_bytes(N, D, T)) return -20;
  const size_t smem = forest_smem(D);
  int dev = 0, smem_max = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (smem + 1024 > (size_t)smem_max) return -2;      // D beyond the per-tree feature arrays in shared memory
  size_t off[7];
  forest_layout(N, D, T, off);
  char* base = static_cast<char*>(ws);
  FitArgs a;
  a.N = N; a.D = D; a.max_features = max_features; a.max_depth = max_depth; a.min_samples_split = min_samples_split;
  a.ldn = ldn;
  a.Xt = reinterpret_cast<float*>(base + off[0]);
  a.y = y; a.w = w; a.rand_r = rand_r_state;
  a.order = reinterpret_cast<int*>(base + off[1]);
  a.lists = reinterpret_cast<int*>(base + off[2]);
  a.tmp = reinterpret_cast<int*>(base + off[3]);
  a.samples = reinterpret_cast<int*>(base + off[4]);
  a.stack = reinterpret_cast<StackRec*>(base + off[5]);
  a.feature = feature; a.left = left; a.right = right; a.n_node_samples = n_node_samples; a.node_count = node_count;
  a.threshold = threshold; a.value = value;
  const long ND = (long)N * D;
  forest_transpose_kernel<<<(unsigned)((ND + 255) / 256), 256, 0, st>>>(N, D, X, const_cast<float*>(a.Xt));
  forest_rank_sort_kernel<<<dim3((N + 255) / 256, D), 256, 0, st>>>(N, a.Xt, const_cast<int*>(a.order));
  if (smem > 48 * 1024) cudaFuncSetAttribute(forest_fit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  timing_begin("forest_fit_kernel", st);
  forest_fit_kernel<<<T, kForestThreads, smem, st>>>(a);
  timing_end(st);
  count_launch(3);
  return check_launch("forest_fit");
}

int forest_predict_ei(int M, int D, int T, int ldn, const float* C, const int* feature, const double* threshold,
                      const int* left, const int* right, const double* value, double best, double* mean, double* var,
                      double* ei, cudaStream_t st) {
  if (M < 0) return -1;
  if (D < 1) return -2;
  if (T < 1) return -3;
  if (ldn < 1) return -4;
  if (!C && M > 0) return -5;
  if (!feature) return -6;
  if (!threshold) return -7;
  if (!left) return -8;
  if (!right) return -9;
  if (!value) return -10;
  if (M == 0) return 0;
  timing_begin("forest_predict_ei_kernel", st);
  forest_predict_ei_kernel<<<(M + 127) / 128, 128, 0, st>>>(M, D, T, ldn, C, feature, threshold, left, right, value, best,
                                                            mean, var, ei);
  timing_end(st);
  count_launch(1);
  return check_launch("forest_predict_ei");
}

}  // namespace smk
