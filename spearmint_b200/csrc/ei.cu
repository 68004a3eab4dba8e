// ei.cu -- the acquisition scan over candidates and the final selection.
//
// EI sweep (reference OPT:551-555; with pending fantasies OPT:613-619; per-second PSEC:490-491, 548):
//     s = sqrt(var); u = (best - mu)/s; EI = s*(u*Phi(u) + phi(u));  mean over the F fantasies;
//     optionally divided by exp(predicted log-duration).
// One thread per candidate, samples in the inner loop: every load is a fully coalesced 128-byte warp
// row of mu[s][f][:] / var[s][:], the kernel is a pure HBM sweep (8 bytes in + 4 out per pair without
// fantasies).  EI is STORED in double and evaluated in double wherever float32 would not do: u*Phi(u) + phi(u) cancels
// catastrophically for u << 0 and the chooser ranks candidates by exactly those tail values late in a run (ei_one_f32).
//
// Selection (reference OPT:270-271 argsort(mean)[-k:], OPT:294 argmax(mean)): two-stage top-k.
#include "common.cuh"

namespace smk {

__device__ __forceinline__ double ei_one(double best, double m, double v) {
  if (!(v > 0.0)) return fmax(best - m, 0.0);   // reference would produce NaN (sqrt of a negative)
  const double s = sqrt(v);
  const double u = (best - m) / s;
  const double cdf = 0.5 * erfc(-u * 0.7071067811865476);
  const double pdf = 0.3989422804014327 * exp(-0.5 * u * u);
  return s * (u * cdf + pdf);
}

// float32 moments (the grid path): the expression is evaluated in float32 wherever that is exact enough -- u > -4, where
// u Phi(u) + phi(u) cancels by less than a factor 20 and erfcf / expf keep the result within ~5e-6 relative of the double
// value (the moments themselves carry 1e-4) -- and in double in the tail, where the chooser ranks candidates by values
// that float32 would flush to zero.  This is what makes the sweep an HBM sweep (12-16 bytes per pair against ~45
// float32 instructions) instead of an fp64-ALU loop.  The result is a double either way.
__device__ __forceinline__ double ei_one(double best, float m, float v) { return ei_one(best, (double)m, (double)v); }
__device__ __forceinline__ double ei_one_f32(float best, float m, float v) {
  if (v > 0.f) {
    const float s = sqrtf(v);
    const float u = (best - m) / s;
    if (u > -4.0f) {
      const float cdf = 0.5f * erfcf(-u * 0.70710678f);
      const float pdf = 0.39894228f * expf(-0.5f * u * u);
      return (double)(s * fmaf(u, cdf, pdf));
    }
  }
  return ei_one((double)best, (double)m, (double)v);
}
__device__ __forceinline__ double ei_fast(float best, float m, float v) { return ei_one_f32(best, m, v); }
__device__ __forceinline__ double ei_fast(double best, double m, double v) { return ei_one(best, m, v); }

// EI of candidate j under sample s (mean over the F fantasies, optional division by the predicted duration)
template <typename T>
__device__ __forceinline__ double ei_cand(int F, const T* mu, const T* var, int ldm, const T* best, const T* log_time, int s,
                                          int j) {
  const T* mrow = mu + (long)s * F * ldm + j;
  const T* brow = best + (long)s * F;
  double acc = 0.0;
  for (int f = 0; f < F; ++f) acc += ei_fast(brow[f], mrow[(long)f * ldm], var[(long)s * ldm + j]);
  double e = (F > 1) ? acc / (double)F : acc;
  if (log_time) e /= exp((double)log_time[(long)s * ldm + j]);
  return e;
}

// Variant of the sweep that also leaves max_j EI[s][j] in ei_max[s] (the accuracy guard of the engine compares it with
// the error bound of the explicit-inverse path).  One warp-level + one atomic reduction per (block, sample).
template <typename T>
__device__ __forceinline__ void ei_sweep_with_max(int M, int S, int F, const T* mu, const T* var, int ldm, const T* best,
                                                  const T* log_time, double* ei, double* ei_sum, unsigned long long* ei_max,
                                                  int j) {
  double total = 0.0;
  for (int s = 0; s < S; ++s) {
    double e = 0.0;
    if (j < M) {
      e = ei_cand<T>(F, mu, var, ldm, best, log_time, s, j);
      if (ei) ei[(long)s * ldm + j] = e;
      total += e;
    }
    double m = (e == e) ? e : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.0) atomicMax(&ei_max[s], (unsigned long long)__double_as_longlong(m));
  }
  if (ei_sum && j < M) ei_sum[j] += total;
}

// EI values leave the kernel as DOUBLE for both element types: in the deep-tail regime (late in a run max EI can be
// 1e-50 and smaller) float32 storage flushes every candidate to zero and the argmax degenerates, while the reference
// ranks those values in float64.
template <typename T>
__global__ void __launch_bounds__(256) ei_sweep_kernel(int M, int S, int F, const T* __restrict__ mu,
                                                        const T* __restrict__ var, int ldm,
                                                        const T* __restrict__ best, const T* __restrict__ log_time,
                                                        double* __restrict__ ei, double* __restrict__ ei_sum,
                                                        unsigned long long* __restrict__ ei_max) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (ei_max) {            // per-sample maximum (bits of a non-negative double order like unsigned integers); small M only costs
    ei_sweep_with_max<T>(M, S, F, mu, var, ldm, best, log_time, ei, ei_sum, ei_max, j);
    return;
  }
  if (j >= M) return;
  double total = 0.0;
  if (F == 1) {
    int s = 0;
    for (; s + 4 <= S; s += 4) {  // 8 independent loads in flight per thread
      T m[4], v[4], lt[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        m[q] = mu[(long)(s + q) * ldm + j];
        v[q] = var[(long)(s + q) * ldm + j];
        lt[q] = log_time ? log_time[(long)(s + q) * ldm + j] : T(0);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        double e = ei_fast(best[s + q], m[q], v[q]);
        if (log_time) e /= exp((double)lt[q]);
        if (ei) ei[(long)(s + q) * ldm + j] = e;
        total += e;
      }
    }
    for (; s < S; ++s) {
      double e = ei_fast(best[s], mu[(long)s * ldm + j], var[(long)s * ldm + j]);
      if (log_time) e /= exp((double)log_time[(long)s * ldm + j]);
      if (ei) ei[(long)s * ldm + j] = e;
      total += e;
    }
  } else {
    for (int s = 0; s < S; ++s) {
      const T* mrow = mu + (long)s * F * ldm + j;
      const T* brow = best + (long)s * F;
      double acc = 0.0;
      int f = 0;
      for (; f + 4 <= F; f += 4) {
        T m[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) m[q] = mrow[(long)(f + q) * ldm];
#pragma unroll
        for (int q = 0; q < 4; ++q) acc += ei_fast(brow[f + q], m[q], var[(long)s * ldm + j]);
      }
      for (; f < F; ++f) acc += ei_fast(brow[f], mrow[(long)f * ldm], var[(long)s * ldm + j]);
      double e = acc / (double)F;
      if (log_time) e /= exp((double)log_time[(long)s * ldm + j]);
      if (ei) ei[(long)s * ldm + j] = e;
      total += e;
    }
  }
  if (ei_sum) ei_sum[j] += total;
}

template <typename T>
int ei_sweep(int M, int S, int F, const T* mu, const T* var, int ldm, const T* best, const T* log_time, double* ei,
             double* ei_sum, unsigned long long* ei_max, cudaStream_t st) {
  if (M <= 0) return -1;
  if (S <= 0) return -2;
  if (F <= 0) return -3;
  if (!mu) return -4;
  if (!var) return -5;
  if (ldm < M) return -6;
  if (!best) return -7;
  if (ei_max) cudaMemsetAsync(ei_max, 0, sizeof(unsigned long long) * S, st);
  ei_sweep_kernel<T><<<(M + 255) / 256, 256, 0, st>>>(M, S, F, mu, var, ldm, best, log_time, ei, ei_sum, ei_max);
  count_launch();
  return check_launch("ei_sweep");
}

template int ei_sweep<float>(int, int, int, const float*, const float*, int, const float*, const float*, double*,
                             double*, unsigned long long*, cudaStream_t);
template int ei_sweep<double>(int, int, int, const double*, const double*, int, const double*, const double*,
                              double*, double*, unsigned long long*, cudaStream_t);

// Probability-weighted sweep of the constrained chooser (CONS:878, 940): EI (mean over the F fantasies first) times the
// probability of feasibility w[s][j] (constraint.cu), otherwise the contract of ei_sweep.  w is double: Phi deep in its
// tail is far below the float32 range, and so is the product the chooser ranks.
template <typename T>
__global__ void __launch_bounds__(256) ei_sweep_weighted_kernel(int M, int S, int F, const T* __restrict__ mu,
                                                                 const T* __restrict__ var, int ldm,
                                                                 const T* __restrict__ best, const double* __restrict__ w,
                                                                 double* __restrict__ ei, double* __restrict__ ei_sum,
                                                                 unsigned long long* __restrict__ ei_max) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  double total = 0.0;
  for (int s = 0; s < S; ++s) {
    double e = 0.0;
    if (j < M) {
      e = ei_cand<T>(F, mu, var, ldm, best, nullptr, s, j) * w[(long)s * ldm + j];
      if (ei) ei[(long)s * ldm + j] = e;
      total += e;
    }
    if (ei_max) {
      double m = (e == e) ? e : 0.0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
      if ((threadIdx.x & 31) == 0 && m > 0.0) atomicMax(&ei_max[s], (unsigned long long)__double_as_longlong(m));
    }
  }
  if (ei_sum && j < M) ei_sum[j] += total;
}

template <typename T>
int ei_sweep_weighted(int M, int S, int F, const T* mu, const T* var, int ldm, const T* best, const double* w, double* ei,
                      double* ei_sum, unsigned long long* ei_max, cudaStream_t st) {
  if (M <= 0) return -1;
  if (S <= 0) return -2;
  if (F <= 0) return -3;
  if (!mu) return -4;
  if (!var) return -5;
  if (ldm < M) return -6;
  if (!best) return -7;
  if (!w) return -8;
  if (ei_max) cudaMemsetAsync(ei_max, 0, sizeof(unsigned long long) * S, st);
  ei_sweep_weighted_kernel<T><<<(M + 255) / 256, 256, 0, st>>>(M, S, F, mu, var, ldm, best, w, ei, ei_sum, ei_max);
  count_launch();
  return check_launch("ei_sweep_weighted");
}

template int ei_sweep_weighted<float>(int, int, int, const float*, const float*, int, const float*, const double*,
                                      double*, double*, unsigned long long*, cudaStream_t);
template int ei_sweep_weighted<double>(int, int, int, const double*, const double*, int, const double*, const double*,
                                       double*, double*, unsigned long long*, cudaStream_t);

// ei_sum[j] += sum_s ei[s][j]  (column sum of the per-sample EI matrix; fixed order -> deterministic)
__global__ void __launch_bounds__(256) ei_colsum_kernel(int M, int S, const double* __restrict__ ei, int ldm,
                                                         double* __restrict__ ei_sum) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= M) return;
  double t = 0.0;
  for (int s = 0; s < S; ++s) t += ei[(long)s * ldm + j];
  ei_sum[j] += t;
}
int ei_colsum(int M, int S, const double* ei, int ldm, double* ei_sum, cudaStream_t st) {
  if (M <= 0 || S <= 0) return -1;
  if (!ei || !ei_sum || ldm < M) return -3;
  ei_colsum_kernel<<<(M + 255) / 256, 256, 0, st>>>(M, S, ei, ldm, ei_sum);
  count_launch();
  return check_launch("ei_colsum");
}

// ------------------------------------------------------------------------------------------- top-k
constexpr int kSlice = 4096;   // candidates per stage-1 block
constexpr int kMaxK = 256;

template <typename T>
__device__ __forceinline__ bool better(T v, int i, T bv, int bi) {
  return (v > bv) || (v == bv && i < bi);   // larger value, ties to the lower index (numpy first-max)
}

// Extracts the k best of vals[0..n) (shared memory, destroyed) into out_val/out_idx (descending).
template <typename T>
__device__ void extract_topk(T* vals, const int* idx, int n, int k, T* out_val, int* out_idx, T* wv, int* wi) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int it = 0; it < k; ++it) {
    T bv = -INFINITY;
    int bi = 0x7fffffff, bpos = -1;
    for (int e = tid; e < n; e += 256) {
      T v = vals[e];
      int gi = idx ? idx[e] : e;
      if (v == v && (bpos < 0 || better(v, gi, bv, bi))) { bv = v; bi = gi; bpos = e; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      T ov = __shfl_xor_sync(0xffffffffu, bv, o);
      int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      int op = __shfl_xor_sync(0xffffffffu, bpos, o);
      if (op >= 0 && (bpos < 0 || better(ov, oi, bv, bi))) { bv = ov; bi = oi; bpos = op; }
    }
    __syncthreads();
    if (lane == 0) { wv[warp] = bv; wi[warp] = bi; wi[8 + warp] = bpos; }
    __syncthreads();
    if (tid == 0) {
      T fv = wv[0]; int fi = wi[0], fp = wi[8];
      for (int w = 1; w < 8; ++w)
        if (wi[8 + w] >= 0 && (fp < 0 || better(wv[w], wi[w], fv, fi))) { fv = wv[w]; fi = wi[w]; fp = wi[8 + w]; }
      out_val[it] = (fp >= 0) ? fv : (T)(-INFINITY);
      out_idx[it] = (fp >= 0) ? fi : -1;
      if (fp >= 0) vals[fp] = NAN;   // NaN marks "taken" (and genuine NaNs are never selected)
    }
    __syncthreads();
  }
}

template <typename T>
__global__ void __launch_bounds__(256) topk_stage1(int M, int k, const T* __restrict__ score, T* pv, int* pi) {
  __shared__ T vals[kSlice];
  __shared__ T wv[8];
  __shared__ int wi[16];
  __shared__ T ov[kMaxK];
  __shared__ int oi[kMaxK];
  const int b0 = blockIdx.x * kSlice;
  const int n = min(kSlice, M - b0);
  for (int e = threadIdx.x; e < n; e += 256) vals[e] = score[b0 + e];
  __syncthreads();
  extract_topk<T>(vals, nullptr, n, k, ov, oi, wv, wi);
  for (int e = threadIdx.x; e < k; e += 256) {
    pv[(long)blockIdx.x * k + e] = ov[e];
    pi[(long)blockIdx.x * k + e] = (oi[e] >= 0) ? oi[e] + b0 : -1;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) topk_stage2(int n, int k, T* pv, int* pi, int* idx_out, T* val_out) {
  __shared__ T wv[8];
  __shared__ int wi[16];
  __shared__ T ov[kMaxK];
  __shared__ int oi[kMaxK];
  // stage-1 partials stay in global memory (n = blocks*k can exceed shared memory); -1 indices are
  // empty slots and carry -inf values.
  for (int e = threadIdx.x; e < n; e += 256)
    if (pi[e] < 0) pv[e] = NAN;
  __syncthreads();
  extract_topk<T>(pv, pi, n, k, ov, oi, wv, wi);
  for (int e = threadIdx.x; e < k; e += 256) {  // ascending score order, argmax last
    idx_out[k - 1 - e] = oi[e];
    if (val_out) val_out[k - 1 - e] = ov[e];
  }
}

size_t topk_workspace_bytes(int M, int k) {
  size_t blocks = ((size_t)M + kSlice - 1) / kSlice;
  return blocks * (size_t)k * (sizeof(double) + sizeof(int));
}

template <typename T>
int topk(int M, int k, const T* score, int* idx_out, T* val_out, void* workspace, size_t workspace_bytes,
         cudaStream_t st) {
  if (M <= 0) return -1;
  if (k <= 0 || k > kMaxK || k > M) return -2;
  if (!score) return -3;
  if (!idx_out) return -4;
  if (!workspace || workspace_bytes < topk_workspace_bytes(M, k)) return -6;
  const int blocks = (M + kSlice - 1) / kSlice;
  T* pv = reinterpret_cast<T*>(workspace);
  int* pi = reinterpret_cast<int*>(reinterpret_cast<unsigned char*>(workspace) + (size_t)blocks * k * sizeof(double));
  topk_stage1<T><<<blocks, 256, 0, st>>>(M, k, score, pv, pi);
  topk_stage2<T><<<1, 256, 0, st>>>(blocks * k, k, pv, pi, idx_out, val_out);
  count_launch(2);
  return check_launch("topk");
}

template int topk<float>(int, int, const float*, int*, float*, void*, size_t, cudaStream_t);
template int topk<double>(int, int, const double*, int*, double*, void*, size_t, cudaStream_t);

}  // namespace smk
