// potrf.cu -- batched blocked right-looking lower Cholesky (reference: spla.cholesky(K, lower=True)
// at OPT:540, OPT:567, OPT:585 and inside every slice-sampler logprob OPT:637, 659, 690).
//
// Per block column j (NB = 128 for float, 64 for double), for ALL hyper-samples at once (grid.z):
//   diag     : L_jj = chol(A_jj) in shared memory, W_jj = L_jj^-1 (kept: every later triangular
//              solve multiplies by W_jj instead of substituting)
//   panel    : L_Ij = A_Ij * W_jj^T                       (block GEMM, I > j)
//   trailing : A_IK -= L_Ij * L_Kj^T   for I >= K > j     (block SYRK/GEMM)
// The trailing update carries N^3/3 of the flops and is the tensor-core candidate (DESIGN.md).
#include "common.cuh"
#include "diag.cuh"

namespace smk {

// ------------------------------------------------------------------------------------------ diag
// Factor one NB x NB diagonal block on one SM (diag.cuh).  This kernel is the serial spine of the factorisation: nblk
// launches per matrix, so its latency -- not its flops -- is what matters.  It leaves the inverses of the four (two)
// 32 x 32 diagonal pieces in the first NB x 32 elements of the block's winv slot; potrf_winv_kernel expands them to the
// full W_jj = L_jj^-1 after the factorisation, off the spine.
template <typename T>
__global__ void __launch_bounds__(256) potrf_diag_kernel(int Npad, int jb, T* __restrict__ A,
                                                          T* __restrict__ winv, int* __restrict__ info) {
  constexpr int NB = Cfg<T>::NB;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int s = blockIdx.x;
  T* Ab = A + (long)s * Npad * Npad + (long)jb * NB * Npad + (long)jb * NB;
  T* Wb = winv + ((long)s * (Npad / NB) + jb) * NB * NB;
  diag_factor_block<T, NB>(Ab, Npad, Wb, info + s, jb * NB, reinterpret_cast<T*>(smem_raw));
}

// ------------------------------------------------------------------------------------------ panel
// L_Ij = A_Ij L_jj^-T by block substitution, 32 rows per CTA (diag.cuh: panel_sub_block); optional tf32 (hi, lo) copies
// of the finished panel for the tensor-core update.  grid = (rows below / 32, 1, S).
template <typename T>
__global__ void __launch_bounds__(256) potrf_panel_kernel(int Npad, int jb, T* __restrict__ A,
                                                           const T* __restrict__ winv, T* __restrict__ hi = nullptr,
                                                           T* __restrict__ lo = nullptr) {
  constexpr int NB = Cfg<T>::NB;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int s = blockIdx.z;
  const long base = (long)s * Npad * Npad;
  const long off = base + ((long)(jb + 1) * NB + (long)blockIdx.x * 32) * Npad + (long)jb * NB;
  const T* Ljj = A + base + (long)jb * NB * Npad + (long)jb * NB;
  const T* wd = winv + ((long)s * (Npad / NB) + jb) * NB * NB;
  panel_sub_block<T, NB>(A + off, Npad, Ljj, wd, hi ? hi + off : nullptr, lo ? lo + off : nullptr,
                         reinterpret_cast<T*>(smem_raw));
}

// ------------------------------------------------------------------------------------------ full inverse blocks
// W_jj = L_jj^-1 for every diagonal block of every sample at once (grid = (nblk, S)), after the factorisation.
template <typename T>
__global__ void __launch_bounds__(256) potrf_winv_kernel(int Npad, const T* __restrict__ A, T* __restrict__ winv, int jb0) {
  constexpr int NB = Cfg<T>::NB;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int jb = jb0 + blockIdx.x, s = blockIdx.y;
  const T* Ljj = A + (long)s * Npad * Npad + (long)jb * NB * Npad + (long)jb * NB;
  T* Wb = winv + ((long)s * (Npad / NB) + jb) * NB * NB;
  winv_assemble_block<T, NB>(Ljj, Npad, Wb, Wb, reinterpret_cast<T*>(smem_raw));
}

template <typename T>
static void potrf_set_attrs() {
  constexpr int NB = Cfg<T>::NB;
  static bool done = false;
  if (done) return;
  cudaFuncSetAttribute(potrf_diag_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)DiagSmem<T, NB>::bytes);
  cudaFuncSetAttribute(potrf_panel_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PanelSmem<T, NB>::bytes);
  cudaFuncSetAttribute(potrf_winv_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WinvSmem<T, NB>::bytes);
  done = true;
}

// --------------------------------------------------------------------------------------- trailing
// A_IK -= L[I, jb:jb+kd] * L[K, jb:jb+kd]^T   for c0 <= K <= I   (grid.x = I - c0, grid.y = K - c0), kd = depth in
// block columns: the driver updates block columns in PAIRS (rank 2*NB), halving the accumulator load/store traffic.
template <typename T>
__global__ void __launch_bounds__(256, 2) potrf_trailing_kernel(int Npad, int jb, int kd, int c0, T* __restrict__ A) {
  using C = Cfg<T>;
  constexpr int NB = C::NB;
  if (blockIdx.y > blockIdx.x) return;
  __shared__ TileSmem<T> sm;
  const int s = blockIdx.z, I = c0 + blockIdx.x, K = c0 + blockIdx.y;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  T* As = A + (long)s * Npad * Npad;
  T* Aik = As + (long)I * NB * Npad + (long)K * NB;
  const T* Lij = As + (long)I * NB * Npad + (long)jb * NB;
  const T* Lkj = As + (long)K * NB * Npad + (long)jb * NB;
  T acc[C::TM][C::TN];
#pragma unroll
  for (int r = 0; r < C::TM; ++r)
#pragma unroll
    for (int g = 0; g < C::TN / 4; ++g) {
      V4<T> v = ld4(Aik + (long)tile_row(ty, r) * Npad + tile_col(tx, g * 4));
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[r][g * 4 + e] = v.v[e];
    }
  TileGemm<T, Lay::KContig, Lay::KContig, true>::run(acc, Lij, Npad, Lkj, Npad, kd * NB, sm);
#pragma unroll
  for (int r = 0; r < C::TM; ++r)
#pragma unroll
    for (int g = 0; g < C::TN / 4; ++g) {
      V4<T> v;
#pragma unroll
      for (int e = 0; e < 4; ++e) v.v[e] = acc[r][g * 4 + e];
      st4(Aik + (long)tile_row(ty, r) * Npad + tile_col(tx, g * 4), v);
    }
}

template <typename T>
int potrf_lower_batched(int Npad, int S, T* A, T* winv, int* info, cudaStream_t st) {
  constexpr int NB = Cfg<T>::NB;
  if (Npad <= 0 || Npad % kNpadMult) return -1;
  if (S <= 0) return -2;
  if (!A) return -3;
  if (!winv) return -4;
  if (!info) return -5;
  const int nblk = Npad / NB;
  const size_t dsm = DiagSmem<T, NB>::bytes, psm = PanelSmem<T, NB>::bytes, wsm = WinvSmem<T, NB>::bytes;
  potrf_set_attrs<T>();
  cudaMemsetAsync(info, 0, sizeof(int) * S, st);
  // Block columns in pairs (jb, jb+1): factor jb, bring only column jb+1 up to date (rank NB), factor jb+1, then ONE
  // rank-2*NB update of everything to the right.
  for (int jb = 0; jb < nblk; jb += 2) {
    potrf_diag_kernel<T><<<S, 256, dsm, st>>>(Npad, jb, A, winv, info);
    count_launch();
    int rem = nblk - jb - 1;
    if (rem <= 0) break;
    potrf_panel_kernel<T><<<dim3(rem * (NB / 32), 1, S), 256, psm, st>>>(Npad, jb, A, winv);
    potrf_trailing_kernel<T><<<dim3(rem, 1, S), 256, 0, st>>>(Npad, jb, 1, jb + 1, A);      // column jb+1 only
    potrf_diag_kernel<T><<<S, 256, dsm, st>>>(Npad, jb + 1, A, winv, info);
    count_launch(3);
    rem = nblk - jb - 2;
    if (rem <= 0) break;
    potrf_panel_kernel<T><<<dim3(rem * (NB / 32), 1, S), 256, psm, st>>>(Npad, jb + 1, A, winv);
    potrf_trailing_kernel<T><<<dim3(rem, rem, S), 256, 0, st>>>(Npad, jb, 2, jb + 2, A);   // rank 2*NB, columns >= jb+2
    count_launch(2);
  }
  potrf_winv_kernel<T><<<dim3(nblk, S), 256, wsm, st>>>(Npad, A, winv, 0);
  count_launch();
  return check_launch("potrf_lower_batched");
}

// ---- left-looking variant with the rank-(jb*NB) update of each block-column pair on the tensor cores (float32):
//   update(jb)  : A[rows >= jb][cols jb, jb+1] -= L[rows, 0:jb] L[jb:jb+2, 0:jb]^T     wgmma 3xTF32 (predict_tc.cu)
//   diag, panel : as above; the panel kernel also writes the tf32 hi/lo copies the next updates read through TMA
//   column jb+1 is brought up to date w.r.t. column jb by one rank-NB SIMT update.
int tc_chol_update(int Npad, int S, int jb, int ncols, float* A, const float* lhi, const float* llo, cudaStream_t st);

// blk_done (optional, nblk events): blk_done[j] is recorded on st once block column j is final AND the panel below it has
// read the compact diagonal inverses (the full W_jj may then overwrite them); with blk_done the full inverses are NOT
// formed here -- the caller does it per block (potrf_winv_block) as the events fire (potrf_trtri_tc, predict_tc.cu).
int potrf_lower_batched_tc(int Npad, int S, float* A, float* winv, int* info, float* lhi, float* llo, cudaStream_t st,
                           cudaEvent_t* blk_done) {
  constexpr int NB = Cfg<float>::NB;
  if (Npad <= 0 || Npad % kNpadMult) return -1;
  if (S <= 0) return -2;
  if (!A || !winv || !info || !lhi || !llo) return -3;
  const int nblk = Npad / NB;
  const size_t dsm = DiagSmem<float, NB>::bytes, psm = PanelSmem<float, NB>::bytes, wsm = WinvSmem<float, NB>::bytes;
  potrf_set_attrs<float>();
  cudaMemsetAsync(info, 0, sizeof(int) * S, st);
  auto done = [&](int j) { if (blk_done) cudaEventRecord(blk_done[j], st); };
  for (int jb = 0; jb < nblk; jb += 2) {
    if (jb > 0) {
      int rc = tc_chol_update(Npad, S, jb, (jb + 1 < nblk) ? 2 * NB : NB, A, lhi, llo, st);
      if (rc) return rc;
    }
    potrf_diag_kernel<float><<<S, 256, dsm, st>>>(Npad, jb, A, winv, info);
    count_launch();
    int rem = nblk - jb - 1;
    if (rem <= 0) { done(jb); break; }
    potrf_panel_kernel<float><<<dim3(rem * (NB / 32), 1, S), 256, psm, st>>>(Npad, jb, A, winv, lhi, llo);
    done(jb);
    potrf_trailing_kernel<float><<<dim3(rem, 1, S), 256, 0, st>>>(Npad, jb, 1, jb + 1, A);
    potrf_diag_kernel<float><<<S, 256, dsm, st>>>(Npad, jb + 1, A, winv, info);
    count_launch(3);
    rem = nblk - jb - 2;
    if (rem <= 0) { done(jb + 1); break; }
    potrf_panel_kernel<float><<<dim3(rem * (NB / 32), 1, S), 256, psm, st>>>(Npad, jb + 1, A, winv, lhi, llo);
    done(jb + 1);
    count_launch();
  }
  if (!blk_done) {
    potrf_winv_kernel<float><<<dim3(nblk, S), 256, wsm, st>>>(Npad, A, winv, 0);
    count_launch();
  }
  return check_launch("potrf_lower_batched_tc");
}

// full W_jj of block column jb (all samples): see blk_done above
void potrf_winv_block(int Npad, int S, int jb, const float* A, float* winv, cudaStream_t st) {
  potrf_set_attrs<float>();
  potrf_winv_kernel<float><<<dim3(1, S), 256, WinvSmem<float, Cfg<float>::NB>::bytes, st>>>(Npad, A, winv, jb);
  count_launch();
}

template int potrf_lower_batched<float>(int, int, float*, float*, int*, cudaStream_t);
template int potrf_lower_batched<double>(int, int, double*, double*, int*, cudaStream_t);

}  // namespace smk
