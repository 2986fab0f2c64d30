// factor.cu -- dense refactorization of the basis nucleus on the GPU.
//
// Replaces the numerical part of ClpFactorization::factorize
// (/root/reference/src/ClpFactorization.cpp:1649 -> CoinAbcTypeFactorization::factor
// src/CoinAbcBaseFactorization1.cpp:683; the dense tail factorDense ...2.cpp:976 ->
// CoinAbcDgetrf src/AbcSimplexParallel.cpp:2491 with its CoinAbcDgemm trailing update).
//
// The k x k nucleus (structural basic columns restricted to rows whose slack is nonbasic) is
// LU-factorized with partial pivoting by a blocked right-looking algorithm (panel kernel +
// row swaps + unit-lower TRSM + rank-NB DGEMM update) and the factors are then turned into
// the explicit inverse X = U^-1 L^-1 P by blocked forward/backward substitution (TRSM + DGEMM).
// Everything is fp64 FMA; the matrix is column major with leading dimension ld.
#include "engine.cuh"

#include <cooperative_groups.h>

#include <cstdio>
#include <cstdlib>
#include <dlfcn.h>

namespace clpb {

constexpr int NB = 32;

// ---- panel factorization: columns [j0, j0+nb) rows [j0, k) -------------------------------
// Cooperative multi-CTA kernel.  The rows of the panel are dealt round-robin to the CTAs
// (row j0 + c + q*gridDim.x belongs to CTA c) and live in shared memory for the whole panel,
// so global memory is read once and written once.  Per column there is ONE grid barrier: before
// it every CTA publishes its best pivot candidate (packed |value|,row key) together with that
// candidate row, and the owner of the diagonal row publishes the diagonal row; after it every
// CTA knows the pivot row, the two owners exchange the rows, and all CTAs eliminate.
constexpr int kSlabPitch = NB + 1;       // padded row pitch in shared memory (bank conflicts)
constexpr int kPanelMaxRowsPerCta = 640; // 640 rows x 33 x 8 B = 165 KB of shared memory
constexpr int kPanelMinRowsPerCta = 32;  // fewer, fatter CTAs make the per-column grid barrier cheaper

// Monotone arrival counter (never reset inside a factorization: 'target' grows by gridDim.x per
// barrier).  One acq_rel atomic per CTA + an acquire spin -- the formulation rowpass.cu found about
// twice as fast as fence + atomic + volatile spin + fence; with one barrier per matrix column that
// difference is a large share of the panel time.
__device__ __forceinline__ void grid_barrier(unsigned int *counter, unsigned int target)
{
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int o;
    asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(o) : "l"(counter), "r"(1u) : "memory");
    unsigned int v;
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    } while (v < target);
  }
  __syncthreads();
}

// rows [j0 + cta*R, j0 + (cta+1)*R) of the panel belong to CTA 'cta'
__global__ void __launch_bounds__(256)
    lu_panel_coop_kernel(double *__restrict__ A, int k, int ld, int j0, int nb, int R,
                         int *__restrict__ ipiv, int *__restrict__ info, double singularTol,
                         unsigned long long *__restrict__ pubKey, double *__restrict__ pubRows,
                         double *__restrict__ pubDiag, unsigned int *__restrict__ barrierCounter,
                         unsigned int barrierBase)
{
  extern __shared__ double slab[]; // [R][kSlabPitch]
  __shared__ unsigned long long sBest[8];
  __shared__ int sWinCta[8];
  __shared__ double urow[NB];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int G = gridDim.x, cta = blockIdx.x;
  const int r0 = j0 + cta * R;                         // first global row of this CTA
  const int rowsLocal = max(0, min(R, k - r0));
  for (int c = 0; c < nb; c++)
    for (int q = tid; q < rowsLocal; q += 256)
      slab[q * kSlabPitch + c] = A[(size_t)(j0 + c) * ld + r0 + q];
  __syncthreads();
  unsigned int bar = barrierBase;
  for (int jj = 0; jj < nb; jj++) {
    const int j = j0 + jj; // diagonal row / column
    const int ownerJ = (j - j0) / R;
    // ---- local pivot candidate over rows >= j
    unsigned long long best = 0ull;
    for (int q = tid; q < rowsLocal; q += 256) {
      const int gi = r0 + q;
      if (gi >= j) {
        const double a = fabs(slab[q * kSlabPitch + jj]);
        // key: |a| bits (low 20 bits dropped) | (0xFFFFF - relative row): ties take the smallest row
        const unsigned long long key =
            ((unsigned long long)__double_as_longlong(a) & ~0xFFFFFull) | (unsigned long long)(0xFFFFF - (gi - j0));
        best = max(best, key);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0)
      sBest[warp] = best;
    __syncthreads();
    unsigned long long cand = 0ull;
#pragma unroll
    for (int w = 0; w < 8; w++)
      cand = max(cand, sBest[w]);
    if (tid == 0)
      pubKey[(size_t)jj * G + cta] = cand;
    // publish the candidate row and (owner only) the diagonal row
    if (cand != 0ull && tid < NB) {
      const int q = j0 + (0xFFFFF - (int)(cand & 0xFFFFFull)) - r0;
      pubRows[((size_t)jj * G + cta) * NB + tid] = slab[q * kSlabPitch + tid];
    }
    if (ownerJ == cta && tid < NB)
      pubDiag[(size_t)jj * NB + tid] = slab[(j - r0) * kSlabPitch + tid];
    bar += G;
    grid_barrier(barrierCounter, bar);
    // ---- global winner (every CTA scans the G keys: identical result everywhere)
    unsigned long long win = 0ull;
    int winCta = 0;
    for (int c = tid; c < G; c += 256) {
      const unsigned long long b = ((volatile unsigned long long *)pubKey)[(size_t)jj * G + c];
      if (b > win) {
        win = b;
        winCta = c;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ob = __shfl_xor_sync(0xffffffffu, win, o);
      const int oc = __shfl_xor_sync(0xffffffffu, winCta, o);
      if (ob > win) {
        win = ob;
        winCta = oc;
      }
    }
    if (lane == 0) {
      sBest[warp] = win;
      sWinCta[warp] = winCta;
    }
    __syncthreads();
    unsigned long long wkey = 0ull;
    int wCta = 0;
#pragma unroll
    for (int w = 0; w < 8; w++)
      if (sBest[w] > wkey) {
        wkey = sBest[w];
        wCta = sWinCta[w];
      }
    const double pivAbs = __longlong_as_double((long long)(wkey & ~0xFFFFFull));
    const int piv = j0 + (0xFFFFF - (int)(wkey & 0xFFFFFull)); // global pivot row
    const bool singular = (wkey == 0ull) || !(pivAbs >= singularTol);
    if (cta == 0 && tid == 0) {
      ipiv[j] = singular ? j : piv;
      if (singular && *info == 0)
        *info = j + 1;
    }
    if (singular) {
      __syncthreads();
      continue; // uniform across the grid: leave the column, the caller repairs the basis
    }
    // pivot row values (before elimination)
    if (tid < NB)
      urow[tid] = ((volatile double *)pubRows)[((size_t)jj * G + wCta) * NB + tid];
    __syncthreads();
    // exchange: the old diagonal row moves to row piv, the pivot row moves to row j
    if (piv != j && piv >= r0 && piv < r0 + rowsLocal && tid < NB)
      slab[(piv - r0) * kSlabPitch + tid] = ((volatile double *)pubDiag)[(size_t)jj * NB + tid];
    __syncthreads();
    if (ownerJ == cta && tid < NB)
      slab[(j - r0) * kSlabPitch + tid] = urow[tid];
    __syncthreads();
    // ---- eliminate rows below the diagonal
    const double inv = 1.0 / urow[jj];
    for (int q = tid; q < rowsLocal; q += 256) {
      if (r0 + q > j) {
        double *r = slab + q * kSlabPitch;
        const double l = r[jj] * inv;
        r[jj] = l;
        for (int c = jj + 1; c < nb; c++)
          r[c] = fma(-l, urow[c], r[c]);
      }
    }
    __syncthreads();
  }
  for (int c = 0; c < nb; c++)
    for (int q = tid; q < rowsLocal; q += 256)
      A[(size_t)(j0 + c) * ld + r0 + q] = slab[q * kSlabPitch + c];
}

// ---- the same panel on ONE thread-block cluster (16 CTAs of one GPC, distributed shared memory).
// The per-column pivot exchange of lu_panel_coop_kernel costs a grid barrier plus two dependent L2 round
// trips; inside a cluster the candidate
// keys, the pivot row and the diagonal row are read straight out of the peers' shared memory and the two
// synchronisations are hardware cluster barriers.  Panels of up to 16 x kPanelMaxRowsPerCta rows.
constexpr int kPanelCluster = 16;

__global__ void __launch_bounds__(256)
    lu_panel_cluster_kernel(double *__restrict__ A, int k, int ld, int j0, int nb, int R,
                            int *__restrict__ ipiv, int *__restrict__ info, double singularTol)
{
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ double slab[]; // [R][kSlabPitch], same offset in every CTA of the cluster
  __shared__ unsigned long long sBest[8];
  __shared__ unsigned long long sKey;  // this CTA's candidate of the current column
  __shared__ unsigned long long sWin;
  __shared__ double urow[NB], drow[NB];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cta = (int)cluster.block_rank();
  const int r0 = j0 + cta * R;
  const int rowsLocal = max(0, min(R, k - r0));
  for (int c = 0; c < nb; c++)
    for (int q = tid; q < rowsLocal; q += 256)
      slab[q * kSlabPitch + c] = A[(size_t)(j0 + c) * ld + r0 + q];
  __syncthreads();
  for (int jj = 0; jj < nb; jj++) {
    const int j = j0 + jj;
    const int ownerJ = (j - j0) / R;
    unsigned long long best = 0ull;
    for (int q = tid; q < rowsLocal; q += 256) {
      const int gi = r0 + q;
      if (gi >= j) {
        const double a = fabs(slab[q * kSlabPitch + jj]);
        best = max(best, ((unsigned long long)__double_as_longlong(a) & ~0xFFFFFull) |
                             (unsigned long long)(0xFFFFF - (gi - j0)));
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0)
      sBest[warp] = best;
    __syncthreads();
    if (tid == 0) {
      unsigned long long cand = 0ull;
#pragma unroll
      for (int w = 0; w < 8; w++)
        cand = max(cand, sBest[w]);
      sKey = cand;
    }
    cluster.sync(); // every CTA's candidate is published
    if (warp == 0) {
      unsigned long long v = 0ull;
      if (lane < kPanelCluster)
        v = *cluster.map_shared_rank(&sKey, lane);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
      if (lane == 0)
        sWin = v;
    }
    __syncthreads();
    const unsigned long long wkey = sWin;
    const double pivAbs = __longlong_as_double((long long)(wkey & ~0xFFFFFull));
    const int piv = j0 + (0xFFFFF - (int)(wkey & 0xFFFFFull));
    const bool singular = (wkey == 0ull) || !(pivAbs >= singularTol);
    if (cta == 0 && tid == 0) {
      ipiv[j] = singular ? j : piv;
      if (singular && *info == 0)
        *info = j + 1;
    }
    if (singular) {
      cluster.sync(); // keep the barrier count uniform
      continue;
    }
    const int ownerP = (piv - j0) / R;
    if (tid < NB) { // pivot row and diagonal row out of their owners' slabs (distributed shared memory)
      const double *ps = cluster.map_shared_rank(slab, ownerP);
      const double *ds = cluster.map_shared_rank(slab, ownerJ);
      urow[tid] = ps[(piv - (j0 + ownerP * R)) * kSlabPitch + tid];
      drow[tid] = ds[(j - (j0 + ownerJ * R)) * kSlabPitch + tid];
    }
    cluster.sync(); // everybody holds both rows: the owners may overwrite them now
    if (piv != j && ownerP == cta && tid < NB)
      slab[(piv - r0) * kSlabPitch + tid] = drow[tid];
    __syncthreads();
    if (ownerJ == cta && tid < NB)
      slab[(j - r0) * kSlabPitch + tid] = urow[tid];
    __syncthreads();
    const double inv = 1.0 / urow[jj];
    for (int q = tid; q < rowsLocal; q += 256) {
      if (r0 + q > j) {
        double *r = slab + q * kSlabPitch;
        const double l = r[jj] * inv;
        r[jj] = l;
        for (int c = jj + 1; c < nb; c++)
          r[c] = fma(-l, urow[c], r[c]);
      }
    }
    __syncthreads();
  }
  cluster.sync(); // nobody exits while a peer may still read its shared memory
  for (int c = 0; c < nb; c++)
    for (int q = tid; q < rowsLocal; q += 256)
      A[(size_t)(j0 + c) * ld + r0 + q] = slab[q * kSlabPitch + c];
}

// Row interchanges of a panel applied to the columns left and right of it.  The nb interchanges touch
// at most 2*nb rows; lu_perm_kernel composes them into ONE permutation of those rows (perm[0] = count,
// perm[1+i] = touched row, perm[1+2*NB+i] = the row its final content comes from).  The elements are
// then moved by two fully parallel kernels through a scratch buffer -- one thread per (column, touched
// row): gather tmp[i][c] = A[from_i][c], scatter A[row_i][c] = tmp[i][c].  (One thread per column doing
// its 2*nb strided loads serially left the GPU idle.)
__global__ void lu_perm_kernel(const int *__restrict__ ipiv, int j0, int nb, int *__restrict__ perm)
{
  int *rows = perm + 1, *from = perm + 1 + 2 * NB;
  int n = 0;
  for (int jj = 0; jj < nb; jj++) {
    const int j = j0 + jj, p = ipiv[j];
    if (p == j)
      continue;
    int a = -1, b = -1;
    for (int i = 0; i < n; i++) {
      if (rows[i] == j)
        a = i;
      if (rows[i] == p)
        b = i;
    }
    if (a < 0) {
      a = n++;
      rows[a] = j;
      from[a] = j;
    }
    if (b < 0) {
      b = n++;
      rows[b] = p;
      from[b] = p;
    }
    const int t = from[a];
    from[a] = from[b];
    from[b] = t;
  }
  perm[0] = n;
}
// columns are indexed linearly over [0, left) U [right0, right0 + nright)
__global__ void __launch_bounds__(128)
    lu_swap_gather_kernel(const double *__restrict__ A, int ld, const int *__restrict__ perm, int left,
                          int right0, int ncols, double *__restrict__ tmp)
{
  const int i = blockIdx.y;
  if (i >= perm[0])
    return;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= ncols)
    return;
  const int c = q < left ? q : q - left + right0;
  tmp[(size_t)i * ncols + q] = A[(size_t)c * ld + perm[1 + 2 * NB + i]];
}
__global__ void __launch_bounds__(128)
    lu_swap_scatter_kernel(double *__restrict__ A, int ld, const int *__restrict__ perm, int left,
                           int right0, int ncols, const double *__restrict__ tmp)
{
  const int i = blockIdx.y;
  if (i >= perm[0])
    return;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= ncols)
    return;
  if (perm[1 + i] == perm[1 + 2 * NB + i])
    return;
  const int c = q < left ? q : q - left + right0;
  A[(size_t)c * ld + perm[1 + i]] = tmp[(size_t)i * ncols + q];
}

// B[j0..j0+nb, c] := T^-1 B[.., c] for columns c in [c0,c1); T = nb x nb triangle of A at (j0,j0)
//   lower=true : unit lower triangular (forward substitution)
//   lower=false: upper triangular with diagonal (backward substitution)
__global__ void __launch_bounds__(128)
    trsm_kernel(const double *__restrict__ A, int lda, double *__restrict__ B, int ldb, int j0,
                int nb, int c0, int c1, bool lower)
{
  __shared__ double T[NB][NB + 1];
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    int i = e % NB, l = e / NB;
    T[i][l] = (i < nb && l < nb) ? A[(size_t)(j0 + l) * lda + j0 + i] : (i == l ? 1.0 : 0.0);
  }
  __syncthreads();
  int c = c0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= c1)
    return;
  double *col = B + (size_t)c * ldb + j0;
  double x[NB];
#pragma unroll
  for (int i = 0; i < NB; i++)
    x[i] = i < nb ? col[i] : 0.0;
  if (lower) {
#pragma unroll
    for (int i = 1; i < NB; i++) {
      double s = x[i];
#pragma unroll
      for (int l = 0; l < i; l++)
        s = fma(-T[i][l], x[l], s);
      x[i] = s;
    }
  } else {
#pragma unroll
    for (int i = NB - 1; i >= 0; i--) {
      double s = x[i];
#pragma unroll
      for (int l = i + 1; l < NB; l++)
        s = fma(-T[i][l], x[l], s);
      x[i] = s / T[i][i];
    }
  }
#pragma unroll
  for (int i = 0; i < NB; i++)
    if (i < nb)
      col[i] = x[i];
}

// C[M x N] -= A[M x K] * B[K x N]  (column major).  64x64 tile per CTA, 4x4 per thread.
__global__ void __launch_bounds__(256)
    gemm_sub_kernel(double *__restrict__ C, int ldc, const double *__restrict__ A, int lda,
                    const double *__restrict__ B, int ldb, int M, int N, int K)
{
  __shared__ double As[16][64 + 1];
  __shared__ double Bs[16][64 + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
      acc[a][b] = 0.0;
  for (int k0 = 0; k0 < K; k0 += 16) {
    // A tile: 64 rows x 16 cols ; B tile: 16 rows x 64 cols
    for (int e = threadIdx.x; e < 64 * 16; e += 256) {
      int i = e & 63, l = e >> 6;
      int gi = m0 + i, gl = k0 + l;
      As[l][i] = (gi < M && gl < K) ? A[(size_t)gl * lda + gi] : 0.0;
    }
    for (int e = threadIdx.x; e < 64 * 16; e += 256) {
      int l = e & 15, jn = e >> 4;
      int gl = k0 + l, gj = n0 + jn;
      Bs[l][jn] = (gl < K && gj < N) ? B[(size_t)gj * ldb + gl] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int l = 0; l < 16; l++) {
      double av[4], bv[4];
#pragma unroll
      for (int a = 0; a < 4; a++)
        av[a] = As[l][tx + 16 * a];
#pragma unroll
      for (int b = 0; b < 4; b++)
        bv[b] = Bs[l][ty + 16 * b];
#pragma unroll
      for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++)
          acc[a][b] = fma(av[a], bv[b], acc[a][b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int b = 0; b < 4; b++) {
    int gj = n0 + ty + 16 * b;
    if (gj >= N)
      continue;
#pragma unroll
    for (int a = 0; a < 4; a++) {
      int gi = m0 + tx + 16 * a;
      if (gi < M)
        C[(size_t)gj * ldc + gi] -= acc[a][b];
    }
  }
}

// cuBLAS (through dlopen, like NCCL in capi.cu: no link-time dependency) for the plain DGEMMs of
// the refactorization -- the rank-32 trailing updates of the LU and the rank-128 updates of the
// blocked inverse are ordinary C -= A*B with no fusion opportunity.  Falls back to gemm_sub_kernel
// when the library cannot be loaded.
namespace {
typedef void *cublasHandle_t_;
typedef int (*cublasCreate_t)(cublasHandle_t_ *);
typedef int (*cublasSetStream_t)(cublasHandle_t_, cudaStream_t);
typedef int (*cublasDgemm_t)(cublasHandle_t_, int, int, int, int, int, const double *, const double *, int,
                             const double *, int, const double *, double *, int);
cublasHandle_t_ g_blas = nullptr;
cublasSetStream_t p_setStream = nullptr;
cublasDgemm_t p_dgemm = nullptr;
int g_blasState = 0; // 0 untried, 1 ready, -1 unavailable
bool blas_ready()
{
  if (g_blasState != 0)
    return g_blasState > 0;
  g_blasState = -1;
  const char *names[] = {"libcublas.so.12", "/usr/local/cuda/lib64/libcublas.so.12", "libcublas.so", nullptr};
  void *h = nullptr;
  for (int i = 0; names[i] && !h; i++)
    h = dlopen(names[i], RTLD_NOW | RTLD_GLOBAL);
  if (!h)
    return false;
  cublasCreate_t p_create = (cublasCreate_t)dlsym(h, "cublasCreate_v2");
  p_setStream = (cublasSetStream_t)dlsym(h, "cublasSetStream_v2");
  p_dgemm = (cublasDgemm_t)dlsym(h, "cublasDgemm_v2");
  if (!p_create || !p_setStream || !p_dgemm)
    return false;
  if (p_create(&g_blas) != 0 || !g_blas)
    return false;
  g_blasState = 1;
  return true;
}
} // namespace

static void gemm_sub(double *C, int ldc, const double *A, int lda, const double *B, int ldb, int M,
                     int N, int K, cudaStream_t s)
{
  if (M <= 0 || N <= 0 || K <= 0)
    return;
  if ((long)M * N >= 256L * 256L && blas_ready()) {
    const double minusOne = -1.0, one = 1.0;
    p_setStream(g_blas, s);
    if (p_dgemm(g_blas, 0 /* N */, 0 /* N */, M, N, K, &minusOne, A, lda, B, ldb, &one, C, ldc) == 0)
      return;
  }
  dim3 grid((M + 63) / 64, (N + 63) / 64);
  gemm_sub_kernel<<<grid, 256, 0, s>>>(C, ldc, A, lda, B, ldb, M, N, K);
}

__global__ void set_permuted_identity_kernel(double *__restrict__ X, int k, int ld,
                                             const int *__restrict__ perm)
{
  // X = P : row i of P has its one in column perm[i]
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)ld * k;
  if (idx >= total)
    return;
  int i = (int)(idx % ld), c = (int)(idx / ld);
  X[idx] = (i < k && perm[i] == c) ? 1.0 : 0.0;
}

__global__ void transpose_kernel(const double *__restrict__ src, double *__restrict__ dst, int k,
                                 int ld)
{
  __shared__ double tile[32][33];
  int x = blockIdx.x * 32 + threadIdx.x, y0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    int y = y0 + r;
    tile[r][threadIdx.x] = (x < k && y < k) ? src[(size_t)y * ld + x] : 0.0;
  }
  __syncthreads();
  int xo = blockIdx.y * 32 + threadIdx.x, yo0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    int yo = yo0 + r;
    if (xo < ld && yo < k)
      dst[(size_t)yo * ld + xo] = (xo < k) ? tile[threadIdx.x][r] : 0.0;
  }
}
void launch_transpose(const double *src, double *dst, int k, int ld, cudaStream_t s)
{
  if (k <= 0)
    return;
  dim3 grid((ld + 31) / 32, (k + 31) / 32);
  transpose_kernel<<<grid, dim3(32, 8), 0, s>>>(src, dst, k, ld);
}

// zero the padding columns/rows [k, ld) of every row so GEMVs can run over ld
__global__ void zero_padding_kernel(double *__restrict__ M, int k, int ld)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k)
    return;
  for (int j = k; j < ld; j++)
    M[(size_t)i * ld + j] = 0.0;
}

cudaError_t lu_workspace_reserve(LuWorkspace &w, int maxK, int swapK)
{
  cudaError_t e = cudaSuccess;
  auto dev = [&e](auto *&p, size_t count) {
    if (e == cudaSuccess)
      e = cudaMalloc(&p, sizeof(*p) * count);
  };
  if (!w.pubKey) {
    const size_t sms = device_sm_count();
    dev(w.pubKey, NB * sms);
    dev(w.pubRows, NB * sms * NB);
    dev(w.pubDiag, NB * NB);
    dev(w.barrierCounter, 1);
    dev(w.panelPerm, 1 + 4 * NB);
    dev(w.dInfo, 1);
  }
  if (maxK > w.maxK) {
    cudaFree(w.dIpiv);
    cudaFree(w.dPerm);
    free(w.hostIpiv);
    free(w.hostPerm);
    w.dIpiv = w.dPerm = w.hostIpiv = w.hostPerm = nullptr;
    dev(w.dIpiv, maxK);
    dev(w.dPerm, maxK);
    w.hostIpiv = (int *)malloc(sizeof(int) * maxK);
    w.hostPerm = (int *)malloc(sizeof(int) * maxK);
    if (e == cudaSuccess && (!w.hostIpiv || !w.hostPerm))
      e = cudaErrorMemoryAllocation;
    w.maxK = maxK;
  }
  if (swapK > w.swapK) {
    cudaFree(w.swapTmp);
    w.swapTmp = nullptr;
    dev(w.swapTmp, (size_t)2 * NB * swapK);
    w.swapK = swapK;
  }
  if (e != cudaSuccess)
    lu_workspace_release(w);
  return e;
}

void lu_workspace_release(LuWorkspace &w)
{
  for (void *p : {(void *)w.dIpiv, (void *)w.dPerm, (void *)w.dInfo, (void *)w.pubKey, (void *)w.pubRows,
                  (void *)w.pubDiag, (void *)w.barrierCounter, (void *)w.panelPerm, (void *)w.swapTmp})
    cudaFree(p);
  free(w.hostIpiv);
  free(w.hostPerm);
  w = LuWorkspace{};
}

static int lu_failed(const char *what, cudaError_t e)
{
  fprintf(stderr, "clp_b200: dense_invert: %s: %s\n", what, cudaGetErrorString(e));
  return -97;
}
#define LU_OK(call, what)                                                                         \
  do {                                                                                            \
    const cudaError_t e__ = (call);                                                               \
    if (e__ != cudaSuccess)                                                                       \
      return lu_failed(what, e__);                                                                \
  } while (0)

/* In: A = k x k matrix, column major, leading dimension ld (device).  Out: X = A^-1 (same
   layout), A is overwritten by its LU factors.  w: scratch reserved for at least k rows.  Returns 0,
   (1 + index of the first column without an acceptable pivot), or a negative code after one line on
   stderr when a CUDA call or the all-gather fails.  When it returns 0 or a column, w.hostPerm holds the
   row permutation composed from the pivots of all k columns.  Synchronizes the stream once (pivot
   vector -> permutation). */
int dense_invert(double *A, double *X, int k, int ld, LuWorkspace &w, double singularTol, cudaStream_t s,
                 int shardW, int shardRank, int (*allGather)(void *, void *, size_t, void *), void *comm,
                 void (*hostOverlap)(void *), void *overlapCtx)
{
  if (k <= 0)
    return 0;
  if (k > w.maxK || k > w.swapK) {
    fprintf(stderr, "clp_b200: dense_invert: scratch reserved for %d / %d rows, nucleus of %d\n", w.maxK,
            w.swapK, k);
    return -97;
  }
  // Whether the card grants the 16-CTA non-portable cluster depends on its GPC layout: tried once per
  // process, and once refused every panel goes to the cooperative kernel.  0 untried, 1 usable, -1 refused.
  static int clusterState = 0;
  const int numSMs = device_sm_count();
  const int maxSmem = kPanelMaxRowsPerCta * kSlabPitch * (int)sizeof(double);
  cudaGetLastError(); // an error recorded before this call is not one of the factorization's
  LU_OK(cudaFuncSetAttribute(lu_panel_coop_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem),
        "shared-memory opt-in of lu_panel_coop_kernel");
  LU_OK(cudaMemsetAsync(w.dInfo, 0, sizeof(int), s), "clearing info");
  LU_OK(cudaMemsetAsync(w.barrierCounter, 0, sizeof(unsigned int), s), "clearing the barrier counter");
  unsigned int barrierBase = 0;
  for (int j0 = 0; j0 < k; j0 += NB) {
    int nb = k - j0 < NB ? k - j0 : NB;
    const int nrows = k - j0;
    bool panelDone = false;
    if (clusterState >= 0 && nrows <= kPanelCluster * kPanelMaxRowsPerCta) {
      // one 16-CTA cluster (non-portable size: opted in once)
      const int Rc = (nrows + kPanelCluster - 1) / kPanelCluster;
      const size_t smem = (size_t)Rc * kSlabPitch * sizeof(double);
      if (clusterState == 0) {
        clusterState = 1;
        if (cudaFuncSetAttribute(lu_panel_cluster_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
            cudaFuncSetAttribute(lu_panel_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem) != cudaSuccess) {
          cudaGetLastError();
          clusterState = -1;
        }
      }
      if (clusterState > 0) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(kPanelCluster);
        cfg.blockDim = dim3(256);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = s;
        cudaLaunchAttribute attr;
        attr.id = cudaLaunchAttributeClusterDimension;
        attr.val.clusterDim.x = kPanelCluster;
        attr.val.clusterDim.y = 1;
        attr.val.clusterDim.z = 1;
        cfg.attrs = &attr;
        cfg.numAttrs = 1;
        if (cudaLaunchKernelEx(&cfg, lu_panel_cluster_kernel, A, k, ld, j0, nb, Rc, w.dIpiv, w.dInfo,
                               singularTol) == cudaSuccess) {
          panelDone = true;
        } else {
          cudaGetLastError();
          clusterState = -1;
        }
      }
    }
    if (!panelDone) {
      int G = (nrows + kPanelMinRowsPerCta - 1) / kPanelMinRowsPerCta;
      if (G > numSMs)
        G = numSMs;
      int R = (nrows + G - 1) / G;
      if (R > kPanelMaxRowsPerCta) {
        // 640 x SMs rows: the nucleus would need 16 k^2 >= 85 GB for Ninv and NinvT, more than any H100 has
        fprintf(stderr, "clp_b200: dense_invert: a panel of %d rows exceeds the %d x %d rows lu_panel_coop_kernel holds\n",
                nrows, kPanelMaxRowsPerCta, numSMs);
        return -97;
      }
      void *args[] = {&A,         &k,         &ld,        &j0,       &nb,
                      &R,         &w.dIpiv,   &w.dInfo,   &singularTol,
                      &w.pubKey,  &w.pubRows, &w.pubDiag, &w.barrierCounter, &barrierBase};
      LU_OK(cudaLaunchCooperativeKernel((void *)lu_panel_coop_kernel, dim3(G), dim3(256), args,
                                        (size_t)R * kSlabPitch * sizeof(double), s),
            "cooperative launch of lu_panel_coop_kernel");
      barrierBase += (unsigned int)nb * (unsigned int)G;
    }
    // interchanges on the columns left and right of the panel
    int c0 = j0 + nb;
    {
      const int ncols = j0 + (k - c0);
      if (ncols > 0) {
        lu_perm_kernel<<<1, 1, 0, s>>>(w.dIpiv, j0, nb, w.panelPerm);
        dim3 grid((ncols + 127) / 128, 2 * NB);
        lu_swap_gather_kernel<<<grid, 128, 0, s>>>(A, ld, w.panelPerm, j0, c0, ncols, w.swapTmp);
        lu_swap_scatter_kernel<<<grid, 128, 0, s>>>(A, ld, w.panelPerm, j0, c0, ncols, w.swapTmp);
      }
    }
    if (c0 < k) {
      trsm_kernel<<<(k - c0 + 127) / 128, 128, 0, s>>>(A, ld, A, ld, j0, nb, c0, k, true);
      gemm_sub(A + (size_t)c0 * ld + c0, ld, A + (size_t)j0 * ld + c0, ld,
               A + (size_t)c0 * ld + j0, ld, k - c0, k - c0, nb, s);
    }
  }
  LU_OK(cudaGetLastError(), "LU launches");
  int info = 0;
  LU_OK(cudaMemcpyAsync(w.hostIpiv, w.dIpiv, sizeof(int) * k, cudaMemcpyDeviceToHost, s), "copying the pivots");
  LU_OK(cudaMemcpyAsync(&info, w.dInfo, sizeof(int), cudaMemcpyDeviceToHost, s), "copying info");
  if (hostOverlap)
    hostOverlap(overlapCtx); // host work of the caller (S1 of the new basis) while the LU runs
  LU_OK(cudaStreamSynchronize(s), "LU");
  // Also for a singular nucleus: the interchange of a column without a pivot is the identity and later
  // ones never touch its position, so hostPerm[info - 1] is the row the first info - 1 pivots parked there.
  for (int i = 0; i < k; i++)
    w.hostPerm[i] = i;
  for (int j = 0; j < k; j++) {
    int p = w.hostIpiv[j];
    if (p != j) {
      int t = w.hostPerm[j];
      w.hostPerm[j] = w.hostPerm[p];
      w.hostPerm[p] = t;
    }
  }
  if (info != 0)
    return info;
  LU_OK(cudaMemcpyAsync(w.dPerm, w.hostPerm, sizeof(int) * k, cudaMemcpyHostToDevice, s), "copying the permutation");
  {
    size_t total = (size_t)ld * k;
    set_permuted_identity_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(X, k, ld, w.dPerm);
  }
  // Two-level blocking: triangular solves with the NB x NB diagonal blocks, rank-NB updates only
  // inside an outer block of OB columns, one rank-OB update per outer block for the rest (the bulk
  // of the 2k^3 flops then runs with K = OB, where the DGEMM is not bound by the C traffic).
  constexpr int OB = 128;
  // Multi-GPU: the columns of X are independent in both substitutions, so rank r computes the block
  // [xc0, xc1) only (2k^3/W of the 2k^3 flops of this phase) and ONE in-place all-gather of
  // perC*ld doubles per rank completes X on every rank; the LU above (2/3 k^3) stays replicated.
  int xc0 = 0, xc1 = k, perC = k;
  if (shardW > 1 && allGather != nullptr) {
    perC = (k + shardW - 1) / shardW;
    xc0 = shardRank * perC < k ? shardRank * perC : k;
    xc1 = xc0 + perC < k ? xc0 + perC : k;
  }
  double *const Xr = X + (size_t)xc0 * ld; // this rank's columns, all k rows of them
  const int ncol = xc1 - xc0;
  // forward: Xr := L^-1 Xr
  for (int J0 = 0; J0 < k; J0 += OB) {
    const int J1 = J0 + OB < k ? J0 + OB : k;
    for (int j0 = J0; j0 < J1; j0 += NB) {
      int nb = J1 - j0 < NB ? J1 - j0 : NB;
      if (ncol > 0)
        trsm_kernel<<<(ncol + 127) / 128, 128, 0, s>>>(A, ld, Xr, ld, j0, nb, 0, ncol, true);
      int r0 = j0 + nb;
      if (r0 < J1)
        gemm_sub(Xr + r0, ld, A + (size_t)j0 * ld + r0, ld, Xr + j0, ld, J1 - r0, ncol, nb, s);
    }
    if (J1 < k)
      gemm_sub(Xr + J1, ld, A + (size_t)J0 * ld + J1, ld, Xr + J0, ld, k - J1, ncol, J1 - J0, s);
  }
  // backward: Xr := U^-1 Xr
  const int lastOuter = ((k - 1) / OB) * OB;
  for (int J0 = lastOuter; J0 >= 0; J0 -= OB) {
    const int J1 = J0 + OB < k ? J0 + OB : k;
    const int lastInner = J0 + ((J1 - J0 - 1) / NB) * NB;
    for (int j0 = lastInner; j0 >= J0; j0 -= NB) {
      int nb = J1 - j0 < NB ? J1 - j0 : NB;
      if (ncol > 0)
        trsm_kernel<<<(ncol + 127) / 128, 128, 0, s>>>(A, ld, Xr, ld, j0, nb, 0, ncol, false);
      if (j0 > J0)
        gemm_sub(Xr + J0, ld, A + (size_t)j0 * ld + J0, ld, Xr + j0, ld, j0 - J0, ncol, nb, s);
    }
    if (J0 > 0)
      gemm_sub(Xr, ld, A + (size_t)J0 * ld, ld, Xr + J0, ld, J0, ncol, J1 - J0, s);
  }
  LU_OK(cudaGetLastError(), "substitution launches");
  if (shardW > 1 && allGather != nullptr) {
    if (allGather(comm, X, sizeof(double) * (size_t)perC * ld, s) != 0)
      return -98;
  }
  zero_padding_kernel<<<(k + 255) / 256, 256, 0, s>>>(X, k, ld);
  LU_OK(cudaGetLastError(), "zero_padding_kernel launch");
  return 0;
}

} // namespace clpb
