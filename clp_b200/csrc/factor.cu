// factor.cu -- dense refactorization of the basis nucleus on the GPU.
//
// Replaces the numerical part of ClpFactorization::factorize
// (/root/reference/src/ClpFactorization.cpp:1649 -> CoinAbcTypeFactorization::factor
// src/CoinAbcBaseFactorization1.cpp:683; the dense tail factorDense ...2.cpp:976 ->
// CoinAbcDgetrf src/AbcSimplexParallel.cpp:2491 with its CoinAbcDgemm trailing update).
//
// The k x k nucleus (structural basic columns restricted to rows whose slack is nonbasic) is
// LU-factorized with partial pivoting by a blocked right-looking algorithm (panel kernel +
// fused row interchanges and unit-lower TRSM + rank-NB DGEMM update) and the factors are then turned
// into the explicit inverse X = U^-1 L^-1 P by blocked forward/backward substitution of the identity
// (TRSM + DGEMM) and a permuted transpose.
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

// The nb interchanges (j0 + jj <-> piv[jj]) of a panel composed into one row permutation, by one warp
// at the end of the panel kernel.  perm[1 + l] is the row whose content ends in panel row j0 + l; the
// rows below the panel that some interchange touched are perm[1 + NB + t], t < perm[0], and their
// content comes from panel row perm[1 + 2*NB + t] (a pivot row only ever receives the current content
// of a panel row, and panel rows only ever hold original panel rows or pivot rows).
__device__ __forceinline__ void compose_panel_perm(const int *__restrict__ piv, int j0, int nb,
                                                   int *__restrict__ perm)
{
  const int lane = threadIdx.x & 31;
  int cur = j0 + lane, outRow = -1, outSrc = j0, nOut = 0;
  for (int jj = 0; jj < nb; jj++) {
    const int p = piv[jj];
    if (p == j0 + jj)
      continue;
    const int a = __shfl_sync(0xffffffffu, cur, jj);
    if (p - j0 < nb) {
      const int b = __shfl_sync(0xffffffffu, cur, p - j0);
      if (lane == jj)
        cur = b;
      if (lane == p - j0)
        cur = a;
    } else {
      const unsigned int hit = __ballot_sync(0xffffffffu, outRow == p);
      const int t = hit ? __ffs(hit) - 1 : nOut++;
      const int b = hit ? __shfl_sync(0xffffffffu, outSrc, t) : p;
      if (lane == jj)
        cur = b;
      if (lane == t) {
        outRow = p;
        outSrc = a;
      }
    }
  }
  if (lane < nb)
    perm[1 + lane] = cur;
  if (lane < nOut) {
    perm[1 + NB + lane] = outRow;
    perm[1 + 2 * NB + lane] = outSrc;
  }
  if (lane == 0)
    perm[0] = nOut;
}

// rows [j0 + cta*R, j0 + (cta+1)*R) of the panel belong to CTA 'cta'
__global__ void __launch_bounds__(256)
    lu_panel_coop_kernel(double *__restrict__ A, int k, int ld, int j0, int nb, int R,
                         int *__restrict__ panelPerm, int *__restrict__ info, double singularTol,
                         unsigned long long *__restrict__ pubKey, double *__restrict__ pubRows,
                         double *__restrict__ pubDiag, unsigned int *__restrict__ barrierCounter,
                         unsigned int barrierBase)
{
  extern __shared__ double slab[]; // [R][kSlabPitch]
  __shared__ unsigned long long sBest[8];
  __shared__ int sWinCta[8];
  __shared__ int sPiv[NB];
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
    if (tid == 0)
      sPiv[jj] = singular ? j : piv;
    if (cta == 0 && tid == 0 && singular && *info == 0)
      *info = j + 1;
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
  if (cta == 0 && warp == 0)
    compose_panel_perm(sPiv, j0, nb, panelPerm);
}

// ---- the same panel on ONE thread-block cluster (16 CTAs of one GPC, distributed shared memory).
// The per-column pivot exchange of lu_panel_coop_kernel costs a grid barrier plus two dependent L2 round
// trips; inside a cluster it costs ONE hardware cluster barrier per column.  Before it every CTA copies
// its candidate key and row (and the owner of the diagonal row that row) into a publication slot in its
// own shared memory; after it every CTA reads the winner's row and the diagonal row out of the peers'
// slots and swaps and eliminates locally.  The slots are double-buffered by column parity: slot jj & 1
// is rewritten at column jj + 2, after every peer has passed the barrier of column jj + 1 and so has
// finished reading it.  Panels of up to 16 x kPanelMaxRowsPerCta rows.
constexpr int kPanelCluster = 16;

__global__ void __launch_bounds__(256)
    lu_panel_cluster_kernel(double *__restrict__ A, int k, int ld, int j0, int nb, int R,
                            int *__restrict__ panelPerm, int *__restrict__ info, double singularTol)
{
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ double slab[]; // [R][kSlabPitch]
  __shared__ unsigned long long sBest[8];
  __shared__ unsigned long long sWin;
  __shared__ int sPiv[NB];
  __shared__ double urow[NB], drow[NB];
  __shared__ unsigned long long slotKey[2];      // publication slots, same offset in every CTA
  __shared__ double slotRow[2][NB], slotDiag[2][NB];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cta = (int)cluster.block_rank();
  const int r0 = j0 + cta * R;
  const int rowsLocal = max(0, min(R, k - r0));
  for (int c = 0; c < nb; c++)
    for (int q = tid; q < rowsLocal; q += 256)
      slab[q * kSlabPitch + c] = A[(size_t)(j0 + c) * ld + r0 + q];
  __syncthreads();
  for (int jj = 0; jj < nb; jj++) {
    const int j = j0 + jj, par = jj & 1;
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
    __syncthreads(); // also: the elimination of the previous column is complete
    unsigned long long cand = 0ull;
#pragma unroll
    for (int w = 0; w < 8; w++)
      cand = max(cand, sBest[w]);
    if (tid == 0)
      slotKey[par] = cand;
    if (cand != 0ull && tid < NB)
      slotRow[par][tid] = slab[(j0 + (0xFFFFF - (int)(cand & 0xFFFFFull)) - r0) * kSlabPitch + tid];
    if (ownerJ == cta && tid < NB)
      slotDiag[par][tid] = slab[(j - r0) * kSlabPitch + tid];
    cluster.sync(); // every CTA's slot of this column is published
    if (warp == 0) {
      unsigned long long v = 0ull;
      if (lane < kPanelCluster)
        v = *cluster.map_shared_rank(&slotKey[par], lane);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
      if (lane == 0)
        sWin = v;
      if (v != 0ull) { // pivot row out of the winner's slot, diagonal row out of its owner's
        const int ownerP = (0xFFFFF - (int)(v & 0xFFFFFull)) / R;
        urow[lane] = *cluster.map_shared_rank(&slotRow[par][lane], ownerP);
        drow[lane] = *cluster.map_shared_rank(&slotDiag[par][lane], ownerJ);
      }
    }
    __syncthreads();
    const unsigned long long wkey = sWin;
    const double pivAbs = __longlong_as_double((long long)(wkey & ~0xFFFFFull));
    const int piv = j0 + (0xFFFFF - (int)(wkey & 0xFFFFFull));
    const bool singular = (wkey == 0ull) || !(pivAbs >= singularTol);
    if (tid == 0)
      sPiv[jj] = singular ? j : piv;
    if (cta == 0 && tid == 0 && singular && *info == 0)
      *info = j + 1;
    if (singular)
      continue; // one barrier per column on both paths: the count stays uniform across the cluster
    const int ownerP = (piv - j0) / R;
    if (tid < NB) { // exchange: the old diagonal row moves to row piv, the pivot row moves to row j
      if (piv != j && ownerP == cta)
        slab[(piv - r0) * kSlabPitch + tid] = drow[tid];
      if (ownerJ == cta)
        slab[(j - r0) * kSlabPitch + tid] = urow[tid];
    }
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
  }
  cluster.sync(); // nobody exits while a peer may still read its shared memory
  for (int c = 0; c < nb; c++)
    for (int q = tid; q < rowsLocal; q += 256)
      A[(size_t)(j0 + c) * ld + r0 + q] = slab[q * kSlabPitch + c];
  if (cta == 0 && warp == 0)
    compose_panel_perm(sPiv, j0, nb, panelPerm);
}

// The panel's composed row permutation (compose_panel_perm) applied to one column of the rows outside
// the panel's own columns; the warp holds the <= 2*NB touched rows in registers.  Returns the new value
// of panel row j0 + lane (lane < nb); the touched rows below the panel are written here.
template <typename T>
__device__ __forceinline__ T interchange_column(T *__restrict__ col, int j0, int nb, int src, int nOut, int outRow,
                                                int outSrc)
{
  const int lane = threadIdx.x & 31;
  const T orig = lane < nb ? col[j0 + lane] : T(0);
  const bool inPanel = src - j0 < nb;
  const T fromPanel = __shfl_sync(0xffffffffu, orig, inPanel ? src - j0 : 0);
  const T x = inPanel ? fromPanel : col[src];
  const T toOut = __shfl_sync(0xffffffffu, orig, outSrc - j0);
  __syncwarp(); // every load of the column is done before a touched row is overwritten
  if (lane < nOut)
    col[outRow] = toOut;
  return x;
}

// Row interchanges of a panel on the columns left and right of it, and the unit-lower solve with the
// panel's L11 on the columns right of it, one warp per column; warp ncols applies the interchanges to
// the row permutation rowPerm of the whole factorization.  Columns are indexed linearly over
// [0, j0) U [j0 + nb, k).  Lane i holds row i of L11 and sweeps l ascending, which is trsm_kernel's
// s = fma(-T[i][l], x[l], s) order.
__global__ void __launch_bounds__(256)
    lu_interchange_trsm_kernel(double *__restrict__ A, int k, int ld, int j0, int nb,
                               const int *__restrict__ perm, int *__restrict__ rowPerm)
{
  __shared__ double L11[NB][NB + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = j0 + nb, ncols = j0 + (k - c0);
  for (int e = threadIdx.x; e < NB * NB; e += blockDim.x) {
    const int i = e % NB, l = e / NB;
    L11[i][l] = (i < nb && l < nb) ? A[(size_t)(j0 + l) * ld + j0 + i] : 0.0;
  }
  const int nOut = perm[0];
  const int src = lane < nb ? perm[1 + lane] : j0;
  const int outRow = lane < nOut ? perm[1 + NB + lane] : 0;
  const int outSrc = lane < nOut ? perm[1 + 2 * NB + lane] : j0;
  __syncthreads();
  double t[NB];
#pragma unroll
  for (int l = 0; l < NB; l++)
    t[l] = L11[lane][l];
  for (int q = blockIdx.x * 8 + warp; q <= ncols; q += gridDim.x * 8) {
    if (q == ncols) {
      const int v = interchange_column(rowPerm, j0, nb, src, nOut, outRow, outSrc);
      if (lane < nb)
        rowPerm[j0 + lane] = v;
      continue;
    }
    const int c = q < j0 ? q : q - j0 + c0;
    double *col = A + (size_t)c * ld;
    double x = interchange_column(col, j0, nb, src, nOut, outRow, outSrc);
    if (c >= c0) {
#pragma unroll
      for (int l = 0; l < NB - 1; l++) {
        const double xl = __shfl_sync(0xffffffffu, x, l);
        if (lane > l)
          x = fma(-t[l], xl, x);
      }
    }
    if (lane < nb)
      col[j0 + lane] = x;
  }
}

__global__ void iota_kernel(int *__restrict__ v, int k)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k)
    v[i] = i;
}

// B[j0..j0+nb, c] := T^-1 B[.., c] for columns c in [c0,c1); T = nb x nb triangle of A at (j0,j0)
//   lower=true : unit lower triangular (forward substitution)
//   lower=false: upper triangular with diagonal (backward substitution)
//   BS threads per CTA; the triangle is loaded with all of a thread's loads in flight at once
template <int BS>
__global__ void __launch_bounds__(BS)
    trsm_kernel(const double *__restrict__ A, int lda, double *__restrict__ B, int ldb, int j0,
                int nb, int c0, int c1, bool lower)
{
  __shared__ double T[NB][NB + 1];
  double t[NB * NB / BS];
#pragma unroll
  for (int u = 0; u < NB * NB / BS; u++) {
    const int e = threadIdx.x + u * BS, i = e % NB, l = e / NB;
    t[u] = (i < nb && l < nb) ? A[(size_t)(j0 + l) * lda + j0 + i] : (i == l ? 1.0 : 0.0);
  }
#pragma unroll
  for (int u = 0; u < NB * NB / BS; u++) {
    const int e = threadIdx.x + u * BS;
    T[e % NB][e / NB] = t[u];
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

// cuBLAS from M x Nsel >= 256^2 on: the forward substitution passes its full column count, so the choice
// (and with it the rounding) of an element does not depend on how many columns a step updates
static void gemm_sub(double *C, int ldc, const double *A, int lda, const double *B, int ldb, int M,
                     int N, int K, cudaStream_t s, int Nsel = 0)
{
  if (M <= 0 || N <= 0 || K <= 0)
    return;
  if ((long)M * (Nsel > 0 ? Nsel : N) >= 256L * 256L && blas_ready()) {
    const double minusOne = -1.0, one = 1.0;
    p_setStream(g_blas, s);
    if (p_dgemm(g_blas, 0 /* N */, 0 /* N */, M, N, K, &minusOne, A, lda, B, ldb, &one, C, ldc) == 0)
      return;
  }
  dim3 grid((M + 63) / 64, (N + 63) / 64);
  gemm_sub_kernel<<<grid, 256, 0, s>>>(C, ldc, A, lda, B, ldb, M, N, K);
}

__global__ void set_identity_kernel(double *__restrict__ X, int k, int ld)
{
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)ld * k;
  if (idx >= total)
    return;
  X[idx] = (idx % ld == idx / ld) ? 1.0 : 0.0;
}

__global__ void invert_perm_kernel(const int *__restrict__ perm, int *__restrict__ inv, int k)
{
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k)
    inv[perm[i]] = i;
}

// dst = src^T with its rows [k, ld) zero; with colMap, column y of src is read from column colMap[y]
__global__ void transpose_kernel(const double *__restrict__ src, double *__restrict__ dst, int k,
                                 int ld, const int *__restrict__ colMap)
{
  __shared__ double tile[32][33];
  int x = blockIdx.x * 32 + threadIdx.x, y0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    int y = y0 + r;
    tile[r][threadIdx.x] = (x < k && y < k) ? src[(size_t)(colMap ? colMap[y] : y) * ld + x] : 0.0;
  }
  __syncthreads();
  int xo = blockIdx.y * 32 + threadIdx.x, yo0 = blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    int yo = yo0 + r;
    if (xo < ld && yo < k)
      dst[(size_t)yo * ld + xo] = (xo < k) ? tile[threadIdx.x][r] : 0.0;
  }
}
static void launch_transpose(const double *src, double *dst, int k, int ld, const int *colMap, cudaStream_t s)
{
  dim3 grid((ld + 31) / 32, (k + 31) / 32);
  transpose_kernel<<<grid, dim3(32, 8), 0, s>>>(src, dst, k, ld, colMap);
}

cudaError_t lu_workspace_reserve(LuWorkspace &w, int maxK)
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
    dev(w.panelPerm, 1 + 3 * NB);
    dev(w.dInfo, 1);
  }
  if (maxK > w.maxK) {
    cudaFree(w.dPerm);
    cudaFree(w.dInvPerm);
    free(w.hostPerm);
    w.dPerm = w.dInvPerm = w.hostPerm = nullptr;
    dev(w.dPerm, maxK);
    dev(w.dInvPerm, maxK);
    w.hostPerm = (int *)malloc(sizeof(int) * maxK);
    if (e == cudaSuccess && !w.hostPerm)
      e = cudaErrorMemoryAllocation;
    w.maxK = maxK;
  }
  if (e != cudaSuccess)
    lu_workspace_release(w);
  return e;
}

void lu_workspace_release(LuWorkspace &w)
{
  for (void *p : {(void *)w.dPerm, (void *)w.dInvPerm, (void *)w.dInfo, (void *)w.pubKey, (void *)w.pubRows,
                  (void *)w.pubDiag, (void *)w.barrierCounter, (void *)w.panelPerm})
    cudaFree(p);
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

/* In: A = k x k matrix, column major, leading dimension ld (device).  Out: X = A^-1 and A = X^T (same
   layout, rows [k, ld) of both zero).  w: scratch reserved for at least k rows.  Returns 0, (1 + index of
   the first column without an acceptable pivot), or a negative code after one line on stderr when a CUDA
   call or the all-gather fails.  When it returns 0 or a column, w.hostPerm holds the row permutation
   composed from the pivots of all k columns; after a column, A and X hold garbage.  The LU, the
   substitutions and the transposes are enqueued without a host round trip; hostOverlap runs while they
   execute, and the stream is synchronized once, at the end. */
int dense_invert(double *A, double *X, int k, int ld, LuWorkspace &w, double singularTol, cudaStream_t s,
                 int shardW, int shardRank, int (*allGather)(void *, void *, size_t, void *), void *comm,
                 void (*hostOverlap)(void *), void *overlapCtx)
{
  if (k <= 0)
    return 0;
  if (k > w.maxK) {
    fprintf(stderr, "clp_b200: dense_invert: scratch reserved for %d rows, nucleus of %d\n", w.maxK, k);
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
  iota_kernel<<<(k + 255) / 256, 256, 0, s>>>(w.dPerm, k);
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
        if (cudaLaunchKernelEx(&cfg, lu_panel_cluster_kernel, A, k, ld, j0, nb, Rc, w.panelPerm, w.dInfo,
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
      void *args[] = {&A,         &k,           &ld,        &j0,       &nb,
                      &R,         &w.panelPerm, &w.dInfo,   &singularTol,
                      &w.pubKey,  &w.pubRows,   &w.pubDiag, &w.barrierCounter, &barrierBase};
      LU_OK(cudaLaunchCooperativeKernel((void *)lu_panel_coop_kernel, dim3(G), dim3(256), args,
                                        (size_t)R * kSlabPitch * sizeof(double), s),
            "cooperative launch of lu_panel_coop_kernel");
      barrierBase += (unsigned int)nb * (unsigned int)G;
    }
    // interchanges on the columns left and right of the panel (and on dPerm), L11^-1 on the right ones
    const int c0 = j0 + nb;
    {
      const int warps = j0 + (k - c0) + 1;
      int blocks = (warps + 7) / 8;
      if (blocks > 4 * numSMs)
        blocks = 4 * numSMs;
      lu_interchange_trsm_kernel<<<blocks, 256, 0, s>>>(A, k, ld, j0, nb, w.panelPerm, w.dPerm);
    }
    if (c0 < k)
      gemm_sub(A + (size_t)c0 * ld + c0, ld, A + (size_t)j0 * ld + c0, ld,
               A + (size_t)c0 * ld + j0, ld, k - c0, k - c0, nb, s);
  }
  LU_OK(cudaGetLastError(), "LU launches");
  // A^-1 = U^-1 L^-1 P.  Y = U^-1 L^-1 I is computed in X, and X[:, perm[i]] = Y[:, i] is applied by the
  // transposes at the end.  Column i of L^-1 I is zero above row i, so the forward substitution's outer
  // step [J0, J1) works on columns < J1 only: k^3 / 3 flops instead of k^3.  Every computed element sees
  // the operations it saw with all k columns (the skipped ones are exact zeros), and the cuBLAS-or-kernel
  // choice of each DGEMM is made from the full column count.
  set_identity_kernel<<<(unsigned)(((size_t)ld * k + 255) / 256), 256, 0, s>>>(X, k, ld);
  // Two-level blocking: triangular solves with the NB x NB diagonal blocks, rank-NB updates only
  // inside an outer block of OB columns, one rank-OB update per outer block for the rest (the bulk
  // of the flops then runs with K = OB, where the DGEMM is not bound by the C traffic).
  constexpr int OB = 128;
  // Multi-GPU: the columns of Y are independent in both substitutions, so rank r computes the block
  // [xc0, xc1) only and ONE in-place all-gather of perC*ld doubles per rank completes Y on every rank;
  // the LU above (2/3 k^3) stays replicated.  The forward work of a rank grows with its column index.
  int xc0 = 0, xc1 = k, perC = k;
  if (shardW > 1 && allGather != nullptr) {
    perC = (k + shardW - 1) / shardW;
    xc0 = shardRank * perC < k ? shardRank * perC : k;
    xc1 = xc0 + perC < k ? xc0 + perC : k;
  }
  double *const Xr = X + (size_t)xc0 * ld; // this rank's columns, all k rows of them
  const int ncol = xc1 - xc0;
  // one thread per column, 32 per CTA: the k columns spread over all SMs
  auto trsm = [&](int j0, int nb, int n, bool lower) {
    if (n > 0)
      trsm_kernel<32><<<(n + 31) / 32, 32, 0, s>>>(A, ld, Xr, ld, j0, nb, 0, n, lower);
  };
  // forward: Y := L^-1 Y on columns [xc0, min(xc1, J1))
  for (int J0 = 0; J0 < k; J0 += OB) {
    const int J1 = J0 + OB < k ? J0 + OB : k;
    const int nf = (xc1 < J1 ? xc1 : J1) - xc0;
    if (nf <= 0)
      continue;
    for (int j0 = J0; j0 < J1; j0 += NB) {
      int nb = J1 - j0 < NB ? J1 - j0 : NB;
      trsm(j0, nb, nf, true);
      int r0 = j0 + nb;
      if (r0 < J1)
        gemm_sub(Xr + r0, ld, A + (size_t)j0 * ld + r0, ld, Xr + j0, ld, J1 - r0, nf, nb, s, ncol);
    }
    if (J1 < k)
      gemm_sub(Xr + J1, ld, A + (size_t)J0 * ld + J1, ld, Xr + J0, ld, k - J1, nf, J1 - J0, s, ncol);
  }
  // backward: Y := U^-1 Y
  const int lastOuter = ((k - 1) / OB) * OB;
  for (int J0 = lastOuter; J0 >= 0; J0 -= OB) {
    const int J1 = J0 + OB < k ? J0 + OB : k;
    const int lastInner = J0 + ((J1 - J0 - 1) / NB) * NB;
    for (int j0 = lastInner; j0 >= J0; j0 -= NB) {
      int nb = J1 - j0 < NB ? J1 - j0 : NB;
      trsm(j0, nb, ncol, false);
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
  // A := X^T (the LU factors are dead): row perm[i] of A is column i of Y, read from column invPerm[r]
  // for row r; then X := A^T
  invert_perm_kernel<<<(k + 255) / 256, 256, 0, s>>>(w.dPerm, w.dInvPerm, k);
  launch_transpose(X, A, k, ld, w.dInvPerm, s);
  launch_transpose(A, X, k, ld, nullptr, s);
  LU_OK(cudaGetLastError(), "transpose launches");
  if (hostOverlap)
    hostOverlap(overlapCtx); // host work of the caller (S1 of the new basis) while the GPU works
  // pageable destinations: these copies wait for the stream, so they come after all launches
  LU_OK(cudaMemcpyAsync(w.hostPerm, w.dPerm, sizeof(int) * k, cudaMemcpyDeviceToHost, s), "copying the permutation");
  int info = 0;
  LU_OK(cudaMemcpyAsync(&info, w.dInfo, sizeof(int), cudaMemcpyDeviceToHost, s), "copying info");
  LU_OK(cudaStreamSynchronize(s), "dense_invert");
  return info;
}

} // namespace clpb
