// solve.cu -- FTRAN / BTRAN through the basis factors (device resident).
//
// Replaces ClpFactorization::updateColumn / updateColumnFT / updateTwoColumnsFT
// (/root/reference/src/ClpFactorization.cpp:2803,2723,2889 -> CoinAbcBaseFactorization3.cpp
// updateColumnL/R/U) and ClpFactorization::updateColumnTranspose (ClpFactorization.cpp:2993 ->
// CoinAbcBaseFactorization4.cpp:3216).  See engine.cuh for the factor layout.
//
//   FTRAN  x = B_t^-1 b :   yN = Ninv * b_N                      (GEMV, HBM stream of Ninv)
//                           x_N = yN ; x_C = S1*yN - b_C          (CSR SpMV)
//                           mu = Ginv * x[P] ; x -= W * mu        (eta panel GEMV)
//   BTRAN  rho = B_t^-T e_r: nu = Ginv^T * W[r,:] ; u = e_r - sum_j e_{p_j} nu_j
//                           rho_C = -u_C ; s = u_N + S1^T u_C
//                           rho_N = Ninv^T * s                    (GEMV, HBM stream of NinvT)
// Up to three right-hand sides share one pass over Ninv / W (the reference's
// updateTwoColumnsFT fusion, plus the bound-flip column of ClpSimplexDual.cpp:1533).
#include "kernels_common.cuh"

#include <stdexcept>

namespace clpb {

static inline int roundUp8(int v) { return (v + 7) / 8 * 8; }

ShardCtx g_shardCtx;
// launch-shape experiments (tests/ab_probe.py): rows per CTA pass / 16-byte loads in flight / CTAs per SM
int g_gemvVariantF = 0, g_gemvVariantB = 0, g_gemvGridMul = 8;
int g_pfiApplyVariant = 0; // 0: warp per panel row, 1: GEMV-shaped (two rows per CTA); "pfiApplyVariant"

// ---------------------------------------------------------------------------------------
// gather b_N : xg[c][j] = b_c[nucRow[j]]
__global__ void gather_nucleus_kernel(DeviceModel d, const double *__restrict__ b, int bstride,
                                      double *__restrict__ xg, int nrhs, bool checkState)
{
  if (checkState && !iter_active(d.st))
    return;
  const int k = d.fd->k, ldk = d.fd->ldk;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < ldk; j += gridDim.x * blockDim.x) {
    if (j >= k) { // zero padding so the GEMV can run over the padded row length
      for (int c = 0; c < nrhs; c++)
        xg[(size_t)c * ldk + j] = 0.0;
    } else {
      int p = d.nucRow[j];
      for (int c = 0; c < nrhs; c++)
        xg[(size_t)c * ldk + j] = b[(size_t)c * bstride + p];
    }
  }
}

// y[c][i] = sum_j M[i][j] * x[c][j]   (M row-major k x ldk).  One CTA streams R consecutive rows with
// DEPTH 16-byte loads per row in flight per thread, i.e. R*DEPTH*4 KB contiguous per row and step:
// few, long DRAM streams (tests/microbench/iter_kernels.cu compares the shapes: one right-hand side
// R=1 DEPTH=8, three right-hand sides R=2 DEPTH=2 -- x goes through L1, so more rows per CTA pay
// once there are three of them).  outIndex != nullptr: the result is scattered,
// out[c*ostride + outIndex[i]].
template <int NRHS, int R, int DEPTH>
__global__ void __launch_bounds__(256)
    gemv_rows_kernel(const FactorDesc *__restrict__ fd, int transposed,
                     const double *__restrict__ x, double *__restrict__ out, int ostride,
                     const int *__restrict__ outIndex, const IterState *st, bool checkState,
                     int shardW, int shardRank, int shardPer)
{
  if (checkState && !iter_active(st))
    return;
  __shared__ double part[8][R * NRHS];
  const int k = fd->k, ldk = fd->ldk;
  // row-sharded run: this rank streams rows [rowBegin, rowEnd) and writes them to its chunk of the
  // gather buffer out[rank][c][shardPer] (completed by one in-place all-gather)
  int rowBegin = 0, rowEnd = k;
  if (shardW > 1) {
    const int perK = ((k + shardW - 1) / shardW + 7) & ~7;
    rowBegin = min(k, shardRank * perK);
    rowEnd = min(k, rowBegin + perK);
  }
  const double *__restrict__ M = transposed ? fd->NinvT : fd->Ninv;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int half = ldk >> 1; // ldk is a multiple of 8, padding is zero
  const int ngroups = (rowEnd - rowBegin + R - 1) / R;
  for (int g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int i0 = rowBegin + g * R;
    const double2 *row[R];
#pragma unroll
    for (int r = 0; r < R; r++) // rows beyond k alias the last row (results discarded)
      row[r] = reinterpret_cast<const double2 *>(M + (size_t)min(i0 + r, k - 1) * ldk);
    double acc[R][NRHS];
#pragma unroll
    for (int r = 0; r < R; r++)
#pragma unroll
      for (int c = 0; c < NRHS; c++)
        acc[r][c] = 0.0;
    for (int j = threadIdx.x; j < half; j += 256 * DEPTH) {
      double2 a[DEPTH][R];
#pragma unroll
      for (int u = 0; u < DEPTH; u++) {
        const bool p = j + 256 * u < half;
#pragma unroll
        for (int r = 0; r < R; r++)
          a[u][r] = p ? __ldcs(row[r] + j + 256 * u) : make_double2(0.0, 0.0);
      }
#pragma unroll
      for (int u = 0; u < DEPTH; u++) {
        const int jj = min(j + 256 * u, half - 1);
#pragma unroll
        for (int c = 0; c < NRHS; c++) {
          const double2 xv = __ldg(reinterpret_cast<const double2 *>(x + (size_t)c * ldk) + jj);
#pragma unroll
          for (int r = 0; r < R; r++) {
            acc[r][c] = fma(a[u][r].x, xv.x, acc[r][c]);
            acc[r][c] = fma(a[u][r].y, xv.y, acc[r][c]);
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < R; r++)
#pragma unroll
      for (int c = 0; c < NRHS; c++) {
        const double v = warp_sum(acc[r][c]);
        if (lane == 0)
          part[warp][r * NRHS + c] = v;
      }
    __syncthreads();
    if (threadIdx.x < R * NRHS) {
      double sum = 0.0;
#pragma unroll
      for (int w = 0; w < 8; w++)
        sum += part[w][threadIdx.x];
      const int r = threadIdx.x / NRHS, c = threadIdx.x % NRHS;
      if (i0 + r < rowEnd) {
        if (shardW > 1) {
          out[((size_t)shardRank * NRHS + c) * shardPer + (i0 + r - rowBegin)] = sum;
        } else {
          const int o = outIndex ? outIndex[i0 + r] : i0 + r;
          const int os = ostride < 0 ? ldk : ostride;
          out[(size_t)c * os + o] = sum;
        }
      }
    }
    __syncthreads();
  }
}

// Same product with one WARP per row (no block-level reduction, no __syncthreads): lanes stride the row
// in 16-byte pieces, DEPTH loads per lane in flight.  Launch-shape experiment (gemvVariantF = 7 /
// gemvVariantB = 6); not sharded.
template <int NRHS, int DEPTH>
__global__ void __launch_bounds__(256)
    gemv_warp_rows_kernel(const FactorDesc *__restrict__ fd, int transposed, const double *__restrict__ x,
                          double *__restrict__ out, int ostride, const int *__restrict__ outIndex,
                          const IterState *st, bool checkState)
{
  if (checkState && !iter_active(st))
    return;
  const int k = fd->k, ldk = fd->ldk;
  const double *__restrict__ M = transposed ? fd->NinvT : fd->Ninv;
  const int lane = threadIdx.x & 31;
  const int half = ldk >> 1;
  const int warpsTotal = gridDim.x * (blockDim.x >> 5);
  for (int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < k; i += warpsTotal) {
    const double2 *row = reinterpret_cast<const double2 *>(M + (size_t)i * ldk);
    double acc[NRHS];
#pragma unroll
    for (int c = 0; c < NRHS; c++)
      acc[c] = 0.0;
    for (int j = lane; j < half; j += 32 * DEPTH) {
      double2 a[DEPTH];
#pragma unroll
      for (int u = 0; u < DEPTH; u++)
        a[u] = j + 32 * u < half ? __ldcs(row + j + 32 * u) : make_double2(0.0, 0.0);
#pragma unroll
      for (int u = 0; u < DEPTH; u++) {
        const int jj = min(j + 32 * u, half - 1);
#pragma unroll
        for (int c = 0; c < NRHS; c++) {
          const double2 xv = __ldg(reinterpret_cast<const double2 *>(x + (size_t)c * ldk) + jj);
          acc[c] = fma(a[u].x, xv.x, acc[c]);
          acc[c] = fma(a[u].y, xv.y, acc[c]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < NRHS; c++) {
      const double v = warp_sum(acc[c]);
      if (lane == 0) {
        const int o = outIndex ? outIndex[i] : i;
        const int os = ostride < 0 ? ldk : ostride;
        out[(size_t)c * os + o] = v;
      }
    }
  }
}

// entry j of GEMV result c: plain [c][ldk] layout, or the gathered [rank][c][shardPerK] layout
template <int NRHS>
__device__ __forceinline__ double gemv_result(const DeviceModel &d, const double *__restrict__ y, int c, int j,
                                              int ldk, int perK)
{
  if (d.shardW == 1)
    return y[(size_t)c * ldk + j];
  const int rk = j / perK;
  return y[((size_t)rk * NRHS + c) * d.shardPerK + (j - rk * perK)];
}

// x_N = yN ; x_C = S1*yN - b_C   (in place on b, 8 lanes per position).  etaTail: the last CTA
// then gathers the finished columns at the eta positions, xp[c][j] = b_c[etaPos[j]], the compact
// right-hand side of the t x t system G mu = v0[P] (pfi_mu_kernel reads it coalesced).
template <int NRHS>
__global__ void __launch_bounds__(256)
    ftran_spread_kernel(DeviceModel d, double *__restrict__ b, int bstride,
                        const double *__restrict__ y, bool checkState, bool etaTail)
{
  if (checkState && !iter_active(d.st))
    return;
  const int sub = threadIdx.x & 7;
  const int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  if (p < d.m) { // whole 8-lane groups take the same branch
    const unsigned gmask = 0xFFu << ((threadIdx.x & 31) & ~7);
    const int ldk = d.fd->ldk;
    const int perK = d.shardW > 1 ? (((d.fd->k + d.shardW - 1) / d.shardW + 7) & ~7) : 1;
    const int *__restrict__ s1Col = d.fd->s1Col;
    const double *__restrict__ s1Val = d.fd->s1Val;
    const int ni = d.posToNuc[p];
    if (ni >= 0) {
      if (sub == 0)
        for (int c = 0; c < NRHS; c++)
          b[(size_t)c * bstride + p] = gemv_result<NRHS>(d, y, c, ni, ldk, perK);
    } else {
      double acc[NRHS];
#pragma unroll
      for (int c = 0; c < NRHS; c++)
        acc[c] = 0.0;
      if (d.fd->k > 0) {
        int e0 = d.s1RowStart[p], e1 = d.s1RowStart[p + 1];
        for (int e = e0 + sub; e < e1; e += 8) {
          double v = s1Val[e];
          int j = s1Col[e];
#pragma unroll
          for (int c = 0; c < NRHS; c++)
            acc[c] = fma(v, gemv_result<NRHS>(d, y, c, j, ldk, perK), acc[c]);
        }
      }
#pragma unroll
      for (int c = 0; c < NRHS; c++) {
        acc[c] += __shfl_xor_sync(gmask, acc[c], 4);
        acc[c] += __shfl_xor_sync(gmask, acc[c], 2);
        acc[c] += __shfl_xor_sync(gmask, acc[c], 1);
      }
      if (sub == 0)
        for (int c = 0; c < NRHS; c++)
          b[(size_t)c * bstride + p] = acc[c] - b[(size_t)c * bstride + p];
    }
  }
  if (!etaTail)
    return;
  if (!last_block_done(d.tailCounter + TAIL_SPREAD))
    return;
  const int t = d.st->numEtas;
  for (int j0 = threadIdx.x; j0 < t; j0 += 8 * 256) { // eight independent gathers in flight per thread
    int pj[8];
#pragma unroll
    for (int u = 0; u < 8; u++)
      pj[u] = (j0 + 256 * u < t) ? d.etaPos[j0 + 256 * u] : 0;
    double v[8][NRHS];
#pragma unroll
    for (int u = 0; u < 8; u++)
#pragma unroll
      for (int c = 0; c < NRHS; c++)
        v[u][c] = __ldcg(b + (size_t)c * bstride + pj[u]);
#pragma unroll
    for (int u = 0; u < 8; u++)
      if (j0 + 256 * u < t)
#pragma unroll
        for (int c = 0; c < NRHS; c++)
          d.xp[(size_t)c * d.tmax + j0 + 256 * u] = v[u][c];
  }
}

// mu[c][i] = sum_{j<=i} Ginv[i][j] * xp_c[j]   (one CTA per eta i: the whole row is in flight at once,
// the kernel is a single wave of t CTAs -- latency, not bandwidth, is what matters for 8 t^2/2 bytes)
template <int NRHS>
__global__ void __launch_bounds__(256) pfi_mu_kernel(DeviceModel d, bool checkState)
{
  __shared__ double part[8][NRHS];
  if (checkState && !iter_active(d.st))
    return;
  const int t = d.st->numEtas;
  const int i = blockIdx.x;
  if (i >= t)
    return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double *__restrict__ grow = d.Ginv + (size_t)i * d.tmax;
  const double *__restrict__ xp = d.xp;
  double acc[NRHS];
#pragma unroll
  for (int c = 0; c < NRHS; c++)
    acc[c] = 0.0;
  for (int j = threadIdx.x; j <= i; j += 1024) {
    double g[4];
#pragma unroll
    for (int u = 0; u < 4; u++)
      g[u] = (j + 256 * u <= i) ? __ldcs(grow + j + 256 * u) : 0.0;
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int jj = min(j + 256 * u, i);
#pragma unroll
      for (int c = 0; c < NRHS; c++)
        acc[c] = fma(g[u], __ldg(xp + (size_t)c * d.tmax + jj), acc[c]);
    }
  }
#pragma unroll
  for (int c = 0; c < NRHS; c++) {
    acc[c] = warp_sum(acc[c]);
    if (lane == 0)
      part[warp][c] = acc[c];
  }
  __syncthreads();
  if (threadIdx.x < NRHS) {
    double sum = 0.0;
#pragma unroll
    for (int w = 0; w < 8; w++)
      sum += part[w][threadIdx.x];
    d.mu[(size_t)threadIdx.x * d.tmax + i] = sum;
  }
}

// x_c[p] -= sum_{i<t} W[p][i] * mu_c[i] : a GEMV over the first t columns of the m x tmax panel,
// same shape as gemv_rows_kernel (one CTA streams R = 2 rows, DEPTH = 2 sixteen-byte loads per row in
// flight per thread; mu goes through L1).  pivotTail: the last CTA then evaluates the accuracy gate
// and the primal step (pivot_scalars_body) on the finished columns.
template <int NRHS>
__global__ void __launch_bounds__(256) pfi_apply_kernel(DeviceModel d, double *__restrict__ x, int xstride,
                                                        bool checkState, bool pivotTail)
{
  constexpr int R = 2, DEPTH = 2;
  __shared__ double part[8][R * NRHS];
  if (checkState && !iter_active(d.st))
    return;
  const int t = d.st->numEtas;
  if (t > 0) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int half = (t + 1) >> 1; // double2 per row; an odd t reads one stale entry, masked below
    const int ngroups = (d.m + R - 1) / R;
    for (int g = blockIdx.x; g < ngroups; g += gridDim.x) {
      const int p0 = g * R;
      const double2 *row[R];
#pragma unroll
      for (int r = 0; r < R; r++)
        row[r] = reinterpret_cast<const double2 *>(d.W + (size_t)min(p0 + r, d.m - 1) * d.tmax);
      double acc[R][NRHS];
#pragma unroll
      for (int r = 0; r < R; r++)
#pragma unroll
        for (int c = 0; c < NRHS; c++)
          acc[r][c] = 0.0;
      for (int j = threadIdx.x; j < half; j += 256 * DEPTH) {
        double2 a[DEPTH][R];
#pragma unroll
        for (int u = 0; u < DEPTH; u++) {
          const bool p = j + 256 * u < half;
#pragma unroll
          for (int r = 0; r < R; r++)
            a[u][r] = p ? __ldcs(row[r] + j + 256 * u) : make_double2(0.0, 0.0);
        }
#pragma unroll
        for (int u = 0; u < DEPTH; u++) {
          const int jj = min(j + 256 * u, half - 1);
          const bool second = 2 * jj + 1 < t;
#pragma unroll
          for (int c = 0; c < NRHS; c++) {
            const double m0 = __ldg(d.mu + (size_t)c * d.tmax + 2 * jj);
            const double m1 = second ? __ldg(d.mu + (size_t)c * d.tmax + 2 * jj + 1) : 0.0;
#pragma unroll
            for (int r = 0; r < R; r++) {
              acc[r][c] = fma(a[u][r].x, m0, acc[r][c]);
              acc[r][c] = fma(second ? a[u][r].y : 0.0, m1, acc[r][c]);
            }
          }
        }
      }
#pragma unroll
      for (int r = 0; r < R; r++)
#pragma unroll
        for (int c = 0; c < NRHS; c++) {
          const double v = warp_sum(acc[r][c]);
          if (lane == 0)
            part[warp][r * NRHS + c] = v;
        }
      __syncthreads();
      if (threadIdx.x < R * NRHS) {
        double sum = 0.0;
#pragma unroll
        for (int w = 0; w < 8; w++)
          sum += part[w][threadIdx.x];
        const int r = threadIdx.x / NRHS, c = threadIdx.x % NRHS;
        if (p0 + r < d.m)
          x[(size_t)c * xstride + p0 + r] -= sum;
      }
      __syncthreads();
    }
  }
  if (!pivotTail)
    return;
  if (!last_block_done(d.tailCounter + TAIL_PFI_APPLY))
    return;
  if (threadIdx.x == 0)
    pivot_scalars_body(d);
}

// x_c[p] -= sum_{i<t} W[p][i] * mu_c[i]   (one warp per position, eight loads of the panel row in
// flight per lane, 64 warps per SM).  pivotTail: the last CTA then evaluates the accuracy gate and
// the primal step (pivot_scalars_body) on the finished columns.
template <int NRHS>
__global__ void __launch_bounds__(256) pfi_apply_warp_kernel(DeviceModel d, double *__restrict__ x, int xstride,
                                                        bool checkState, bool pivotTail)
{
  if (checkState && !iter_active(d.st))
    return;
  const int t = d.st->numEtas;
  // row-sharded run: this rank's positions only, results into its chunk of gatherP (written even
  // when there is no eta: the all-gather and the merge that follow are part of a fixed sequence)
  const bool sharded = d.shardW > 1 && d.shardPanel;
  const int pBegin = sharded ? min(d.m, d.shardRank * d.shardPerM) : 0;
  const int pEnd = sharded ? min(d.m, pBegin + d.shardPerM) : d.m;
  if (t > 0 || sharded) {
    const int lane = threadIdx.x & 31;
    const int warpsPerBlock = blockDim.x >> 5;
    for (int p = pBegin + blockIdx.x * warpsPerBlock + (threadIdx.x >> 5); p < pEnd;
         p += gridDim.x * warpsPerBlock) {
      const double *wrow = d.W + (size_t)p * d.tmax;
      double acc[NRHS];
#pragma unroll
      for (int c = 0; c < NRHS; c++)
        acc[c] = 0.0;
      for (int i = lane; i < t; i += 256) {
        double w[8];
#pragma unroll
        for (int u = 0; u < 8; u++)
          w[u] = (i + 32 * u < t) ? __ldcs(wrow + i + 32 * u) : 0.0;
#pragma unroll
        for (int u = 0; u < 8; u++) {
          const int ii = min(i + 32 * u, t - 1);
#pragma unroll
          for (int c = 0; c < NRHS; c++)
            acc[c] = fma(w[u], __ldg(d.mu + (size_t)c * d.tmax + ii), acc[c]);
        }
      }
#pragma unroll
      for (int c = 0; c < NRHS; c++)
        acc[c] = warp_sum(acc[c]);
      if (lane == 0)
        for (int c = 0; c < NRHS; c++) {
          if (sharded)
            d.gatherP[((size_t)d.shardRank * NRHS + c) * d.shardPerM + (p - pBegin)] = x[(size_t)c * xstride + p] - acc[c];
          else
            x[(size_t)c * xstride + p] -= acc[c];
        }
    }
  }
  if (!pivotTail || sharded) // sharded: the gate runs as the tail of pfi_merge_kernel, after the gather
    return;
  if (!last_block_done(d.tailCounter + TAIL_PFI_APPLY))
    return;
  if (threadIdx.x == 0)
    pivot_scalars_body(d);
}

// sharded run, after the all-gather of gatherP: x_c[p] = gathered value (thread per position);
// pivotTail as in pfi_apply_warp_kernel
template <int NRHS>
__global__ void __launch_bounds__(256) pfi_merge_kernel(DeviceModel d, double *__restrict__ x, int xstride,
                                                        bool checkState, bool pivotTail)
{
  if (checkState && !iter_active(d.st))
    return;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < d.m) {
    const int rk = p / d.shardPerM, off = p - rk * d.shardPerM;
#pragma unroll
    for (int c = 0; c < NRHS; c++)
      x[(size_t)c * xstride + p] = d.gatherP[((size_t)rk * NRHS + c) * d.shardPerM + off];
  }
  if (!pivotTail)
    return;
  if (!last_block_done(d.tailCounter + TAIL_PFI_APPLY))
    return;
  if (threadIdx.x == 0)
    pivot_scalars_body(d);
}

// rho[nucRow[i]] = gathered BTRAN GEMV result i (sharded run)
__global__ void btran_scatter_kernel(DeviceModel d, double *__restrict__ rhoOut, bool checkState)
{
  if (checkState && !iter_active(d.st))
    return;
  const int k = d.fd->k;
  const int perK = ((k + d.shardW - 1) / d.shardW + 7) & ~7;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < k; i += gridDim.x * blockDim.x) {
    const int rk = i / perK;
    rhoOut[d.nucRow[i]] = d.gatherB[(size_t)rk * d.shardPerK + (i - rk * perK)];
  }
}

static void shard_all_gather(void *buf, size_t bytesPerRank, cudaStream_t s)
{
  if (g_shardCtx.allGather(g_shardCtx.comm, buf, bytesPerRank, s) != 0)
    throw std::runtime_error("clp_b200: all-gather failed");
}

template <int NRHS>
static void ftran_impl(const DeviceModel &d, double *b, bool applyEtas, bool checkState,
                       cudaStream_t s, bool pivotTail = false, bool pregathered = false)
{
  const int m = d.m;
  // fixed launch shapes (grid-stride kernels read k from the device-side FactorDesc)
  const int maxk = d.m;
  int gblocks = (roundUp8(maxk) + 255) / 256;
  if (gblocks > device_sm_count())
    gblocks = device_sm_count();
  double *xg = d.ywork + (size_t)3 * roundUp8(maxk);
  if (!pregathered) // the row pass (rowpass.cu) writes xg together with the right-hand sides
    gather_nucleus_kernel<<<gblocks, 256, 0, s>>>(d, b, m, xg, NRHS, checkState);
  int blocks = maxk < device_sm_count() * g_gemvGridMul ? maxk : device_sm_count() * g_gemvGridMul;
  if (g_kernelTimers && checkState)
    cudaEventRecord(g_kernelTimers->ftranGemv[0], s);
  const bool sharded = d.shardW > 1;
  double *y = sharded ? d.gatherY : d.ywork;
#define CLPB_GEMV_F(R_, D_)                                                                                   \
  gemv_rows_kernel<NRHS, R_, D_><<<blocks, 256, 0, s>>>(d.fd, 0, xg, y, -1, nullptr, d.st, checkState, d.shardW, \
                                                        d.shardRank, d.shardPerK)
  if (NRHS == 1)
    CLPB_GEMV_F(1, 8);
  else if (g_gemvVariantF == 1)
    CLPB_GEMV_F(1, 4);
  else if (g_gemvVariantF == 2)
    CLPB_GEMV_F(1, 8);
  else if (g_gemvVariantF == 3)
    CLPB_GEMV_F(2, 4);
  else if (g_gemvVariantF == 4)
    CLPB_GEMV_F(4, 1);
  else if (g_gemvVariantF == 5)
    CLPB_GEMV_F(4, 2);
  else if (g_gemvVariantF == 6)
    CLPB_GEMV_F(1, 2);
  else if (g_gemvVariantF == 7 && !sharded)
    gemv_warp_rows_kernel<NRHS, 4><<<device_sm_count() * g_gemvGridMul, 256, 0, s>>>(d.fd, 0, xg, y, -1, nullptr, d.st, checkState);
  else if (g_gemvVariantF == 8 && !sharded)
    gemv_warp_rows_kernel<NRHS, 8><<<device_sm_count() * g_gemvGridMul, 256, 0, s>>>(d.fd, 0, xg, y, -1, nullptr, d.st, checkState);
  else
    CLPB_GEMV_F(2, 2);
#undef CLPB_GEMV_F
  if (g_kernelTimers && checkState)
    cudaEventRecord(g_kernelTimers->ftranGemv[1], s);
  if (sharded)
    shard_all_gather(d.gatherY, sizeof(double) * NRHS * d.shardPerK, s);
  ftran_spread_kernel<NRHS><<<(m * 8 + 255) / 256, 256, 0, s>>>(d, b, m, y, checkState, applyEtas);
  if (applyEtas) {
    pfi_mu_kernel<NRHS><<<d.tmax, 256, 0, s>>>(d, checkState);
    if (sharded && d.shardPanel) {
      int pblocks = (d.shardPerM + 7) / 8;
      if (pblocks > device_sm_count() * 8)
        pblocks = device_sm_count() * 8;
      pfi_apply_warp_kernel<NRHS><<<pblocks, 256, 0, s>>>(d, b, m, checkState, false);
      shard_all_gather(d.gatherP, sizeof(double) * NRHS * d.shardPerM, s);
      pfi_merge_kernel<NRHS><<<(m + 255) / 256, 256, 0, s>>>(d, b, m, checkState, pivotTail);
    } else if (g_pfiApplyVariant == 1) {
      int pblocks = (m + 1) / 2;
      if (pblocks > device_sm_count() * 8)
        pblocks = device_sm_count() * 8;
      pfi_apply_kernel<NRHS><<<pblocks, 256, 0, s>>>(d, b, m, checkState, pivotTail);
    } else {
      int pblocks = (m + 7) / 8;
      if (pblocks > device_sm_count() * 8)
        pblocks = device_sm_count() * 8;
      pfi_apply_warp_kernel<NRHS><<<pblocks, 256, 0, s>>>(d, b, m, checkState, pivotTail);
    }
  }
}

// FTRAN of the first nrhs vectors of d.rhs3 (in place).
void launch_ftran(const DeviceModel &d, int nrhs, bool applyEtas, cudaStream_t s)
{
  if (nrhs == 1)
    ftran_impl<1>(d, d.rhs3, applyEtas, applyEtas, s);
  else if (nrhs == 2)
    ftran_impl<2>(d, d.rhs3, applyEtas, applyEtas, s);
  else
    ftran_impl<3>(d, d.rhs3, applyEtas, applyEtas, s);
}

// The three FTRANs of a simplex iteration (a_q, rho -> tau, bound-flip column) with the eta panel
// and, as the tail of the last kernel, the pivot accuracy gate / primal step length.
void launch_ftran_iteration(const DeviceModel &d, bool pregathered, cudaStream_t s)
{
  ftran_impl<3>(d, d.rhs3, true, true, s, true, pregathered);
}

// ---------------------------------------------------------------------------------------
// out[j] = scale * sum_{i>=j, i<t} Ginv[i][j] * W[row][i]   for j < t
//   mode 0 : nu (BTRAN eta transposes), vec = W[pivot row][:]
//   (the new row t of Ginv is -nu / alphaCol for the same vec: eta_append_row, kernels_common.cuh)
//   mode 2 : nu for a general BTRAN, vec = d.mu (the t dot products W_i . v)
// nu[j] = sum_{i=j}^{t-1} Ginv[i][j] * vec[i] = (row j of GinvT) . vec : one CTA per j, coalesced
__global__ void __launch_bounds__(256) eta_rowvec_kernel(DeviceModel d, int mode, bool checkState)
{
  __shared__ double part[8];
  if (checkState && !iter_active(d.st))
    return;
  const int t = d.st->numEtas;
  const int j = blockIdx.x;
  if (j >= t)
    return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const double *__restrict__ vec = mode == 2 ? d.mu : d.W + (size_t)d.st->pivotRow * d.tmax;
  const double *__restrict__ grow = d.GinvT + (size_t)j * d.tmax;
  double acc = 0.0;
  for (int i = j + threadIdx.x; i < t; i += 1024) {
    double g[4];
#pragma unroll
    for (int u = 0; u < 4; u++)
      g[u] = (i + 256 * u < t) ? __ldcs(grow + i + 256 * u) : 0.0;
#pragma unroll
    for (int u = 0; u < 4; u++)
      acc = fma(g[u], __ldg(vec + min(i + 256 * u, t - 1)), acc);
  }
  acc = warp_sum(acc);
  if (lane == 0)
    part[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sum = 0.0;
#pragma unroll
    for (int w = 0; w < 8; w++)
      sum += part[w];
    d.nu[j] = sum;
  }
}
void launch_eta_rowvec(const DeviceModel &d, int mode, bool checkState, cudaStream_t s)
{
  eta_rowvec_kernel<<<d.tmax, 256, 0, s>>>(d, mode, checkState);
}

// u = e_r - sum_j e_{p_j} nu_j ; rho_C = -u_C    (thread per position)
__global__ void btran_build_u_kernel(DeviceModel d, double *rhoOut, bool checkState,
                                     const double *vin)
{
  if (checkState && !iter_active(d.st))
    return;
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= d.m)
    return;
  const int r = d.st->pivotRow;
  double u = vin ? vin[p] : ((p == r) ? 1.0 : 0.0);
  if (d.st->numEtas > 0) {
    // etas that pivoted on this position, newest first (fixed order => deterministic sum)
    double sum = 0.0;
    for (int e = d.etaLastOfPos[p]; e >= 0; e = d.etaPrevSame[e])
      sum += d.nu[e];
    u -= sum;
  }
  d.uwork[p] = u;
  if (d.posToNuc[p] < 0)
    rhoOut[p] = -u;
}

// rho_C = -u_C for a dense input u (already in d.uwork)
__global__ void btran_dense_c_kernel(DeviceModel d, double *__restrict__ rhoOut)
{
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= d.m)
    return;
  if (d.posToNuc[p] < 0)
    rhoOut[p] = -d.uwork[p];
}

// s_j = u[nucRow[j]] + sum_{rows i in C of column nucCol[j]} a_ij u[i]   (warp per nucleus col)
__global__ void btran_s_kernel(DeviceModel d, bool checkState)
{
  if (checkState && !iter_active(d.st))
    return;
  const int lane = threadIdx.x & 31;
  const int k = d.fd->k, ldk = d.fd->ldk;
  const int warpsPerBlock = blockDim.x >> 5;
  for (int j = blockIdx.x * warpsPerBlock + (threadIdx.x >> 5); j < k;
       j += gridDim.x * warpsPerBlock) {
    const int col = d.nucCol[j];
    double acc = 0.0;
    for (int e = d.colStart[col] + lane; e < d.colStart[col + 1]; e += 32) {
      int i = d.rowIdx[e];
      if (d.posToNuc[i] < 0)
        acc = fma(d.val[e], d.uwork[i], acc);
    }
    acc = warp_sum(acc);
    if (lane == 0)
      d.swork[j] = acc + d.uwork[d.nucRow[j]];
  }
  // zero the padding so the GEMV can run over ldk
  if (blockIdx.x == 0 && threadIdx.x < 8 && k + threadIdx.x < ldk)
    d.swork[k + threadIdx.x] = 0.0;
}

// u_p = [p == r] - sum of nu over the etas that pivoted on position p (newest first: fixed order)
__device__ __forceinline__ double btran_u_of(const DeviceModel &d, int p, int r, int t)
{
  double u = (p == r) ? 1.0 : 0.0;
  if (t > 0) {
    double sum = 0.0;
    for (int e = d.etaLastOfPos[p]; e >= 0; e = d.etaPrevSame[e])
      sum += d.nu[e];
    u -= sum;
  }
  return u;
}

// Simplex BTRAN prelude in one kernel (u is sparse: nonzero only on r and the eta positions, so it
// is evaluated where needed instead of being materialised first):
//   rho_C = -u_C                                      (thread per position)
//   s_j = u[nucRow[j]] + sum_{i in C} a_{i,col j} u_i (warp per nucleus column)
__global__ void __launch_bounds__(256) btran_us_kernel(DeviceModel d, double *__restrict__ rhoOut)
{
  if (!iter_active(d.st))
    return;
  const int r = d.st->pivotRow, t = d.st->numEtas;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < d.m; p += gridDim.x * blockDim.x)
    if (d.posToNuc[p] < 0)
      rhoOut[p] = -btran_u_of(d, p, r, t);
  const int lane = threadIdx.x & 31;
  const int k = d.fd->k, ldk = d.fd->ldk;
  const int warpsPerBlock = blockDim.x >> 5;
  const int *__restrict__ s1cRow = d.fd->s1cRow;
  const double *__restrict__ s1cVal = d.fd->s1cVal;
  for (int j = blockIdx.x * warpsPerBlock + (threadIdx.x >> 5); j < k; j += gridDim.x * warpsPerBlock) {
    double acc = 0.0;
    const int e1 = d.s1cStart[j + 1];
    for (int e = d.s1cStart[j] + lane; e < e1; e += 32) { // entries of column j in rows of C only
      const double u = btran_u_of(d, s1cRow[e], r, t);
      if (u != 0.0)
        acc = fma(s1cVal[e], u, acc);
    }
    acc = warp_sum(acc);
    if (lane == 0)
      d.swork[j] = acc + btran_u_of(d, d.nucRow[j], r, t);
  }
  // zero the padding so the GEMV can run over ldk
  if (blockIdx.x == 0 && threadIdx.x < 8 && k + threadIdx.x < ldk)
    d.swork[k + threadIdx.x] = 0.0;
}

static void btran_gemv(const DeviceModel &d, double *rhoOut, bool checkState, cudaStream_t s);

static void btran_tail(const DeviceModel &d, double *rhoOut, bool checkState, cudaStream_t s)
{
  int sblocks = (d.m + 7) / 8;
  if (sblocks > device_sm_count() * 8)
    sblocks = device_sm_count() * 8;
  btran_s_kernel<<<sblocks, 256, 0, s>>>(d, checkState);
  btran_gemv(d, rhoOut, checkState, s);
}

static void btran_gemv(const DeviceModel &d, double *rhoOut, bool checkState, cudaStream_t s)
{
  int blocks = d.m < device_sm_count() * g_gemvGridMul ? d.m : device_sm_count() * g_gemvGridMul;
  if (g_kernelTimers && checkState)
    cudaEventRecord(g_kernelTimers->btranGemv[0], s);
  const bool sharded = d.shardW > 1;
#define CLPB_GEMV_B(R_, D_)                                                                              \
  gemv_rows_kernel<1, R_, D_><<<blocks, 256, 0, s>>>(d.fd, 1, d.swork, sharded ? d.gatherB : rhoOut, d.m, \
                                                     d.nucRow, d.st, checkState, d.shardW, d.shardRank, d.shardPerK)
  if (g_gemvVariantB == 1)
    CLPB_GEMV_B(1, 4);
  else if (g_gemvVariantB == 2)
    CLPB_GEMV_B(2, 4);
  else if (g_gemvVariantB == 3)
    CLPB_GEMV_B(2, 8);
  else if (g_gemvVariantB == 4)
    CLPB_GEMV_B(4, 4);
  else if (g_gemvVariantB == 5)
    CLPB_GEMV_B(4, 2);
  else if (g_gemvVariantB == 6 && !sharded)
    gemv_warp_rows_kernel<1, 8><<<device_sm_count() * g_gemvGridMul, 256, 0, s>>>(d.fd, 1, d.swork, rhoOut, d.m, d.nucRow, d.st, checkState);
  else if (g_gemvVariantB == 7 && !sharded)
    gemv_warp_rows_kernel<1, 4><<<device_sm_count() * g_gemvGridMul, 256, 0, s>>>(d.fd, 1, d.swork, rhoOut, d.m, d.nucRow, d.st, checkState);
  else
    CLPB_GEMV_B(1, 8);
#undef CLPB_GEMV_B
  if (g_kernelTimers && checkState)
    cudaEventRecord(g_kernelTimers->btranGemv[1], s);
  if (sharded) {
    shard_all_gather(d.gatherB, sizeof(double) * d.shardPerK, s);
    int sb = (d.m + 255) / 256;
    btran_scatter_kernel<<<sb > device_sm_count() * 4 ? device_sm_count() * 4 : sb, 256, 0, s>>>(d, rhoOut, checkState);
  }
}

// rho = B_t^-T e_r with r = st->pivotRow ; result in d.rho
void launch_btran_unit(const DeviceModel &d, bool checkState, cudaStream_t s)
{
  (void)checkState;
  launch_eta_rowvec(d, 0, true, s); // no-op when numEtas == 0
  int sblocks = (d.m + 7) / 8;
  if (sblocks > device_sm_count() * 8)
    sblocks = device_sm_count() * 8;
  btran_us_kernel<<<sblocks, 256, 0, s>>>(d, d.rho);
  btran_gemv(d, d.rho, true, s);
}

// s_i = W[:,i] . v   (one warp per eta; general BTRAN only -- the simplex BTRAN starts from a
// unit vector and reads a row of W instead)
__global__ void eta_dot_kernel(DeviceModel d, const double *__restrict__ v)
{
  const int t = d.st->numEtas;
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= t)
    return;
  double acc = 0.0;
  for (int p = lane; p < d.m; p += 32)
    acc = fma(d.W[(size_t)p * d.tmax + i], v[p], acc);
  acc = warp_sum(acc);
  if (lane == 0)
    d.mu[i] = acc;
}

// vec = B_t^-T vec for a dense vector (computeDuals right after a refactorization uses
// applyEtas=false; the general form backs the updateColumnTranspose entry point)
void launch_btran_dense(const DeviceModel &d, double *vec, bool applyEtas, cudaStream_t s)
{
  if (applyEtas) {
    eta_dot_kernel<<<(d.tmax + 7) / 8, 256, 0, s>>>(d, vec);
    launch_eta_rowvec(d, 2, false, s);
    btran_build_u_kernel<<<(d.m + 255) / 256, 256, 0, s>>>(d, vec, false, vec);
  } else {
    cudaMemcpyAsync(d.uwork, vec, sizeof(double) * d.m, cudaMemcpyDeviceToDevice, s);
    btran_dense_c_kernel<<<(d.m + 255) / 256, 256, 0, s>>>(d, vec);
  }
  btran_tail(d, vec, false, s);
}

// FTRAN on an arbitrary device buffer of nrhs vectors (stride m), optional etas, no state check
void launch_ftran_buffer(const DeviceModel &d, double *buf, int nrhs, bool applyEtas, cudaStream_t s)
{
  if (nrhs == 1)
    ftran_impl<1>(d, buf, applyEtas, false, s);
  else if (nrhs == 2)
    ftran_impl<2>(d, buf, applyEtas, false, s);
  else
    ftran_impl<3>(d, buf, applyEtas, false, s);
}

} // namespace clpb
