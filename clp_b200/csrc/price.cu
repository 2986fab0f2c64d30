// price.cu -- PRICE (tableau row) and the plain matrix products, device resident.
//
// Replaces ClpPackedMatrix::transposeTimes (/root/reference/src/ClpPackedMatrix.cpp:706 ->
// transposeTimesByColumn :961 -> gutsOfTransposeTimesUnscaled :1640/:1799, the variant that
// skips basic columns by status).  PRICE streams the CSC copy of A once (12 B per nonzero) with
// one warp per column and leaves raw dot products; the status mask, the zero tolerance, the slack
// part of the row and the ratio test (ClpSimplexDual::dualColumn) follow in the row pass
// (rowpass.cu).
#include "kernels_common.cuh"

namespace clpb {

// alphaRow[j] = rho^T a_j (raw dot product) for the nonbasic, non-fixed columns j of
// [colBegin,colEnd); basic / fixed columns get 0 without touching their entries.
// One warp per column, the matrix goes from HBM straight into registers: while a column is being
// reduced the NEXT column of the warp (4 x 32 entries: 4-byte row indices + 8-byte values) is
// already in flight, and the column bounds are fetched two columns ahead.  Only rho lives in
// shared memory.  tests/microbench/iter_kernels.cu compares it (m = 10^4, n = 10^5, 10^7 entries)
// with the variants that stage the CSC tiles through shared memory with cp.async.bulk (TMA) --
// those are bound by shared-memory wavefronts (TMA writes + index/value reads + rho gathers), not
// by HBM.
template <int THREADS, int CTAS, bool SMEM_RHO>
__global__ void __launch_bounds__(THREADS, CTAS)
    price_ldg_kernel(DeviceModel d, int colBegin, int colEnd)
{
  extern __shared__ __align__(16) unsigned char rawRho[];
  if (!iter_active(d.st))
    return;
  double *srho = reinterpret_cast<double *>(rawRho);
  const double *__restrict__ rhoG = d.rho;
  if (SMEM_RHO) {
    for (int i = threadIdx.x; i < d.m; i += THREADS)
      srho[i] = rhoG[i];
    __syncthreads();
  }
  const int *__restrict__ rowIdx = d.rowIdx;
  const double *__restrict__ val = d.val;
  const int *__restrict__ colStart = d.colStart;
  const unsigned char *__restrict__ status = d.status;
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (THREADS >> 5) + (threadIdx.x >> 5);
  const int GW = gridDim.x * (THREADS >> 5);
  int nb0 = 0, nb1 = 0;
  int ni[4];
  double nv[4];
  auto fetchBounds = [&](int jj) {
    nb0 = nb1 = 0;
    if (jj < colEnd) {
      const unsigned char st = status[jj];
      if (st != basic && st != isFixed) {
        nb0 = __ldg(colStart + jj);
        nb1 = __ldg(colStart + jj + 1);
      }
    }
  };
  auto fetchEntries = [&](int b0, int b1) {
#pragma unroll
    for (int u = 0; u < 4; u++) {
      const int e = b0 + lane + 32 * u;
      const bool p = e < b1;
      ni[u] = p ? __ldcs(rowIdx + e) : 0;
      nv[u] = p ? __ldcs(val + e) : 0.0;
    }
  };
  int j = colBegin + gw;
  fetchBounds(j);
  int b0 = nb0, b1 = nb1;
  fetchEntries(b0, b1);
  fetchBounds(j + GW);
  for (; j < colEnd; j += GW) {
    int ci[4];
    double cv[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      ci[u] = ni[u];
      cv[u] = nv[u];
    }
    const int cb0 = b0, cb1 = b1;
    b0 = nb0;
    b1 = nb1;
    fetchEntries(b0, b1);    // next column's entries in flight
    fetchBounds(j + 2 * GW); // bounds two columns ahead
    double acc0 = cv[0] * (SMEM_RHO ? srho[ci[0]] : __ldg(rhoG + ci[0]));
    double acc1 = cv[1] * (SMEM_RHO ? srho[ci[1]] : __ldg(rhoG + ci[1]));
    acc0 = fma(cv[2], SMEM_RHO ? srho[ci[2]] : __ldg(rhoG + ci[2]), acc0);
    acc1 = fma(cv[3], SMEM_RHO ? srho[ci[3]] : __ldg(rhoG + ci[3]), acc1);
    for (int e = cb0 + 128 + lane; e < cb1; e += 32) { // columns longer than 128 entries
      const int r = __ldg(rowIdx + e);
      acc0 = fma(__ldg(val + e), SMEM_RHO ? srho[r] : __ldg(rhoG + r), acc0);
    }
    const double acc = warp_sum(acc0 + acc1);
    if (lane == 0)
      d.alphaRow[j] = acc; // the row pass applies the zero tolerance
  }
}

// The shape follows from the size of rho: in shared memory with two 640-thread CTAs per SM, with
// one 1024-thread CTA per SM, or read through L1/L2 when it does not fit.
void launch_price(const DeviceModel &d, int colBegin, int colEnd, cudaStream_t s)
{
  int ncol = colEnd - colBegin;
  if (ncol <= 0)
    return;
  const size_t rhoBytes = sizeof(double) * (size_t)d.m;
  static bool attrSet = false;
  if (!attrSet) {
    cudaFuncSetAttribute(price_ldg_kernel<640, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
    cudaFuncSetAttribute(price_ldg_kernel<1024, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
    attrSet = true;
  }
  const int numSMs = device_sm_count();
  if (g_kernelTimers)
    cudaEventRecord(g_kernelTimers->price[0], s);
  if (rhoBytes <= 112 * 1024) {
    price_ldg_kernel<640, 2, true><<<numSMs * 2, 640, rhoBytes, s>>>(d, colBegin, colEnd);
  } else if (rhoBytes <= 224 * 1024) {
    price_ldg_kernel<1024, 1, true><<<numSMs, 1024, rhoBytes, s>>>(d, colBegin, colEnd);
  } else {
    price_ldg_kernel<640, 2, false><<<numSMs * 2, 640, 0, s>>>(d, colBegin, colEnd);
  }
  if (g_kernelTimers)
    cudaEventRecord(g_kernelTimers->price[1], s);
}

// ---------------------------------------------------------------------------------------
// z[j] = scalar * pi^T a_j for all columns (ClpPackedMatrix::transposeTimes, plain variant :1484)
__global__ void __launch_bounds__(256)
    transpose_times_kernel(DeviceModel d, const double *__restrict__ pi, double *__restrict__ z,
                           double scalar)
{
  const int lane = threadIdx.x & 31;
  const int warpsPerBlock = blockDim.x >> 5;
  for (int j = blockIdx.x * warpsPerBlock + (threadIdx.x >> 5); j < d.n;
       j += gridDim.x * warpsPerBlock) {
    double acc = 0.0;
    for (int e = d.colStart[j] + lane; e < d.colStart[j + 1]; e += 32)
      acc = fma(__ldg(d.val + e), __ldg(pi + __ldg(d.rowIdx + e)), acc);
    acc = warp_sum(acc);
    if (lane == 0)
      z[j] = scalar * acc;
  }
}
void launch_transpose_times(const DeviceModel &d, const double *pi, double *z, double scalar,
                            cudaStream_t s)
{
  int blocks = (d.n + 7) / 8;
  if (blocks > device_sm_count() * 16)
    blocks = device_sm_count() * 16;
  if (d.n > 0)
    transpose_times_kernel<<<blocks, 256, 0, s>>>(d, pi, z, scalar);
}

// y[i] = scalar * sum_j A_ij x_j  via the row copy (ClpPackedMatrix::times :296)
__global__ void __launch_bounds__(256)
    times_rows_kernel(DeviceModel d, const double *__restrict__ x, double *__restrict__ y,
                      double scalar)
{
  const int lane = threadIdx.x & 31;
  const int warpsPerBlock = blockDim.x >> 5;
  for (int i = blockIdx.x * warpsPerBlock + (threadIdx.x >> 5); i < d.m;
       i += gridDim.x * warpsPerBlock) {
    double acc = 0.0;
    for (int e = d.rowStart[i] + lane; e < d.rowStart[i + 1]; e += 32)
      acc = fma(__ldg(d.rval + e), __ldg(x + __ldg(d.colIdx + e)), acc);
    acc = warp_sum(acc);
    if (lane == 0)
      y[i] = scalar * acc;
  }
}
void launch_times_rows(const DeviceModel &d, const double *x, double *y, double scalar,
                       cudaStream_t s)
{
  int blocks = (d.m + 7) / 8;
  if (blocks > device_sm_count() * 16)
    blocks = device_sm_count() * 16;
  times_rows_kernel<<<blocks, 256, 0, s>>>(d, x, y, scalar);
}

} // namespace clpb
