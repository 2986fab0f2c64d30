// iter_kernels.cu -- micro-benchmarks for the second generation of the per-iteration kernels:
//   * GEMV over the nucleus inverse: current CTA-per-4-rows kernel vs. "items" kernel
//     (x staged in shared memory, (row, quarter) work items, last-arriver combine)
//   * PRICE over a realistic CSC matrix: current 4x2x1024-entry TMA pipelines vs. one deep ring of
//     large tiles per CTA (u32 or u16 row indices)
//   * rank-32 DGEMM update of the refactorization: SIMT 4x4 kernel vs. DMMA (mma.m8n8k4.f64)
// Not part of the product; built and run by hand:
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o ik iter_kernels.cu && ./ik
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

// SMs of device 0 (132 on an H100 SXM): launch shapes are multiples of it
static int numSms()
{
  static int s = 0;
  if (s == 0)
    cudaDeviceGetAttribute(&s, cudaDevAttrMultiProcessorCount, 0);
  return s;
}
#include <random>
#include <vector>

#define CK(x)                                                                                      \
  do {                                                                                             \
    cudaError_t e = (x);                                                                           \
    if (e != cudaSuccess) {                                                                        \
      printf("CUDA error %s line %d\n", cudaGetErrorString(e), __LINE__);                          \
      exit(1);                                                                                     \
    }                                                                                              \
  } while (0)

__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity)
{
  asm volatile("{\n.reg .pred p;\nWL:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra WD;\nbra WL;\nWD:\n}\n" ::"r"(smem_u32(bar)),
               "r"(parity)
               : "memory");
}
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// =================================================================== GEMV
// current kernel (solve.cu gemv_rows_kernel): CTA per group of four rows, x through L1
template <int NRHS>
__global__ void __launch_bounds__(256)
    gemv_cur(const double *__restrict__ M, int k, int ldk, const double *__restrict__ x, double *__restrict__ out)
{
  constexpr int R = 4;
  __shared__ double part[8][R * NRHS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int half = ldk >> 1;
  const int ngroups = (k + R - 1) / R;
  for (int g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int i0 = g * R;
    const double2 *row[R];
#pragma unroll
    for (int r = 0; r < R; r++)
      row[r] = reinterpret_cast<const double2 *>(M + (size_t)min(i0 + r, k - 1) * ldk);
    double acc[R][NRHS];
#pragma unroll
    for (int r = 0; r < R; r++)
#pragma unroll
      for (int c = 0; c < NRHS; c++)
        acc[r][c] = 0.0;
#pragma unroll 2
    for (int j = threadIdx.x; j < half; j += 256) {
      double2 a[R];
#pragma unroll
      for (int r = 0; r < R; r++)
        a[r] = __ldcs(row[r] + j);
#pragma unroll
      for (int c = 0; c < NRHS; c++) {
        const double2 xv = __ldg(reinterpret_cast<const double2 *>(x + (size_t)c * ldk) + j);
#pragma unroll
        for (int r = 0; r < R; r++) {
          acc[r][c] = fma(a[r].x, xv.x, acc[r][c]);
          acc[r][c] = fma(a[r].y, xv.y, acc[r][c]);
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
      if (i0 + r < k)
        out[(size_t)c * ldk + i0 + r] = sum;
    }
    __syncthreads();
  }
}

// "items" kernel: one CTA per SM, all right-hand sides staged in shared memory (gathered through
// 'gather' straight from the m-vectors), work item = (row, segment q of Q); a warp streams its
// segment with DEPTH 16-byte loads in flight per lane; the partial sums go to part[q][c][row] and
// the warp that completes a row (per-row ticket) adds the Q partials in fixed order.
template <int NRHS, int DEPTH, int THREADS>
__global__ void __launch_bounds__(THREADS, 1)
    gemv_items(const double *__restrict__ M, int k, int ldk, const double *__restrict__ b, int bstride,
               const int *__restrict__ gather, double *__restrict__ part, unsigned int *__restrict__ ticket,
               double *__restrict__ out, int ostride, const int *__restrict__ outIndex, int Q, int seg2 /* double2 per segment */)
{
  extern __shared__ __align__(16) unsigned char rawx[];
  double *sx = reinterpret_cast<double *>(rawx); // [NRHS][ldk]
  for (int j = threadIdx.x; j < ldk; j += THREADS) {
    const int p = j < k ? gather[j] : 0;
#pragma unroll
    for (int c = 0; c < NRHS; c++)
      sx[c * ldk + j] = j < k ? b[(size_t)c * bstride + p] : 0.0;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (THREADS >> 5) + (threadIdx.x >> 5);
  const int GW = gridDim.x * (THREADS >> 5);
  const int half = ldk >> 1;
  const long nitems = (long)k * Q;
  for (long item = gw; item < nitems; item += GW) {
    const int i = (int)(item / Q), q = (int)(item % Q);
    const int j0 = q * seg2, j1 = min(half, j0 + seg2);
    const double2 *row = reinterpret_cast<const double2 *>(M + (size_t)i * ldk);
    double acc[NRHS];
#pragma unroll
    for (int c = 0; c < NRHS; c++)
      acc[c] = 0.0;
    for (int j = j0 + lane; j < j1; j += 32 * DEPTH) {
      double2 a[DEPTH];
#pragma unroll
      for (int u = 0; u < DEPTH; u++)
        a[u] = (j + 32 * u < j1) ? __ldcs(row + j + 32 * u) : make_double2(0.0, 0.0);
#pragma unroll
      for (int u = 0; u < DEPTH; u++) {
        const int jj = min(j + 32 * u, half - 1);
#pragma unroll
        for (int c = 0; c < NRHS; c++) {
          const double2 xv = reinterpret_cast<const double2 *>(sx + c * ldk)[jj];
          acc[c] = fma(a[u].x, xv.x, acc[c]);
          acc[c] = fma(a[u].y, xv.y, acc[c]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < NRHS; c++)
      acc[c] = warp_sum(acc[c]);
    unsigned int t = 0;
    if (lane == 0) {
#pragma unroll
      for (int c = 0; c < NRHS; c++)
        part[((size_t)q * NRHS + c) * ldk + i] = acc[c];
      __threadfence();
      t = atomicAdd(ticket + i, 1u);
    }
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t == (unsigned)Q - 1) { // last segment of this row: combine in fixed order
      __threadfence();
      if (lane < NRHS) {
        double s = 0.0;
        for (int qq = 0; qq < Q; qq++)
          s += ((volatile double *)part)[((size_t)qq * NRHS + lane) * ldk + i];
        const int o = outIndex ? outIndex[i] : i;
        out[(size_t)lane * ostride + o] = s;
      }
      if (lane == 0)
        ticket[i] = 0u;
    }
  }
}

// =================================================================== PRICE
// current kernel (price.cu price_tma_kernel<true>)
constexpr int kPriceTile = 1024, kPriceStages = 2, kPriceGroups = 4, kPriceTileAlloc = kPriceTile + 8;
__global__ void __launch_bounds__(1024, 1)
    price_cur(const int *__restrict__ rowIdx, const double *__restrict__ val, const int *__restrict__ colStart,
              const double *__restrict__ rhoG, int m, double *__restrict__ alphaRow, const int4 *__restrict__ tileDesc,
              int ntiles, int descCap)
{
  extern __shared__ __align__(128) unsigned char smemRaw[];
  unsigned long long *fullAll = reinterpret_cast<unsigned long long *>(smemRaw);
  int4 *sdescAll = reinterpret_cast<int4 *>(smemRaw + 128);
  int *sidxAll = reinterpret_cast<int *>(smemRaw + 128 + (size_t)kPriceGroups * descCap * 16);
  double *svalAll = reinterpret_cast<double *>(sidxAll + kPriceGroups * kPriceStages * kPriceTileAlloc);
  double *srho = svalAll + kPriceGroups * kPriceStages * kPriceTileAlloc;
  const int tid = threadIdx.x, lane = tid & 31;
  const int grp = tid >> 8, gt = tid & 255, gwarp = gt >> 5;
  unsigned long long *full = fullAll + grp * kPriceStages;
  int4 *sdesc = sdescAll + grp * descCap;
  int *sidx = sidxAll + grp * kPriceStages * kPriceTileAlloc;
  double *sval = svalAll + grp * kPriceStages * kPriceTileAlloc;
  const int G = gridDim.x * kPriceGroups;
  const int gg = blockIdx.x * kPriceGroups + grp;
  const int myTiles = gg < ntiles ? (ntiles - 1 - gg) / G + 1 : 0;
  for (int i = gt; i < myTiles; i += 256)
    sdesc[i] = tileDesc[gg + (size_t)i * G];
  if (tid == 0) {
    for (int q = 0; q < kPriceGroups * kPriceStages; q++)
      mbar_init(&fullAll[q], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int i, int stage) {
    const int4 ds = sdesc[i];
    const unsigned cnt = (unsigned)ds.w;
    mbar_expect_tx(&full[stage], cnt * 12u);
    bulk_g2s(sidx + stage * kPriceTileAlloc, rowIdx + ds.z, cnt * 4u, &full[stage]);
    bulk_g2s(sval + stage * kPriceTileAlloc, val + ds.z, cnt * 8u, &full[stage]);
  };
  if (gt == 0)
    for (int q = 0; q < kPriceStages && q < myTiles; q++)
      issue(q, q);
  for (int i = tid; i < m; i += 1024)
    srho[i] = rhoG[i];
  __syncthreads();
  int nb0 = 0, nb1 = 0;
  auto fetchBounds = [&](int i) {
    const int4 dn = sdesc[i];
    const int c = dn.x + min(gwarp, dn.y - 1);
    nb0 = __ldg(colStart + c);
    nb1 = __ldg(colStart + c + 1);
  };
  if (myTiles > 0)
    fetchBounds(0);
  for (int it = 0; it < myTiles; it++) {
    const int stage = it % kPriceStages;
    const int4 ds = sdesc[it];
    const int b0 = nb0 - ds.z, b1 = nb1 - ds.z;
    if (it + 1 < myTiles)
      fetchBounds(it + 1);
    mbar_wait(&full[stage], (unsigned)((it / kPriceStages) & 1));
    if (gwarp < ds.y) {
      const double *v = sval + stage * kPriceTileAlloc;
      const int *ix = sidx + stage * kPriceTileAlloc;
      double acc0 = 0.0, acc1 = 0.0;
      int e = b0 + lane;
      for (; e + 32 < b1; e += 64) {
        const int r0 = ix[e], r1 = ix[e + 32];
        const double v0 = v[e], v1 = v[e + 32];
        acc0 = fma(v0, srho[r0], acc0);
        acc1 = fma(v1, srho[r1], acc1);
      }
      if (e < b1)
        acc0 = fma(v[e], srho[ix[e]], acc0);
      const double acc = warp_sum(acc0 + acc1);
      if (lane == 0)
        alphaRow[ds.x + gwarp] = acc;
    }
    asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(256) : "memory");
    if (gt == 0 && it + kPriceStages < myTiles) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      issue(it + kPriceStages, stage);
    }
  }
}

// one deep ring of large tiles per CTA.  Tile = whole columns, first column a multiple of 4, at
// most MAXC columns and E entries (entry window aligned down to 8).  Three bulk copies per tile:
// row indices, values, and the window of colStart.  One warp per column, 4 independent chains.
constexpr int MAXC = 64;
template <int E, int S, typename IdxT, bool SMEM_RHO>
__global__ void __launch_bounds__(1024, 1)
    price_big(const IdxT *__restrict__ rowIdx, const double *__restrict__ val, const int *__restrict__ colStart,
              const double *__restrict__ rhoG, int m, double *__restrict__ alphaRow, const int4 *__restrict__ tileDesc,
              int ntiles, int descCap)
{
  extern __shared__ __align__(128) unsigned char smemRaw[];
  unsigned long long *full = reinterpret_cast<unsigned long long *>(smemRaw);
  int4 *sdesc = reinterpret_cast<int4 *>(smemRaw + 128);
  int *scol = reinterpret_cast<int *>(smemRaw + 128 + (size_t)descCap * 16); // [S][MAXC+8]
  double *sval = reinterpret_cast<double *>(scol + S * (MAXC + 8));           // [S][E]
  IdxT *sidx = reinterpret_cast<IdxT *>(sval + (size_t)S * E);                // [S][E]
  double *srho = reinterpret_cast<double *>(sidx + (size_t)S * E);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int G = gridDim.x;
  const int myTiles = (int)blockIdx.x < ntiles ? (ntiles - 1 - blockIdx.x) / G + 1 : 0;
  for (int i = tid; i < myTiles; i += 1024)
    sdesc[i] = tileDesc[blockIdx.x + (size_t)i * G];
  if (tid == 0) {
    for (int q = 0; q < S; q++)
      mbar_init(&full[q], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int i, int stage) {
    const int4 ds = sdesc[i];
    const unsigned cnt = (unsigned)ds.w;
    const unsigned colBytes = (unsigned)(((ds.y + 1 + 3) & ~3) * 4);
    mbar_expect_tx(&full[stage], cnt * (8u + (unsigned)sizeof(IdxT)) + colBytes);
    bulk_g2s(sval + (size_t)stage * E, val + ds.z, cnt * 8u, &full[stage]);
    bulk_g2s(sidx + (size_t)stage * E, rowIdx + ds.z, cnt * (unsigned)sizeof(IdxT), &full[stage]);
    bulk_g2s(scol + stage * (MAXC + 8), colStart + ds.x, colBytes, &full[stage]);
  };
  if (tid == 0)
    for (int q = 0; q < S && q < myTiles; q++)
      issue(q, q);
  if (SMEM_RHO) {
    for (int i = tid; i < m; i += 1024)
      srho[i] = rhoG[i];
  }
  __syncthreads();
  for (int it = 0; it < myTiles; it++) {
    const int stage = it % S;
    const int4 ds = sdesc[it];
    mbar_wait(&full[stage], (unsigned)((it / S) & 1));
    const double *v = sval + (size_t)stage * E;
    const IdxT *ix = sidx + (size_t)stage * E;
    const int *cs = scol + stage * (MAXC + 8);
    for (int c = warp; c < ds.y; c += 32) {
      const int b0 = cs[c] - ds.z, b1 = cs[c + 1] - ds.z;
      double acc0 = 0.0, acc1 = 0.0, acc2 = 0.0, acc3 = 0.0;
      for (int e = b0 + lane; e < b1; e += 128) {
        const bool p1 = e + 32 < b1, p2 = e + 64 < b1, p3 = e + 96 < b1;
        const int r0 = ix[e];
        const int r1 = p1 ? (int)ix[e + 32] : 0, r2 = p2 ? (int)ix[e + 64] : 0, r3 = p3 ? (int)ix[e + 96] : 0;
        const double v0 = v[e];
        const double v1 = p1 ? v[e + 32] : 0.0, v2 = p2 ? v[e + 64] : 0.0, v3 = p3 ? v[e + 96] : 0.0;
        acc0 = fma(v0, SMEM_RHO ? srho[r0] : __ldg(rhoG + r0), acc0);
        acc1 = fma(v1, SMEM_RHO ? srho[r1] : __ldg(rhoG + r1), acc1);
        acc2 = fma(v2, SMEM_RHO ? srho[r2] : __ldg(rhoG + r2), acc2);
        acc3 = fma(v3, SMEM_RHO ? srho[r3] : __ldg(rhoG + r3), acc3);
      }
      const double acc = warp_sum((acc0 + acc1) + (acc2 + acc3));
      if (lane == 0)
        alphaRow[ds.x + c] = acc;
    }
    __syncthreads();
    if (tid == 0 && it + S < myTiles) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      issue(it + S, stage);
    }
  }
}


// v3: big tiles, deep ring, but only 256 threads and LPC lanes per column (32/LPC columns per warp at
// once): ~7x fewer instructions per column than one-warp-per-column, so the CTA is load bound.
template <int E, int S, typename IdxT, int LPC, int THREADS>
__global__ void __launch_bounds__(THREADS, 1)
    price_v3(const IdxT *__restrict__ rowIdx, const double *__restrict__ val, const int *__restrict__ colStart,
             const double *__restrict__ rhoG, int m, double *__restrict__ alphaRow, const int4 *__restrict__ tileDesc,
             int ntiles, int descCap)
{
  extern __shared__ __align__(128) unsigned char smemRaw[];
  unsigned long long *full = reinterpret_cast<unsigned long long *>(smemRaw);
  int4 *sdesc = reinterpret_cast<int4 *>(smemRaw + 128);
  int *scol = reinterpret_cast<int *>(smemRaw + 128 + (size_t)descCap * 16); // [S][MAXC+8]
  double *sval = reinterpret_cast<double *>(scol + S * (MAXC + 8));           // [S][E]
  IdxT *sidx = reinterpret_cast<IdxT *>(sval + (size_t)S * E);                // [S][E]
  double *srho = reinterpret_cast<double *>(sidx + (size_t)S * E);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int G = gridDim.x;
  const int myTiles = (int)blockIdx.x < ntiles ? (ntiles - 1 - blockIdx.x) / G + 1 : 0;
  for (int i = tid; i < myTiles; i += THREADS)
    sdesc[i] = tileDesc[blockIdx.x + (size_t)i * G];
  if (tid == 0) {
    for (int q = 0; q < S; q++)
      mbar_init(&full[q], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  auto issue = [&](int i, int stage) {
    const int4 ds = sdesc[i];
    const unsigned cnt = (unsigned)ds.w;
    const unsigned colBytes = (unsigned)(((ds.y + 1 + 3) & ~3) * 4);
    mbar_expect_tx(&full[stage], cnt * (8u + (unsigned)sizeof(IdxT)) + colBytes);
    bulk_g2s(sval + (size_t)stage * E, val + ds.z, cnt * 8u, &full[stage]);
    bulk_g2s(sidx + (size_t)stage * E, rowIdx + ds.z, cnt * (unsigned)sizeof(IdxT), &full[stage]);
    bulk_g2s(scol + stage * (MAXC + 8), colStart + ds.x, colBytes, &full[stage]);
  };
  if (tid == 0)
    for (int q = 0; q < S && q < myTiles; q++)
      issue(q, q);
  for (int i = tid; i < m; i += THREADS)
    srho[i] = rhoG[i];
  __syncthreads();
  constexpr int CPW = 32 / LPC;               // columns per warp at once
  constexpr int CPP = CPW * (THREADS / 32);   // columns per pass of the CTA
  const int grp = lane / LPC, sub = lane % LPC;
  for (int it = 0; it < myTiles; it++) {
    const int stage = it % S;
    const int4 ds = sdesc[it];
    mbar_wait(&full[stage], (unsigned)((it / S) & 1));
    const double *v = sval + (size_t)stage * E;
    const IdxT *ix = sidx + (size_t)stage * E;
    const int *cs = scol + stage * (MAXC + 8);
    for (int c0 = 0; c0 < ds.y; c0 += CPP) {
      const int c = c0 + warp * CPW + grp;
      int b0 = 0, b1 = 0;
      if (c < ds.y) {
        b0 = cs[c] - ds.z;
        b1 = cs[c + 1] - ds.z;
      }
      double acc0 = 0.0, acc1 = 0.0;
      for (int e = b0 + sub; e < b1; e += 2 * LPC) {
        const bool p1 = e + LPC < b1;
        const int r0 = ix[e];
        const int r1 = p1 ? (int)ix[e + LPC] : 0;
        const double v0 = v[e];
        const double v1 = p1 ? v[e + LPC] : 0.0;
        acc0 = fma(v0, srho[r0], acc0);
        acc1 = fma(v1, srho[r1], acc1);
      }
      double acc = acc0 + acc1;
#pragma unroll
      for (int o = LPC / 2; o > 0; o >>= 1)
        acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (sub == 0 && c < ds.y)
        alphaRow[ds.x + c] = acc;
    }
    __syncthreads();
    if (tid == 0 && it + S < myTiles) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      issue(it + S, stage);
    }
  }
}


// LDG-direct price: no shared-memory staging of the matrix (only rho lives in shared memory), one
// warp per column, the NEXT column's entries are prefetched into registers while the current one
// is reduced.  Columns longer than 128 entries take an extra (unpipelined) loop.
template <int THREADS, int CTAS>
__global__ void __launch_bounds__(THREADS, CTAS)
    price_ldg(const int *__restrict__ rowIdx, const double *__restrict__ val, const int *__restrict__ colStart,
              const double *__restrict__ rhoG, int m, double *__restrict__ alphaRow, int n)
{
  extern __shared__ __align__(16) unsigned char rawr[];
  double *srho = reinterpret_cast<double *>(rawr);
  for (int i = threadIdx.x; i < m; i += THREADS)
    srho[i] = rhoG[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * (THREADS >> 5) + (threadIdx.x >> 5);
  const int GW = gridDim.x * (THREADS >> 5);
  int j = gw;
  int nb0 = 0, nb1 = 0;
  int ni[4];
  double nv[4];
  auto fetchBounds = [&](int jj) {
    if (jj < n) {
      nb0 = __ldg(colStart + jj);
      nb1 = __ldg(colStart + jj + 1);
    } else {
      nb0 = nb1 = 0;
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
  fetchBounds(j);
  int b0 = nb0, b1 = nb1;
  fetchEntries(b0, b1);
  fetchBounds(j + GW);
  for (; j < n; j += GW) {
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
    fetchEntries(b0, b1);      // next column's entries in flight
    fetchBounds(j + 2 * GW);   // bounds two columns ahead
    double acc0 = cv[0] * srho[ci[0]], acc1 = cv[1] * srho[ci[1]];
    acc0 = fma(cv[2], srho[ci[2]], acc0);
    acc1 = fma(cv[3], srho[ci[3]], acc1);
    for (int e = cb0 + 128 + lane; e < cb1; e += 32) // long columns
      acc0 = fma(__ldg(val + e), srho[__ldg(rowIdx + e)], acc0);
    const double acc = warp_sum(acc0 + acc1);
    if (lane == 0)
      alphaRow[j] = acc;
  }
}

// CTA per row, DEPTH 16-byte loads in flight per thread, x through L1 (NRHS right-hand sides)
template <int NRHS, int DEPTH>
__global__ void __launch_bounds__(256)
    gemv_row(const double *__restrict__ M, int k, int ldk, const double *__restrict__ x, double *__restrict__ out)
{
  __shared__ double part[8][NRHS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int half = ldk >> 1;
  for (int i = blockIdx.x; i < k; i += gridDim.x) {
    const double2 *row = reinterpret_cast<const double2 *>(M + (size_t)i * ldk);
    double acc[NRHS];
#pragma unroll
    for (int c = 0; c < NRHS; c++)
      acc[c] = 0.0;
    for (int j = threadIdx.x; j < half; j += 256 * DEPTH) {
      double2 a[DEPTH];
#pragma unroll
      for (int u = 0; u < DEPTH; u++)
        a[u] = (j + 256 * u < half) ? __ldcs(row + j + 256 * u) : make_double2(0.0, 0.0);
#pragma unroll
      for (int u = 0; u < DEPTH; u++) {
        const int jj = min(j + 256 * u, half - 1);
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
      if (lane == 0)
        part[warp][c] = v;
    }
    __syncthreads();
    if (threadIdx.x < NRHS) {
      double sum = 0.0;
#pragma unroll
      for (int w = 0; w < 8; w++)
        sum += part[w][threadIdx.x];
      out[(size_t)threadIdx.x * ldk + i] = sum;
    }
    __syncthreads();
  }
}
// two rows per CTA
template <int NRHS, int DEPTH>
__global__ void __launch_bounds__(256)
    gemv_row2(const double *__restrict__ M, int k, int ldk, const double *__restrict__ x, double *__restrict__ out)
{
  __shared__ double part[8][2 * NRHS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int half = ldk >> 1;
  const int ngroups = (k + 1) / 2;
  for (int g = blockIdx.x; g < ngroups; g += gridDim.x) {
    const int i0 = g * 2;
    const double2 *row0 = reinterpret_cast<const double2 *>(M + (size_t)i0 * ldk);
    const double2 *row1 = reinterpret_cast<const double2 *>(M + (size_t)min(i0 + 1, k - 1) * ldk);
    double acc[2][NRHS];
#pragma unroll
    for (int c = 0; c < NRHS; c++)
      acc[0][c] = acc[1][c] = 0.0;
    for (int j = threadIdx.x; j < half; j += 256 * DEPTH) {
      double2 a[DEPTH], b[DEPTH];
#pragma unroll
      for (int u = 0; u < DEPTH; u++) {
        const bool p = j + 256 * u < half;
        a[u] = p ? __ldcs(row0 + j + 256 * u) : make_double2(0.0, 0.0);
        b[u] = p ? __ldcs(row1 + j + 256 * u) : make_double2(0.0, 0.0);
      }
#pragma unroll
      for (int u = 0; u < DEPTH; u++) {
        const int jj = min(j + 256 * u, half - 1);
#pragma unroll
        for (int c = 0; c < NRHS; c++) {
          const double2 xv = __ldg(reinterpret_cast<const double2 *>(x + (size_t)c * ldk) + jj);
          acc[0][c] = fma(a[u].x, xv.x, acc[0][c]);
          acc[0][c] = fma(a[u].y, xv.y, acc[0][c]);
          acc[1][c] = fma(b[u].x, xv.x, acc[1][c]);
          acc[1][c] = fma(b[u].y, xv.y, acc[1][c]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 2; r++)
#pragma unroll
      for (int c = 0; c < NRHS; c++) {
        const double v = warp_sum(acc[r][c]);
        if (lane == 0)
          part[warp][r * NRHS + c] = v;
      }
    __syncthreads();
    if (threadIdx.x < 2 * NRHS) {
      double sum = 0.0;
#pragma unroll
      for (int w = 0; w < 8; w++)
        sum += part[w][threadIdx.x];
      const int r = threadIdx.x / NRHS, c = threadIdx.x % NRHS;
      if (i0 + r < k)
        out[(size_t)c * ldk + i0 + r] = sum;
    }
    __syncthreads();
  }
}


// ---- eta panel apply: x_c[p] -= sum_{i<t} W[p][i] * mu_c[i], W row-major m x tmax (round-2 candidates)
template <int NRHS, int DEPTH>
__global__ void __launch_bounds__(256) panel_warp8(const double *__restrict__ W, int m, int tmax, int t,
                                                   const double *__restrict__ mu, double *__restrict__ x)
{
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int p = blockIdx.x * wpb + (threadIdx.x >> 5); p < m; p += gridDim.x * wpb) {
    const double *wrow = W + (size_t)p * tmax;
    double acc[NRHS];
#pragma unroll
    for (int c = 0; c < NRHS; c++) acc[c] = 0.0;
    for (int i = lane; i < t; i += 32 * DEPTH) {
      double w[DEPTH];
#pragma unroll
      for (int u = 0; u < DEPTH; u++) w[u] = (i + 32 * u < t) ? __ldcs(wrow + i + 32 * u) : 0.0;
#pragma unroll
      for (int u = 0; u < DEPTH; u++) {
        const int ii = min(i + 32 * u, t - 1);
#pragma unroll
        for (int c = 0; c < NRHS; c++) acc[c] = fma(w[u], __ldg(mu + (size_t)c * tmax + ii), acc[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < NRHS; c++) acc[c] = warp_sum(acc[c]);
    if (lane == 0)
      for (int c = 0; c < NRHS; c++) x[(size_t)c * m + p] -= acc[c];
  }
}
// same with 16-byte loads and mu staged in shared memory
template <int NRHS, int DEPTH>
__global__ void __launch_bounds__(256) panel_warp16_smem(const double *__restrict__ W, int m, int tmax, int t,
                                                         const double *__restrict__ mu, double *__restrict__ x)
{
  extern __shared__ __align__(16) unsigned char rawmu[];
  double *smu = reinterpret_cast<double *>(rawmu); // [NRHS][tpad]
  const int tpad = (t + 1) & ~1;
  for (int i = threadIdx.x; i < tpad; i += blockDim.x)
#pragma unroll
    for (int c = 0; c < NRHS; c++) smu[c * tpad + i] = i < t ? mu[(size_t)c * tmax + i] : 0.0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const int half = tpad >> 1;
  for (int p = blockIdx.x * wpb + (threadIdx.x >> 5); p < m; p += gridDim.x * wpb) {
    const double2 *wrow = reinterpret_cast<const double2 *>(W + (size_t)p * tmax);
    double acc[NRHS];
#pragma unroll
    for (int c = 0; c < NRHS; c++) acc[c] = 0.0;
    for (int i = lane; i < half; i += 32 * DEPTH) {
      double2 w[DEPTH];
#pragma unroll
      for (int u = 0; u < DEPTH; u++) w[u] = (i + 32 * u < half) ? __ldcs(wrow + i + 32 * u) : make_double2(0.0, 0.0);
#pragma unroll
      for (int u = 0; u < DEPTH; u++) {
        const int ii = min(i + 32 * u, half - 1);
#pragma unroll
        for (int c = 0; c < NRHS; c++) {
          const double2 mv = reinterpret_cast<const double2 *>(smu + c * tpad)[ii];
          acc[c] = fma(w[u].x, mv.x, acc[c]);
          acc[c] = fma((2 * ii + 1 < t) ? w[u].y : 0.0, mv.y, acc[c]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < NRHS; c++) acc[c] = warp_sum(acc[c]);
    if (lane == 0)
      for (int c = 0; c < NRHS; c++) x[(size_t)c * m + p] -= acc[c];
  }
}

// naive reference: warp per column
__global__ void price_ref(const int *__restrict__ rowIdx, const double *__restrict__ val, const int *__restrict__ colStart,
                          const double *__restrict__ rho, int n, double *__restrict__ alpha)
{
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (j >= n)
    return;
  double acc = 0.0;
  for (int e = colStart[j] + lane; e < colStart[j + 1]; e += 32)
    acc = fma(val[e], rho[rowIdx[e]], acc);
  acc = warp_sum(acc);
  if (lane == 0)
    alpha[j] = acc;
}

// =================================================================== DGEMM  C -= A*B (column major)
__global__ void __launch_bounds__(256)
    gemm_sub_simt(double *__restrict__ C, int ldc, const double *__restrict__ A, int lda, const double *__restrict__ B,
                  int ldb, int M, int N, int K)
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

__device__ __forceinline__ void dmma(double &d0, double &d1, double a, double b)
{
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(d0), "+d"(d1)
               : "d"(a), "d"(b));
}

// 128x128 tile per CTA, 8 warps as 2 (M) x 4 (N), warp tile 64x32 = 8x4 mma tiles, K chunks of 32
constexpr int kLdA = 132, kLdB = 36;
__global__ void __launch_bounds__(256)
    gemm_sub_dmma(double *__restrict__ C, int ldc, const double *__restrict__ A, int lda, const double *__restrict__ B,
                  int ldb, int M, int N, int K)
{
  extern __shared__ __align__(16) double sm[];
  double *As = sm;              // [32][kLdA]  As[kk][i]
  double *Bs = sm + 32 * kLdA;  // [128][kLdB] Bs[j][kk]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp & 1, wn = warp >> 1;
  const int m0 = blockIdx.x * 128, n0 = blockIdx.y * 128;
  const int g = lane >> 2, t4 = lane & 3;
  double acc[8][4][2];
#pragma unroll
  for (int a = 0; a < 8; a++)
#pragma unroll
    for (int b = 0; b < 4; b++)
      acc[a][b][0] = acc[a][b][1] = 0.0;
  for (int k0 = 0; k0 < K; k0 += 32) {
    for (int e = tid; e < 128 * 32; e += 256) {
      const int i = e & 127, kk = e >> 7;
      const int gi = m0 + i, gk = k0 + kk;
      As[kk * kLdA + i] = (gi < M && gk < K) ? A[(size_t)gk * lda + gi] : 0.0;
    }
    for (int e = tid; e < 128 * 32; e += 256) {
      const int kk = e & 31, j = e >> 5;
      const int gk = k0 + kk, gj = n0 + j;
      Bs[j * kLdB + kk] = (gk < K && gj < N) ? B[(size_t)gj * ldb + gk] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < 8; ks++) {
      double a[8], b[4];
#pragma unroll
      for (int mt = 0; mt < 8; mt++)
        a[mt] = As[(ks * 4 + t4) * kLdA + wm * 64 + mt * 8 + g];
#pragma unroll
      for (int nt = 0; nt < 4; nt++)
        b[nt] = Bs[(wn * 32 + nt * 8 + g) * kLdB + ks * 4 + t4];
#pragma unroll
      for (int mt = 0; mt < 8; mt++)
#pragma unroll
        for (int nt = 0; nt < 4; nt++)
          dmma(acc[mt][nt][0], acc[mt][nt][1], a[mt], b[nt]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int mt = 0; mt < 8; mt++) {
    const int gi = m0 + wm * 64 + mt * 8 + g;
    if (gi >= M)
      continue;
#pragma unroll
    for (int nt = 0; nt < 4; nt++) {
      const int gj = n0 + wn * 32 + nt * 8 + t4 * 2;
      if (gj < N)
        C[(size_t)gj * ldc + gi] -= acc[mt][nt][0];
      if (gj + 1 < N)
        C[(size_t)(gj + 1) * ldc + gi] -= acc[mt][nt][1];
    }
  }
}

template <class F> float timeit(F f, int reps = 12)
{
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  f();
  CK(cudaDeviceSynchronize());
  float best = 1e30f, sum = 0;
  for (int r = 0; r < reps; r++) {
    cudaEventRecord(a);
    f();
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    best = std::min(best, ms);
    sum += ms;
  }
  CK(cudaGetLastError());
  (void)sum;
  return best;
}

static double maxdiff(const std::vector<double> &a, const std::vector<double> &b, size_t n)
{
  double d = 0, s = 0;
  for (size_t i = 0; i < n; i++) {
    d = std::max(d, std::fabs(a[i] - b[i]));
    s = std::max(s, std::fabs(b[i]));
  }
  return d / (s > 0 ? s : 1);
}

int main(int argc, char **argv)
{
  const int which = argc > 1 ? atoi(argv[1]) : 7;
  std::mt19937_64 rng(12345);
  std::uniform_real_distribution<double> U(-1.0, 1.0);
  // ------------------------------------------------------------------ GEMV
  if (which & 1) {
    for (int k : {4682, 5787}) {
      const int ldk = (k + 7) / 8 * 8, m = 10000;
      const int NW = 4; // rotate over 4 copies (> L2)
      double *M, *b, *x3, *out, *part, *ref;
      int *gather;
      unsigned int *ticket;
      CK(cudaMalloc(&M, sizeof(double) * (size_t)NW * k * ldk));
      CK(cudaMalloc(&b, sizeof(double) * 3 * m));
      CK(cudaMalloc(&x3, sizeof(double) * 3 * ldk));
      CK(cudaMalloc(&out, sizeof(double) * 3 * ldk));
      CK(cudaMalloc(&ref, sizeof(double) * 3 * ldk));
      CK(cudaMalloc(&part, sizeof(double) * 8 * 3 * ldk));
      CK(cudaMalloc(&gather, sizeof(int) * ldk));
      CK(cudaMalloc(&ticket, sizeof(unsigned) * ldk));
      CK(cudaMemset(ticket, 0, sizeof(unsigned) * ldk));
      std::vector<double> hM((size_t)k * ldk, 0.0), hb(3 * m), hx(3 * (size_t)ldk, 0.0);
      for (int i = 0; i < k; i++)
        for (int j = 0; j < k; j++)
          hM[(size_t)i * ldk + j] = U(rng);
      for (auto &v : hb)
        v = U(rng);
      std::vector<int> hg(ldk, 0);
      for (int j = 0; j < k; j++)
        hg[j] = (int)(((long)j * 7919) % m);
      for (int c = 0; c < 3; c++)
        for (int j = 0; j < k; j++)
          hx[(size_t)c * ldk + j] = hb[(size_t)c * m + hg[j]];
      for (int w = 0; w < NW; w++)
        CK(cudaMemcpy(M + (size_t)w * k * ldk, hM.data(), sizeof(double) * (size_t)k * ldk, cudaMemcpyHostToDevice));
      CK(cudaMemcpy(b, hb.data(), sizeof(double) * 3 * m, cudaMemcpyHostToDevice));
      CK(cudaMemcpy(x3, hx.data(), sizeof(double) * 3 * ldk, cudaMemcpyHostToDevice));
      CK(cudaMemcpy(gather, hg.data(), sizeof(int) * ldk, cudaMemcpyHostToDevice));
      const double bytes = 8.0 * k * ldk;
      int win = 0;
      auto Mw = [&]() { win = (win + 1) % NW; return M + (size_t)win * k * ldk; };
      std::vector<double> hr(3 * (size_t)ldk), ho(3 * (size_t)ldk);
      gemv_cur<3><<<1184, 256>>>(M, k, ldk, x3, ref);
      CK(cudaMemcpy(hr.data(), ref, sizeof(double) * 3 * ldk, cudaMemcpyDeviceToHost));
      auto report = [&](const char *name, float ms, int nrhs) {
        CK(cudaMemcpy(ho.data(), out, sizeof(double) * 3 * ldk, cudaMemcpyDeviceToHost));
        double d = 0;
        for (int c = 0; c < nrhs; c++) {
          std::vector<double> a(ho.begin() + (size_t)c * ldk, ho.begin() + (size_t)c * ldk + k);
          std::vector<double> r(hr.begin() + (size_t)c * ldk, hr.begin() + (size_t)c * ldk + k);
          d = std::max(d, maxdiff(a, r, k));
        }
        printf("k=%d %-46s %7.1f us  %7.1f GB/s  relerr %.1e\n", k, name, ms * 1000, bytes / ms / 1e6, d);
      };
      for (int grid : {8 * numSms(), 10 * numSms(), 16 * numSms()}) {
        char nm[96];
        CK(cudaMemset(out, 0, sizeof(double) * 3 * ldk));
        float t1 = timeit([&] { gemv_cur<1><<<grid, 256>>>(Mw(), k, ldk, x3, out); });
        snprintf(nm, 96, "cur<1> grid %d", grid);
        report(nm, t1, 1);
        float t3 = timeit([&] { gemv_cur<3><<<grid, 256>>>(Mw(), k, ldk, x3, out); });
        snprintf(nm, 96, "cur<3> grid %d", grid);
        report(nm, t3, 3);
      }
      if (which & 16) {
        for (int grid : {592, 1184, 2368}) {
          char nm[96];
#define RUN_ROW(KERN, LABEL, NR)                                                                   \
  do {                                                                                             \
    CK(cudaMemset(out, 0, sizeof(double) * 3 * ldk));                                              \
    float t = timeit([&] { KERN<<<grid, 256>>>(Mw(), k, ldk, x3, out); });                         \
    snprintf(nm, 96, LABEL " grid %d", grid);                                                      \
    report(nm, t, NR);                                                                             \
  } while (0)
          RUN_ROW((gemv_row<1, 4>), "row<1,D4>", 1);
          RUN_ROW((gemv_row<1, 8>), "row<1,D8>", 1);
          RUN_ROW((gemv_row<3, 4>), "row<3,D4>", 3);
          RUN_ROW((gemv_row<3, 8>), "row<3,D8>", 3);
          RUN_ROW((gemv_row2<1, 4>), "row2<1,D4>", 1);
          RUN_ROW((gemv_row2<3, 2>), "row2<3,D2>", 3);
          RUN_ROW((gemv_row2<3, 4>), "row2<3,D4>", 3);
        }
      }
      auto runItems = [&](auto kern, const char *name, int nrhs, int threads, int Q) {
        const int half = ldk / 2;
        int seg2 = ((half + Q - 1) / Q + 31) / 32 * 32;
        size_t sm = sizeof(double) * (size_t)nrhs * ldk;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        CK(cudaMemset(out, 0, sizeof(double) * 3 * ldk));
        float t = timeit([&] {
          kern<<<numSms(), threads, sm>>>(Mw(), k, ldk, b, m, gather, part, ticket, out, ldk, nullptr, Q, seg2);
        });
        char nm[96];
        snprintf(nm, 96, "%s Q=%d", name, Q);
        report(nm, t, nrhs);
      };
      for (int Q : {1, 2, 4, 8}) {
        runItems(gemv_items<1, 8, 1024>, "items<1,D8,1024>", 1, 1024, Q);
        runItems(gemv_items<3, 8, 1024>, "items<3,D8,1024>", 3, 1024, Q);
      }
      runItems(gemv_items<1, 4, 1024>, "items<1,D4,1024>", 1, 1024, 4);
      runItems(gemv_items<3, 4, 1024>, "items<3,D4,1024>", 3, 1024, 4);
      runItems(gemv_items<1, 16, 512>, "items<1,D16,512>", 1, 512, 4);
      runItems(gemv_items<3, 16, 512>, "items<3,D16,512>", 3, 512, 4);
      runItems(gemv_items<3, 12, 768>, "items<3,D12,768>", 3, 768, 4);
      cudaFree(M); cudaFree(b); cudaFree(x3); cudaFree(out); cudaFree(ref); cudaFree(part); cudaFree(gather); cudaFree(ticket);
    }
  }
  // ------------------------------------------------------------------ PRICE
  if (which & 2) {
    const int m = 10000, n = 100000;
    std::vector<int> cs(n + 1 + 16, 0);
    std::vector<int> ri;
    std::vector<double> va;
    ri.reserve(10200000);
    va.reserve(10200000);
    std::binomial_distribution<int> Bn(m, 0.01);
    std::vector<char> mark(m, 0);
    for (int j = 0; j < n; j++) {
      int cnt = std::max(1, Bn(rng));
      std::vector<int> rows;
      while ((int)rows.size() < cnt) {
        int r = (int)(rng() % m);
        if (!mark[r]) {
          mark[r] = 1;
          rows.push_back(r);
        }
      }
      std::sort(rows.begin(), rows.end());
      for (int r : rows) {
        mark[r] = 0;
        ri.push_back(r);
        va.push_back(U(rng));
      }
      cs[j + 1] = (int)ri.size();
    }
    const long nnz = ri.size();
    for (int q = n + 1; q < n + 1 + 16; q++)
      cs[q] = (int)nnz;
    printf("price matrix: m=%d n=%d nnz=%ld\n", m, n, nnz);
    const int NW = 4;
    const long pad = 64;
    const long stride = (nnz + pad + 63) / 64 * 64;
    int *dIdx, *dCs;
    unsigned short *dIdx16;
    double *dVal, *dRho, *dAlpha, *dRef;
    CK(cudaMalloc(&dIdx, sizeof(int) * stride * NW));
    CK(cudaMalloc(&dIdx16, sizeof(unsigned short) * stride * NW));
    CK(cudaMalloc(&dVal, sizeof(double) * stride * NW));
    CK(cudaMalloc(&dCs, sizeof(int) * (n + 17)));
    CK(cudaMalloc(&dRho, sizeof(double) * m));
    CK(cudaMalloc(&dAlpha, sizeof(double) * n));
    CK(cudaMalloc(&dRef, sizeof(double) * n));
    CK(cudaMemset(dIdx, 0, sizeof(int) * stride * NW));
    CK(cudaMemset(dIdx16, 0, sizeof(unsigned short) * stride * NW));
    CK(cudaMemset(dVal, 0, sizeof(double) * stride * NW));
    std::vector<unsigned short> ri16(ri.begin(), ri.end());
    std::vector<double> rho(m);
    for (auto &v : rho)
      v = U(rng);
    for (int w = 0; w < NW; w++) {
      CK(cudaMemcpy(dIdx + w * stride, ri.data(), sizeof(int) * nnz, cudaMemcpyHostToDevice));
      CK(cudaMemcpy(dIdx16 + w * stride, ri16.data(), sizeof(unsigned short) * nnz, cudaMemcpyHostToDevice));
      CK(cudaMemcpy(dVal + w * stride, va.data(), sizeof(double) * nnz, cudaMemcpyHostToDevice));
    }
    CK(cudaMemcpy(dCs, cs.data(), sizeof(int) * (n + 17), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(dRho, rho.data(), sizeof(double) * m, cudaMemcpyHostToDevice));
    price_ref<<<(n + 7) / 8, 256>>>(dIdx, dVal, dCs, dRho, n, dRef);
    std::vector<double> href(n), hout(n);
    CK(cudaMemcpy(href.data(), dRef, sizeof(double) * n, cudaMemcpyDeviceToHost));
    int win = 0;
    auto report = [&](const char *name, float ms, double bytesPerNz) {
      CK(cudaMemcpy(hout.data(), dAlpha, sizeof(double) * n, cudaMemcpyDeviceToHost));
      printf("%-52s %7.1f us  %7.1f GB/s moved  (%.1f GB/s at 12 B/nz)  relerr %.1e\n", name, ms * 1000,
             bytesPerNz * nnz / ms / 1e6, 12.0 * nnz / ms / 1e6, maxdiff(hout, href, n));
    };
    { // current kernel
      std::vector<int> tiles;
      int c = 0;
      while (c < n) {
        tiles.push_back(c);
        const int ea = cs[c] & ~3;
        int c1 = c;
        while (c1 < n && c1 - c < 8 && ((cs[c1 + 1] + 3) & ~3) - ea <= kPriceTile)
          c1++;
        if (c1 == c) { printf("column too long\n"); return 1; }
        c = c1;
      }
      tiles.push_back(n);
      const int ntl = (int)tiles.size() - 1;
      std::vector<int> desc((size_t)ntl * 4);
      for (int t = 0; t < ntl; t++) {
        const int t0 = tiles[t], t1 = tiles[t + 1];
        const int ea = cs[t0] & ~3;
        desc[4 * t + 0] = t0; desc[4 * t + 1] = t1 - t0; desc[4 * t + 2] = ea; desc[4 * t + 3] = ((cs[t1] + 3) & ~3) - ea;
      }
      int4 *dDesc;
      CK(cudaMalloc(&dDesc, sizeof(int) * desc.size()));
      CK(cudaMemcpy(dDesc, desc.data(), sizeof(int) * desc.size(), cudaMemcpyHostToDevice));
      const int pipes = numSms() * kPriceGroups;
      const int descCap = ((ntl + pipes - 1) / pipes + 7) / 8 * 8;
      const size_t smem = 128 + (size_t)kPriceGroups * descCap * 16 + (size_t)kPriceGroups * kPriceStages * kPriceTileAlloc * 12 + sizeof(double) * m;
      CK(cudaFuncSetAttribute(price_cur, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      CK(cudaMemset(dAlpha, 0, sizeof(double) * n));
      float t = timeit([&] {
        win = (win + 1) % NW;
        price_cur<<<numSms(), 1024, smem>>>(dIdx + win * stride, dVal + win * stride, dCs, dRho, m, dAlpha, dDesc, ntl, descCap);
      });
      char nm[96];
      snprintf(nm, 96, "price_cur 4x2x1024 (%d tiles, smem %zu)", ntl, smem);
      report(nm, t, 12.0);
      cudaFree(dDesc);
    }
#define RUN_BIG(EE, SS, IDXT, SR, IDXPTR)                                                                         \
  do {                                                                                                            \
    const int E = EE, S = SS;                                                                                     \
    std::vector<int> desc;                                                                                        \
    int c = 0, ntl = 0;                                                                                           \
    bool ok = true;                                                                                               \
    while (c < n) {                                                                                               \
      const int ea = cs[c] & ~7;                                                                                  \
      int c1 = c;                                                                                                 \
      while (c1 < n && c1 - c < MAXC) {                                                                           \
        int c2 = std::min(n, c1 + 4);                                                                             \
        if (((cs[c2] + 7) & ~7) - ea > E)                                                                         \
          break;                                                                                                  \
        c1 = c2;                                                                                                  \
      }                                                                                                           \
      if (c1 == c) { ok = false; break; }                                                                         \
      desc.push_back(c); desc.push_back(c1 - c); desc.push_back(ea); desc.push_back(((cs[c1] + 7) & ~7) - ea);    \
      c = c1;                                                                                                     \
      ntl++;                                                                                                      \
    }                                                                                                             \
    const int descCap = ((ntl + numSms() - 1) / numSms() + 7) / 8 * 8;                                                          \
    const size_t smem = 128 + (size_t)descCap * 16 + (size_t)S * (MAXC + 8) * 4 + (size_t)S * E * (8 + sizeof(IDXT)) + (SR ? sizeof(double) * m : 0); \
    char nm[128];                                                                                                 \
    snprintf(nm, 128, "price_big E=%d S=%d idx%zu rho:%s (%d tiles, smem %zu)", E, S, sizeof(IDXT) * 8, SR ? "smem" : "ldg", ntl, smem); \
    if (!ok || smem > 227 * 1024) { printf("%s: skipped\n", nm); break; }                                          \
    int4 *dDesc;                                                                                                  \
    CK(cudaMalloc(&dDesc, sizeof(int) * desc.size()));                                                            \
    CK(cudaMemcpy(dDesc, desc.data(), sizeof(int) * desc.size(), cudaMemcpyHostToDevice));                        \
    CK(cudaFuncSetAttribute(price_big<EE, SS, IDXT, SR>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); \
    CK(cudaMemset(dAlpha, 0, sizeof(double) * n));                                                                \
    float t = timeit([&] {                                                                                        \
      win = (win + 1) % NW;                                                                                       \
      price_big<EE, SS, IDXT, SR><<<numSms(), 1024, smem>>>(IDXPTR + win * stride, dVal + win * stride, dCs, dRho, m, dAlpha, dDesc, ntl, descCap); \
    });                                                                                                           \
    report(nm, t, 8.0 + sizeof(IDXT));                                                                            \
    cudaFree(dDesc);                                                                                              \
  } while (0)
#define RUN_V3(EE, SS, IDXT, LPCV, THR, MAXCOLS, IDXPTR)                                                          \
  do {                                                                                                            \
    const int E = EE, S = SS;                                                                                     \
    std::vector<int> desc;                                                                                        \
    int c = 0, ntl = 0;                                                                                           \
    bool ok = true;                                                                                               \
    while (c < n) {                                                                                               \
      const int ea = cs[c] & ~7;                                                                                  \
      int c1 = c;                                                                                                 \
      while (c1 < n && c1 - c < MAXCOLS) {                                                                        \
        int c2 = std::min(n, c1 + 4);                                                                             \
        if (((cs[c2] + 7) & ~7) - ea > E)                                                                         \
          break;                                                                                                  \
        c1 = c2;                                                                                                  \
      }                                                                                                           \
      if (c1 == c) { ok = false; break; }                                                                         \
      desc.push_back(c); desc.push_back(c1 - c); desc.push_back(ea); desc.push_back(((cs[c1] + 7) & ~7) - ea);    \
      c = c1;                                                                                                     \
      ntl++;                                                                                                      \
    }                                                                                                             \
    const int descCap = ((ntl + numSms() - 1) / numSms() + 7) / 8 * 8;                                                          \
    const size_t smem = 128 + (size_t)descCap * 16 + (size_t)S * (MAXC + 8) * 4 + (size_t)S * E * (8 + sizeof(IDXT)) + sizeof(double) * m; \
    char nm[160];                                                                                                 \
    snprintf(nm, 160, "price_v3 E=%d S=%d idx%zu lpc=%d thr=%d maxc=%d (%d tiles, smem %zu)", E, S, sizeof(IDXT) * 8, LPCV, THR, MAXCOLS, ntl, smem); \
    if (!ok || smem > 227 * 1024) { printf("%s: skipped\n", nm); break; }                                          \
    int4 *dDesc;                                                                                                  \
    CK(cudaMalloc(&dDesc, sizeof(int) * desc.size()));                                                            \
    CK(cudaMemcpy(dDesc, desc.data(), sizeof(int) * desc.size(), cudaMemcpyHostToDevice));                        \
    CK(cudaFuncSetAttribute(price_v3<EE, SS, IDXT, LPCV, THR>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); \
    CK(cudaMemset(dAlpha, 0, sizeof(double) * n));                                                                \
    float t = timeit([&] {                                                                                        \
      win = (win + 1) % NW;                                                                                       \
      price_v3<EE, SS, IDXT, LPCV, THR><<<numSms(), THR, smem>>>(IDXPTR + win * stride, dVal + win * stride, dCs, dRho, m, dAlpha, dDesc, ntl, descCap); \
    });                                                                                                           \
    report(nm, t, 8.0 + sizeof(IDXT));                                                                            \
    cudaFree(dDesc);                                                                                              \
  } while (0)
    if (which & 32) {
#define RUN_LDG(THR, CT)                                                                           \
  do {                                                                                             \
    CK(cudaFuncSetAttribute(price_ldg<THR, CT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(double) * m)); \
    CK(cudaMemset(dAlpha, 0, sizeof(double) * n));                                                 \
    float t = timeit([&] {                                                                         \
      win = (win + 1) % NW;                                                                        \
      price_ldg<THR, CT><<<numSms() * CT, THR, sizeof(double) * m>>>(dIdx + win * stride, dVal + win * stride, dCs, dRho, m, dAlpha, n); \
    });                                                                                            \
    char nm[96];                                                                                   \
    snprintf(nm, 96, "price_ldg thr=%d ctas/SM=%d", THR, CT);                                      \
    report(nm, t, 12.0);                                                                           \
  } while (0)
      RUN_LDG(768, 2);
      RUN_LDG(1024, 2);
      RUN_LDG(512, 2);
      RUN_LDG(1024, 1);
      RUN_LDG(640, 2);
    }
    if (which & 8) {
    RUN_V3(2816, 4, int, 8, 256, 32, dIdx);
    RUN_V3(2816, 4, int, 16, 256, 32, dIdx);
    RUN_V3(2816, 4, int, 8, 512, 64, dIdx);
    RUN_V3(2816, 4, int, 16, 512, 32, dIdx);
    RUN_V3(2816, 4, int, 4, 256, 64, dIdx);
    RUN_V3(3584, 3, int, 8, 256, 32, dIdx);
    RUN_V3(2048, 5, int, 8, 256, 32, dIdx);
    RUN_V3(1792, 6, int, 8, 256, 16, dIdx);
    RUN_V3(3328, 4, unsigned short, 8, 256, 32, dIdx16);
    RUN_V3(3328, 4, unsigned short, 16, 256, 32, dIdx16);
    RUN_V3(2816, 4, int, 8, 1024, 64, dIdx);
    }
    RUN_BIG(2816, 4, int, true, dIdx);
    RUN_BIG(2048, 5, int, true, dIdx);
    RUN_BIG(1536, 7, int, true, dIdx);
    RUN_BIG(3584, 3, int, true, dIdx);
    RUN_BIG(1024, 11, int, true, dIdx);
    RUN_BIG(3328, 4, unsigned short, true, dIdx16);
    RUN_BIG(2048, 6, unsigned short, true, dIdx16);
    RUN_BIG(1536, 9, unsigned short, true, dIdx16);
    RUN_BIG(4096, 4, int, false, dIdx);
    RUN_BIG(3072, 6, int, false, dIdx);
    RUN_BIG(3072, 7, unsigned short, false, dIdx16);
  }

  // ------------------------------------------------------------------ eta panel apply (round-2 candidates)
  if (which & 64) {
    const int m = 10000, tmax = 2048, NW = 4;
    double *W, *mu, *x;
    CK(cudaMalloc(&W, sizeof(double) * (size_t)NW * m * tmax));
    CK(cudaMalloc(&mu, sizeof(double) * 3 * tmax));
    CK(cudaMalloc(&x, sizeof(double) * 3 * m));
    std::vector<double> hW((size_t)m * tmax), hmu(3 * tmax);
    for (auto &v : hW) v = U(rng);
    for (auto &v : hmu) v = U(rng);
    for (int w = 0; w < NW; w++)
      CK(cudaMemcpy(W + (size_t)w * m * tmax, hW.data(), sizeof(double) * hW.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(mu, hmu.data(), sizeof(double) * hmu.size(), cudaMemcpyHostToDevice));
    int win = 0;
    auto Ww = [&]() { win = (win + 1) % NW; return W + (size_t)win * m * tmax; };
    for (int t : {500, 1000, 2000}) {
      const double bytes = 8.0 * m * t;
      std::vector<double> ref(3 * m), got(3 * m);
      auto check = [&](const char *name, float ms) {
        CK(cudaMemset(x, 0, sizeof(double) * 3 * m));
        return ms;
      };
      (void)check;
      auto run = [&](const char *name, auto launch) {
        CK(cudaMemset(x, 0, sizeof(double) * 3 * m));
        launch();
        CK(cudaMemcpy(got.data(), x, sizeof(double) * 3 * m, cudaMemcpyDeviceToHost));
        double d = 0, sc = 0;
        for (int p = 0; p < 3 * m; p += 997) {
          const int c = p / m, pp = p % m;
          double r = 0;
          for (int i = 0; i < t; i++) r -= hW[(size_t)pp * tmax + i] * hmu[(size_t)c * tmax + i];
          d = std::max(d, std::fabs(r - got[p]));
          sc = std::max(sc, std::fabs(r));
        }
        float ms = timeit(launch);
        printf("t=%4d %-40s %7.1f us  %7.1f GB/s  relerr %.1e\n", t, name, ms * 1000, bytes / ms / 1e6, d / (sc > 0 ? sc : 1));
      };
      run("panel_warp8<3,8> grid 1184", [&] { panel_warp8<3, 8><<<1184, 256>>>(Ww(), m, tmax, t, mu, x); });
      run("panel_warp8<3,4> grid 1184", [&] { panel_warp8<3, 4><<<1184, 256>>>(Ww(), m, tmax, t, mu, x); });
      run("panel_warp8<3,8> grid 1250", [&] { panel_warp8<3, 8><<<1250, 256>>>(Ww(), m, tmax, t, mu, x); });
      const size_t sm = sizeof(double) * 3 * ((t + 1) & ~1);
      CK(cudaFuncSetAttribute(panel_warp16_smem<3, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
      CK(cudaFuncSetAttribute(panel_warp16_smem<3, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
      run("panel_warp16_smem<3,4> grid 592", [&] { panel_warp16_smem<3, 4><<<592, 256, sm>>>(Ww(), m, tmax, t, mu, x); });
      run("panel_warp16_smem<3,4> grid 1184", [&] { panel_warp16_smem<3, 4><<<1184, 256, sm>>>(Ww(), m, tmax, t, mu, x); });
      run("panel_warp16_smem<3,8> grid 592", [&] { panel_warp16_smem<3, 8><<<592, 256, sm>>>(Ww(), m, tmax, t, mu, x); });
    }
    cudaFree(W); cudaFree(mu); cudaFree(x);
  }
  // ------------------------------------------------------------------ DGEMM
  if (which & 4) {
    const int Mx = 4096, K = 32, ld = 4104;
    double *C, *C2, *A, *B;
    CK(cudaMalloc(&C, sizeof(double) * (size_t)ld * Mx));
    CK(cudaMalloc(&C2, sizeof(double) * (size_t)ld * Mx));
    CK(cudaMalloc(&A, sizeof(double) * (size_t)ld * 128));
    CK(cudaMalloc(&B, sizeof(double) * (size_t)ld * Mx));
    std::vector<double> hC((size_t)ld * Mx), hA((size_t)ld * 128), hB((size_t)ld * Mx);
    for (auto &v : hC) v = U(rng);
    for (auto &v : hA) v = U(rng);
    for (auto &v : hB) v = U(rng);
    CK(cudaMemcpy(A, hA.data(), sizeof(double) * hA.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(B, hB.data(), sizeof(double) * hB.size(), cudaMemcpyHostToDevice));
    CK(cudaFuncSetAttribute(gemm_sub_dmma, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(double) * (32 * kLdA + 128 * kLdB)));
    const size_t smem = sizeof(double) * (32 * kLdA + 128 * kLdB);
    for (int Kk : {32, 64, 128}) {
      for (int Msz : {4096, 4000, 1000}) {
        const int Nsz = Msz - 3;
        CK(cudaMemcpy(C, hC.data(), sizeof(double) * hC.size(), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(C2, hC.data(), sizeof(double) * hC.size(), cudaMemcpyHostToDevice));
        dim3 g1((Msz + 63) / 64, (Nsz + 63) / 64), g2((Msz + 127) / 128, (Nsz + 127) / 128);
        gemm_sub_simt<<<g1, 256>>>(C, ld, A, ld, B, ld, Msz, Nsz, Kk);
        gemm_sub_dmma<<<g2, 256, smem>>>(C2, ld, A, ld, B, ld, Msz, Nsz, Kk);
        std::vector<double> r1(hC.size()), r2(hC.size());
        CK(cudaMemcpy(r1.data(), C, sizeof(double) * hC.size(), cudaMemcpyDeviceToHost));
        CK(cudaMemcpy(r2.data(), C2, sizeof(double) * hC.size(), cudaMemcpyDeviceToHost));
        const double d = maxdiff(r2, r1, r1.size());
        float t1 = timeit([&] { gemm_sub_simt<<<g1, 256>>>(C, ld, A, ld, B, ld, Msz, Nsz, Kk); }, 5);
        float t2 = timeit([&] { gemm_sub_dmma<<<g2, 256, smem>>>(C2, ld, A, ld, B, ld, Msz, Nsz, Kk); }, 5);
        const double fl = 2.0 * Msz * Nsz * Kk;
        printf("gemm M=%d N=%d K=%d : simt %7.1f us %6.2f TF/s | dmma %7.1f us %6.2f TF/s | relerr %.1e\n", Msz, Nsz, Kk,
               t1 * 1000, fl / t1 / 1e9, t2 * 1000, fl / t2 / 1e9, d);
      }
    }
    (void)K;
  }
  return 0;
}
