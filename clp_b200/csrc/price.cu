// price.cu -- PRICE (tableau row) and CHUZC (bound-flipping ratio test), device resident.
//
// Replaces ClpPackedMatrix::transposeTimes (/root/reference/src/ClpPackedMatrix.cpp:706 ->
// transposeTimesByColumn :961 -> gutsOfTransposeTimesUnscaled :1640/:1799, the variant that
// skips basic columns by status and fuses the first pass of the ratio test) and
// ClpSimplexDual::dualColumn0 / dualColumn (src/ClpSimplexDual.cpp:3665 / :4192).
//
// PRICE streams the CSC copy of A once (12 B per nonzero) with one warp per column; rho is
// gathered through L1/L2.  Fused into the same pass: every ratio-test candidate adds its
// slope contribution |alpha_j|*(u_j-l_j) to a histogram over the (monotone) bit pattern of its
// ratio d_j/|alpha_j| -- in 2^-40 fixed point relative to the primal infeasibility, with
// integer atomics, so the result does not depend on the order of the atomics.
//
// CHUZC then needs no sort: a single CTA scans the 32768-bucket histogram for the bucket in
// which the slope of the dual objective is exhausted (theta*), one pass computes the Harris
// bound beyond theta* (atomicMin) and one pass picks the largest |alpha| inside
// [theta*, harris] (atomicMax on a packed (|alpha|,sequence) key).  Candidates with a ratio
// below theta* are "passed": the dual update flips them to their other bound (BFRT).
#include "kernels_common.cuh"

namespace clpb {

__device__ __forceinline__ void histogram_add(const DeviceModel &d, double a, double dtil,
                                              bool boxed, double range, double infeas)
{
  atomicAdd(d.histWeight + hist1_slot(ratio_bucket(dtil / a)), slope_weight(a, boxed, range, infeas));
}

// alphaRow[j] = rho^T a_j (raw dot product) for the nonbasic, non-fixed columns j of
// [colBegin,colEnd); basic / fixed columns get 0 without touching their entries.
// One warp per column, the matrix goes from HBM straight into registers: while a column is being
// reduced the NEXT column of the warp (4 x 32 entries: 4-byte row indices + 8-byte values) is
// already in flight, and the column bounds are fetched two columns ahead.  Only rho lives in
// shared memory.  tests/microbench/iter_kernels.cu compares it (m = 10^4, n = 10^5, 10^7 entries)
// with the variants that stage the CSC tiles through shared memory with cp.async.bulk (TMA) --
// those are bound by shared-memory wavefronts (TMA writes + index/value reads + rho gathers), not
// by HBM.
// IDX16: row indices are read from the 16-bit copy (m <= 65535): 10 instead of 12 bytes per entry.
template <int THREADS, int CTAS, bool SMEM_RHO, bool IDX16 = false>
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
  const unsigned short *__restrict__ rowIdx16 = d.rowIdx16;
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
      ni[u] = p ? (IDX16 ? (int)__ldcs(rowIdx16 + e) : __ldcs(rowIdx + e)) : 0;
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
      const int r = IDX16 ? (int)__ldg(rowIdx16 + e) : __ldg(rowIdx + e);
      acc0 = fma(__ldg(val + e), SMEM_RHO ? srho[r] : __ldg(rhoG + r), acc0);
    }
    const double acc = warp_sum(acc0 + acc1);
    if (lane == 0)
      d.alphaRow[j] = acc; // row_finalize / the row pass applies the zero tolerance
  }
}

// ---------------------------------------------------------------------------------------
// PRICE, TMA-staged variant.  The CSC arrays are cut into tiles of whole columns with at most
// kPriceTile entries (host, once per matrix).  A persistent CTA per SM walks its tiles with a
// two-stage pipeline: one thread issues cp.async.bulk (TMA, 1-D) copies of the tile's row
// indices and values into shared memory, completion is signalled on an mbarrier; the CTA then
// multiplies by rho (staged in shared memory), reduces per column from shared memory and does
// the ratio-test candidate logic for all columns of the tile in parallel.
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity)
{
  asm volatile("{\n"
               ".reg .pred p;\n"
               "WAIT_LOOP:\n"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
               "@p bra WAIT_DONE;\n"
               "bra WAIT_LOOP;\n"
               "WAIT_DONE:\n"
               "}\n" ::"r"(smem_u32(bar)),
               "r"(parity)
               : "memory");
}

// tile descriptor (host-built): first column, number of columns (<= 8), first entry (multiple
// of 4), number of entries (multiple of 4, <= kPriceTile).
// The CTA (1024 threads) is split into kPriceGroups independent 256-thread pipelines, each with
// its own tiles, mbarriers and named barrier, so that one group's latency chain (mbarrier wait ->
// shared-memory gathers -> warp reduction) overlaps with the others' instead of stalling the
// whole CTA; rho is staged once per CTA and shared by the groups.
template <bool SMEM_RHO>
__global__ void __launch_bounds__(1024, 1)
    price_tma_kernel(DeviceModel d, const int4 *__restrict__ tileDesc, int ntiles, int descCap)
{
  extern __shared__ __align__(128) unsigned char smemRaw[];
  if (!iter_active(d.st))
    return;
  // layout: barriers[groups][stages] | sdesc[groups][descCap] | sidx[groups][stages][tile] |
  //         sval[groups][stages][tile] | srho[m]
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
  const int *__restrict__ colStart = d.colStart;
  const int G = gridDim.x * kPriceGroups;         // pipelines in the grid
  const int gg = blockIdx.x * kPriceGroups + grp; // this pipeline
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
    bulk_g2s(sidx + stage * kPriceTileAlloc, d.rowIdx + ds.z, cnt * 4u, &full[stage]);
    bulk_g2s(sval + stage * kPriceTileAlloc, d.val + ds.z, cnt * 8u, &full[stage]);
  };
  if (gt == 0)
    for (int q = 0; q < kPriceStages && q < myTiles; q++)
      issue(q, q);
  if (SMEM_RHO)
    for (int i = tid; i < d.m; i += 1024)
      srho[i] = d.rho[i];
  __syncthreads();
  const double *__restrict__ rho = d.rho;
  // bounds of this warp's column, fetched one tile ahead (global, L2 resident)
  // (raw values are kept in registers and only consumed one iteration later, so the loads never
  // stall the warp that issued them)
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
    if (gwarp < ds.y) { // one warp per column of the tile
      const double *v = sval + stage * kPriceTileAlloc;
      const int *ix = sidx + stage * kPriceTileAlloc;
      double acc0 = 0.0, acc1 = 0.0;
      int e = b0 + lane;
      for (; e + 32 < b1; e += 64) {
        const int r0 = ix[e], r1 = ix[e + 32];
        const double v0 = v[e], v1 = v[e + 32];
        acc0 = fma(v0, SMEM_RHO ? srho[r0] : __ldg(rho + r0), acc0);
        acc1 = fma(v1, SMEM_RHO ? srho[r1] : __ldg(rho + r1), acc1);
      }
      if (e < b1)
        acc0 = fma(v[e], SMEM_RHO ? srho[ix[e]] : __ldg(rho + ix[e]), acc0);
      const double acc = warp_sum(acc0 + acc1);
      if (lane == 0)
        d.alphaRow[ds.x + gwarp] = acc; // raw dot product; row_finalize_kernel applies status/tolerance
    }
    // group barrier: every warp of this pipeline is done with the stage
    asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(256) : "memory");
    if (gt == 0 && it + kPriceStages < myTiles) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      issue(it + kPriceStages, stage);
    }
  }
}

// Second half of PRICE: one thread per variable of the row.  Columns: apply the status mask and
// the zero tolerance to the raw dot products; rows: alpha_{n+i} = -rho_i; both: ratio-test
// candidate test + level-1 histogram (coalesced reads of status / dj / bounds).
__global__ void __launch_bounds__(256) row_finalize_kernel(DeviceModel d, int colBegin, int colEnd, bool fuseHist)
{
  __shared__ unsigned long long sHot;
  if (!iter_active(d.st))
    return;
  if (threadIdx.x == 0)
    sHot = 0ull;
  __syncthreads();
  const int sigma = d.st->sigma;
  const double infeas = d.st->infeas;
  // warp-uniform trip count: the aggregated histogram add is a warp collective
  for (int base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31; base < d.nm; base += gridDim.x * blockDim.x) {
    const int j = base + (threadIdx.x & 31);
    bool cand = false;
    double a = 1.0, dtil = 0.0, range = 0.0;
    bool boxed = false;
    if (j < d.nm && !(j < d.n && (j < colBegin || j >= colEnd))) {
      double alpha;
      const unsigned char st = d.status[j];
      if (j < d.n)
        alpha = (st == basic || st == isFixed) ? 0.0 : d.alphaRow[j];
      else
        alpha = (st == basic || st == isFixed) ? 0.0 : -d.rho[j - d.n];
      if (fabs(alpha) < d.zeroTolerance)
        alpha = 0.0;
      d.alphaRow[j] = alpha;
      cand = fuseHist && alpha != 0.0 && candidate(d, j, alpha, sigma, a, dtil, boxed, range);
    }
    if (fuseHist)
      hist_add_aggregated(d.histWeight, cand ? hist1_slot(ratio_bucket(dtil / a)) : 0,
                          cand ? slope_weight(a, boxed, range, infeas) : 0ull, cand, &sHot);
  }
  __syncthreads();
  if (threadIdx.x == 0 && sHot != 0ull)
    atomicAdd(d.histWeight, sHot);
}

// stand-alone histogram pass over a complete tableau row (column-sharded runs: after the
// all-gather of the row; also used by the ratio-test parity tests)
__global__ void __launch_bounds__(256) histogram_kernel(DeviceModel d)
{
  if (!iter_active(d.st))
    return;
  const int sigma = d.st->sigma;
  const double infeas = d.st->infeas;
  for (int base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31; base < d.nm; base += gridDim.x * blockDim.x) {
    const int j = base + (threadIdx.x & 31);
    bool cand = false;
    double a = 1.0, dtil = 0.0, range = 0.0;
    bool boxed = false;
    if (j < d.nm) {
      const double alpha = d.alphaRow[j];
      cand = alpha != 0.0 && candidate(d, j, alpha, sigma, a, dtil, boxed, range);
    }
    hist_add_aggregated(d.histWeight, cand ? hist1_slot(ratio_bucket(dtil / a)) : 0,
                        cand ? slope_weight(a, boxed, range, infeas) : 0ull, cand);
  }
}
void launch_histogram(const DeviceModel &d, cudaStream_t s)
{
  int blocks = (d.nm + 255) / 256;
  if (blocks > device_sm_count() * 4)
    blocks = device_sm_count() * 4;
  histogram_kernel<<<blocks, 256, 0, s>>>(d);
}

int g_priceIdx16 = 1; // use the 16-bit copy when the engine built one ("priceIdx16" = 1 before the first solve)

void launch_price(const DeviceModel &d, int colBegin, int colEnd, bool fuseHist, cudaStream_t s)
{
  (void)fuseHist; // both kernels leave raw dot products; the histogram is built by the row kernels
  int ncol = colEnd - colBegin;
  if (ncol <= 0)
    return;
  const size_t rhoBytes = sizeof(double) * (size_t)d.m;
  static bool attrSet = false;
  if (!attrSet) {
    cudaFuncSetAttribute(price_tma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(price_tma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    cudaFuncSetAttribute(price_ldg_kernel<640, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
    cudaFuncSetAttribute(price_ldg_kernel<1024, 1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
    cudaFuncSetAttribute(price_ldg_kernel<640, 2, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
    cudaFuncSetAttribute(price_ldg_kernel<1024, 1, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
    attrSet = true;
  }
  const int numSMs = device_sm_count();
  if (g_kernelTimers)
    cudaEventRecord(g_kernelTimers->price[0], s);
  if (d.priceTileCol != nullptr && d.numPriceTiles > 0) {
    // TMA-staged tiles (tiles were cut for this rank's column range at set-up; "usePriceTma")
    int gridTma = (d.numPriceTiles + kPriceGroups - 1) / kPriceGroups;
    if (gridTma > numSMs)
      gridTma = numSMs;
    if (gridTma < 1)
      gridTma = 1;
    const int pipes = gridTma * kPriceGroups;
    const int descCap = ((d.numPriceTiles + pipes - 1) / pipes + 7) / 8 * 8;
    const size_t tileBytes = 128 + (size_t)kPriceGroups * descCap * 16 +
                             (size_t)kPriceGroups * kPriceStages * (size_t)kPriceTileAlloc * 12;
    const int4 *desc = reinterpret_cast<const int4 *>(d.priceTileCol);
    if (tileBytes + rhoBytes <= 227 * 1024)
      price_tma_kernel<true><<<gridTma, 1024, tileBytes + rhoBytes, s>>>(d, desc, d.numPriceTiles, descCap);
    else
      price_tma_kernel<false><<<gridTma, 1024, tileBytes, s>>>(d, desc, d.numPriceTiles, descCap);
  } else if (d.rowIdx16 != nullptr && g_priceIdx16) {
    // 16-bit row indices (m <= 65535): 10 bytes per entry streamed instead of 12
    if (rhoBytes <= 112 * 1024)
      price_ldg_kernel<640, 2, true, true><<<numSMs * 2, 640, rhoBytes, s>>>(d, colBegin, colEnd);
    else if (rhoBytes <= 224 * 1024)
      price_ldg_kernel<1024, 1, true, true><<<numSMs, 1024, rhoBytes, s>>>(d, colBegin, colEnd);
    else
      price_ldg_kernel<640, 2, false, true><<<numSMs * 2, 640, 0, s>>>(d, colBegin, colEnd);
  } else if (rhoBytes <= 112 * 1024) {
    price_ldg_kernel<640, 2, true><<<numSMs * 2, 640, rhoBytes, s>>>(d, colBegin, colEnd);
  } else if (rhoBytes <= 224 * 1024) {
    price_ldg_kernel<1024, 1, true><<<numSMs, 1024, rhoBytes, s>>>(d, colBegin, colEnd);
  } else {
    price_ldg_kernel<640, 2, false><<<numSMs * 2, 640, 0, s>>>(d, colBegin, colEnd);
  }
  if (g_kernelTimers)
    cudaEventRecord(g_kernelTimers->price[1], s);
}
// second half of PRICE for the separate-kernel path (column-sharded runs): status mask / zero
// tolerance for this rank's columns, slack part of the row, optionally the level-1 histogram.
// colBegin/colEnd: the column range this rank priced; fuseHist=false in column-sharded runs,
// where the histogram is built after the all-gather by launch_histogram.
void launch_price_slacks(const DeviceModel &d, int colBegin, int colEnd, bool fuseHist, cudaStream_t s)
{
  int blocks = (d.nm + 255) / 256;
  if (blocks > device_sm_count() * 8)
    blocks = device_sm_count() * 8;
  row_finalize_kernel<<<blocks, 256, 0, s>>>(d, colBegin, colEnd, fuseHist);
}

// ---------------------------------------------------------------------------------------
// Level-1 scan: 32 CTAs x 1024 buckets.  Each CTA reduces its segment; the last CTA to finish
// locates the segment and then the bucket in which the cumulative slope reaches the primal
// infeasibility (fixed point 2^40).  Outputs st->bucket1 and st->residual (slope still to be
// absorbed inside that bucket).  The histograms are cleared by next iteration's CHUZR kernel.
__global__ void __launch_bounds__(1024) chuzc_scan1_kernel(DeviceModel d)
{
  if (!iter_active(d.st))
    return;
  __shared__ unsigned long long sTot[32];
  __shared__ int sLast[32];
  __shared__ unsigned long long segPrefix[32];
  __shared__ int sIsLast, sSeg, sLastAll;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nseg = gridDim.x; // kHistBuckets / 1024
  {
    const int b = blockIdx.x * 1024 + tid;
    unsigned long long w = d.histWeight[hist1_slot(b)];
    int last = w != 0ull ? b : -1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      w += __shfl_xor_sync(0xffffffffu, w, o);
      last = max(last, __shfl_xor_sync(0xffffffffu, last, o));
    }
    if (lane == 0) {
      sTot[warp] = w;
      sLast[warp] = last;
    }
    __syncthreads();
    if (tid == 0) {
      unsigned long long t = 0;
      int l = -1;
      for (int q = 0; q < 32; q++) {
        t += sTot[q];
        l = max(l, sLast[q]);
      }
      d.segTotal[blockIdx.x] = t;
      d.segLast[blockIdx.x] = l;
      __threadfence();
      unsigned int ticket = atomicAdd(d.scanCounter, 1u);
      sIsLast = (ticket == (unsigned)nseg - 1);
      if (sIsLast)
        *d.scanCounter = 0u;
    }
    __syncthreads();
    if (!sIsLast)
      return;
  }
  __threadfence();
  // ---- last CTA: prefix over segments
  if (tid == 0) {
    unsigned long long c = 0;
    int seg = -1, lastAll = -1;
    for (int q = 0; q < nseg; q++) {
      segPrefix[q] = c;
      unsigned long long t = d.segTotal[q];
      if (seg < 0 && c + t >= kFixOne)
        seg = q;
      c += t;
      lastAll = max(lastAll, d.segLast[q]);
    }
    sSeg = seg;
    sLastAll = lastAll;
  }
  __syncthreads();
  IterState *st = d.st;
  if (sLastAll < 0) {
    if (tid == 0) {
      st->stop = STOP_NO_COLUMN;
      st->bucket1 = -1;
    }
    return;
  }
  if (sSeg < 0) {
    // slope never exhausted: stop at the last break point group (level 2 then takes the last
    // non-empty sub-bucket of the last non-empty bucket)
    if (tid == 0) {
      st->bucket1 = sLastAll;
      st->residual = 0xFFFFFFFFFFFFFFFFull;
    }
    return;
  }
  // ---- scan inside the crossing segment
  const int b = sSeg * 1024 + tid;
  const unsigned long long w = d.histWeight[hist1_slot(b)];
  unsigned long long inc = w;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o)
      inc += t;
  }
  __syncthreads();
  if (lane == 31)
    sTot[warp] = inc;
  __syncthreads();
  unsigned long long base = segPrefix[sSeg];
  for (int q = 0; q < warp; q++)
    base += sTot[q];
  const unsigned long long excl = base + inc - w;
  if (excl < kFixOne && excl + w >= kFixOne) { // exactly one thread
    st->bucket1 = b;
    st->residual = kFixOne - excl;
  }
}

// Level-2 scan (single CTA, 4 sub-buckets per thread) -> theta*; also ||rho||^2 in a fixed order
__device__ __forceinline__ void chuzc_scan2_body(const DeviceModel &d)
{
  __shared__ unsigned long long sTot[32];
  __shared__ int sLast[32];
  __shared__ double sNorm[32];
  __shared__ int sCross;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  IterState *st = d.st;
  const int b1 = st->bucket1;
  unsigned long long w[4], mn[4];
  unsigned long long tot = 0;
  int last = -1;
  if (b1 >= 0) {
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int b = tid * 4 + q;
      w[q] = __ldcg(d.hist2Weight + b); // written by the other CTAs of this kernel (L2)
      mn[q] = __ldcg(d.hist2Min + b);
      tot += w[q];
      if (mn[q] != kSentinel)
        last = b;
    }
  }
  unsigned long long inc = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o)
      inc += t;
  }
  int wl = last;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    wl = max(wl, __shfl_xor_sync(0xffffffffu, wl, o));
  double nrm = 0.0;
  for (int i = tid; i < d.m; i += 1024) {
    double r = d.rho[i];
    nrm = fma(r, r, nrm);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    nrm += __shfl_xor_sync(0xffffffffu, nrm, o);
  if (lane == 31)
    sTot[warp] = inc;
  if (lane == 0) {
    sLast[warp] = wl;
    sNorm[warp] = nrm;
  }
  if (tid == 0)
    sCross = -1;
  __syncthreads();
  if (tid == 0) {
    double nsum = 0.0;
    for (int q = 0; q < 32; q++)
      nsum += sNorm[q];
    st->rhoNorm2 = nsum;
    st->harrisBits = 0x7FF0000000000000ull; // +inf
    st->chuzcKey = 0ull;
  }
  if (b1 < 0)
    return; // thetaStar already set by scan1 (or no candidates)
  unsigned long long base = 0;
  for (int q = 0; q < warp; q++)
    base += sTot[q];
  const unsigned long long resid = st->residual;
  const unsigned long long excl = base + inc - tot;
  if (excl < resid && excl + tot >= resid) {
    unsigned long long c = excl;
    int found = -1;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      c += w[q];
      if (found < 0 && c >= resid)
        found = q;
    }
    sCross = tid * 4 + found;
    st->thetaStar = __longlong_as_double((long long)mn[found]);
  }
  __syncthreads();
  if (sCross < 0 && tid == 0) {
    // numerically possible only through fixed-point truncation: take the last sub-bucket
    int lastAll = -1;
    for (int q = 0; q < 32; q++)
      lastAll = max(lastAll, sLast[q]);
    st->thetaStar = __longlong_as_double((long long)__ldcg(d.hist2Min + lastAll));
  }
}

// Level 2: candidates of the crossing bucket, next 12 bits of the ratio (all CTAs); the last CTA
// then scans the 4096 sub-buckets (chuzc_scan2_body).  1024 threads per CTA.
__global__ void __launch_bounds__(1024) chuzc_hist2_kernel(DeviceModel d)
{
  __shared__ unsigned long long sHot, sHotMin;
  if (!iter_active(d.st))
    return;
  if (threadIdx.x == 0) {
    sHot = 0ull;
    sHotMin = kSentinel;
  }
  __syncthreads();
  const int b1 = d.st->bucket1;
  if (b1 >= 0) {
    const int sigma = d.st->sigma;
    const double infeas = d.st->infeas;
    for (int base = (blockIdx.x * blockDim.x + threadIdx.x) & ~31; base < d.nm; base += gridDim.x * blockDim.x) {
      const int j = base + (threadIdx.x & 31);
      bool cand = false;
      double a = 1.0, dtil = 0.0, range = 0.0;
      bool boxed = false;
      unsigned long long bits = 0ull;
      if (j < d.nm) {
        const double alpha = d.alphaRow[j];
        if (alpha != 0.0 && candidate(d, j, alpha, sigma, a, dtil, boxed, range)) {
          bits = (unsigned long long)__double_as_longlong(dtil / a);
          cand = ((int)(bits >> 48) & (kHistBuckets - 1)) == b1;
        }
      }
      const int sb = (int)(bits >> 36) & (kHist2Buckets - 1);
      hist_add_aggregated(d.hist2Weight, sb, cand ? slope_weight(a, boxed, range, infeas) : 0ull, cand, &sHot);
      hist_min_aggregated(d.hist2Min, sb, bits, cand, &sHotMin);
    }
    __syncthreads();
    if (threadIdx.x == 0 && sHot != 0ull) {
      atomicAdd(d.hist2Weight, sHot);
      atomicMin(d.hist2Min, sHotMin);
    }
  }
  if (!last_block_done(d.tailCounter + TAIL_HIST2))
    return;
  chuzc_scan2_body(d);
}

// Harris bound over candidates with ratio >= theta*  (ClpSimplexDual.cpp:4331-4395 upperTheta)
__global__ void chuzc_harris_kernel(DeviceModel d)
{
  if (!iter_active(d.st))
    return;
  const int sigma = d.st->sigma;
  const double thetaStar = d.st->thetaStar;
  const double tol = d.dualTolerance;
  unsigned long long best = 0x7FF0000000000000ull;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < d.nm; j += gridDim.x * blockDim.x) {
    const double alpha = d.alphaRow[j];
    if (alpha == 0.0)
      continue;
    double a, dtil, range;
    bool boxed;
    if (!candidate(d, j, alpha, sigma, a, dtil, boxed, range))
      continue;
    if (a < d.st->acceptablePivot || dtil / a < thetaStar)
      continue;
    unsigned long long h = (unsigned long long)__double_as_longlong((dtil + tol) / a);
    best = min(best, h);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best != 0x7FF0000000000000ull)
    atomicMin(&d.st->harrisBits, best);
}

// largest |alpha| with theta* <= ratio <= harris  (ClpSimplexDual.cpp:4531-4573)
__global__ void chuzc_select_kernel(DeviceModel d)
{
  if (!iter_active(d.st))
    return;
  const int sigma = d.st->sigma;
  const double thetaStar = d.st->thetaStar;
  const double harris = __longlong_as_double((long long)d.st->harrisBits);
  unsigned long long best = 0ull;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < d.nm; j += gridDim.x * blockDim.x) {
    const double alpha = d.alphaRow[j];
    if (alpha == 0.0)
      continue;
    double a, dtil, range;
    bool boxed;
    if (!candidate(d, j, alpha, sigma, a, dtil, boxed, range))
      continue;
    const double ratio = dtil / a;
    if (a < d.st->acceptablePivot || ratio < thetaStar || ratio > harris)
      continue;
    unsigned long long key = ((unsigned long long)__double_as_longlong(a) & ~0xFFFFFull) |
                             (unsigned long long)(0xFFFFF - j);
    best = max(best, key);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best != 0ull)
    atomicMax(&d.st->chuzcKey, best);
  // tail (last CTA, one thread): decode the winner
  if (!last_block_done(d.tailCounter + TAIL_SELECT))
    return;
  if (threadIdx.x != 0)
    return;
  IterState *st = d.st;
  const unsigned long long key = atomicMax(&st->chuzcKey, 0ull);
  if (key == 0ull) {
    st->stop = STOP_NO_COLUMN;
    return;
  }
  const int q = 0xFFFFF - (int)(key & 0xFFFFFull);
  st->seqIn = q;
  const double alpha = d.alphaRow[q];
  st->alphaRow = alpha;
  const double t = d.dj[q] / (st->sigma * alpha);
  st->thetaDual = t > 0.0 ? t : 0.0;
  st->harrisTheta = __longlong_as_double((long long)st->harrisBits);
}

void launch_chuzc(const DeviceModel &d, cudaStream_t s)
{
  int blocks = (d.nm + 255) / 256;
  if (blocks > device_sm_count() * 4)
    blocks = device_sm_count() * 4;
  int blocks2 = (d.nm + 1023) / 1024;
  if (blocks2 > device_sm_count())
    blocks2 = device_sm_count();
  chuzc_scan1_kernel<<<kHistBuckets / 1024, 1024, 0, s>>>(d);
  chuzc_hist2_kernel<<<blocks2, 1024, 0, s>>>(d); // + level-2 scan in its tail
  chuzc_harris_kernel<<<blocks, 256, 0, s>>>(d);
  chuzc_select_kernel<<<blocks, 256, 0, s>>>(d); // + decode of the winner in its tail
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
