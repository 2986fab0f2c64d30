// rowpass.cu -- everything the iteration does with the tableau row, in ONE cooperative kernel.
//
// The second half of ClpPackedMatrix::transposeTimes (status mask / zero tolerance,
// /root/reference/src/ClpPackedMatrix.cpp:1860-1900), ClpSimplexDual::dualColumn0 / dualColumn
// (src/ClpSimplexDual.cpp:3665 / :4192), ClpSimplexDual::updateDualsInDual (:2430) with its
// bound flips, and the unpack of the entering column (ClpPackedMatrix::unpack :4803).
//
// Ratio test without a sort: every candidate adds its slope contribution |alpha_j|*(u_j-l_j) to a
// histogram over the (monotone) bit pattern of its ratio d_j/|alpha_j| -- in 2^-40 fixed point
// relative to the primal infeasibility, with integer atomics, so the result does not depend on the
// order of the atomics.  The bucket in which the slope of the dual objective is exhausted gives
// theta*; the Harris bound beyond theta* and the largest |alpha| inside [theta*, harris] pick the
// pivot.  Candidates with a ratio below theta* are "passed": the dual update flips them to their
// other bound (BFRT).
//
// One CTA per SM (cooperative launch => co-resident), 1024 threads; every thread owns E entries
// of the row and keeps (alpha, |alpha|, d~, range, flags) in registers across the phases, so the
// row is read from memory once.  Phases are separated by grid barriers instead of
// kernel boundaries; the small scans are done redundantly by every CTA, which saves a barrier.
//   P0 finalize row + level-1 ratio histogram + per-segment totals      | barrier
//   P1 crossing bucket (every CTA)  P2 level-2 histogram of that bucket | barrier
//   P3 theta* (every CTA)  P4/P5 Harris bound + largest |alpha| in [theta*, harris] from the short
//      list of the crossing bucket's candidates (every CTA; two more barriers only if the bound
//      leaves the listed window)
//   P6 decode winner, dual update + bound flips (unordered list)        | barrier
//   P8 flip columns -> fixed-point accumulator; entering column -> aqBuf| barrier
//   P9 three FTRAN right-hand sides rhs3 and their nucleus gather xg
// All reductions are order independent (integer atomics, min/max of packed keys) or done in a
// fixed order.
#include "kernels_common.cuh"

#include <cstdio>

namespace clpb {

// Generation barrier over all CTAs of a cooperative grid; bar[0] = arrival count, bar[1] =
// generation.  One acq_rel atomic per CTA plus an acquire spin on the generation word (which the
// last arriver publishes with a release store): about half the cost of the fence + atomic +
// volatile-spin + fence formulation.  'gen' is thread 0's private copy of the current generation
// (read once at kernel start: nobody can advance it before every CTA has arrived at barrier 1).
__device__ __forceinline__ unsigned int ld_acquire_u32(const unsigned int *p)
{
  unsigned int v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned int atom_add_acq_rel_u32(unsigned int *p, unsigned int v)
{
  unsigned int o;
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(o) : "l"(p), "r"(v) : "memory");
  return o;
}
__device__ __forceinline__ void st_release_u32(unsigned int *p, unsigned int v)
{
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void grid_barrier(unsigned int *bar, unsigned int &gen)
{
  __syncthreads();
  if (threadIdx.x == 0) {
    if (atom_add_acq_rel_u32(bar, 1u) == gridDim.x - 1) {
      bar[0] = 0u; // ordered before the release store below
      st_release_u32(bar + 1, gen + 1u);
    } else {
      while (ld_acquire_u32(bar + 1) == gen) {
      }
    }
    gen++;
  }
  __syncthreads();
}

__device__ __forceinline__ unsigned long long block_min_u64(unsigned long long v, unsigned long long *sm)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
    sm[threadIdx.x >> 5] = v;
  __syncthreads();
  v = sm[threadIdx.x & 31];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v; // same value in every thread
}
__device__ __forceinline__ unsigned long long block_max_u64(unsigned long long v, unsigned long long *sm)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0)
    sm[threadIdx.x >> 5] = v;
  __syncthreads();
  v = sm[threadIdx.x & 31];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

enum : unsigned { F_CAND = 1u, F_BOXED = 2u, F_VALID = 4u };
constexpr int kWindowBuckets = 1; // level-1 buckets beyond the crossing one kept in the short list
constexpr int kListCap = 4096;    // longer lists (degenerate LPs: thousands of ratio-0 ties) take the global path

template <int E>
__global__ void __launch_bounds__(1024, 1) row_pass_kernel(DeviceModel d)
{
  IterState *st = d.st;
  if (!iter_active(st))
    return; // uniform over the grid
  __shared__ unsigned long long sU64[32];
  __shared__ unsigned long long sHot, sHotMin, sResidual, sThetaBits;
  __shared__ int sI32[32];
  __shared__ double sF64[32];
  __shared__ int sSeg, sLastAll, sBucket1, sCross;
  __shared__ unsigned long long sPrefix;
  __shared__ unsigned long long sSegTot[kHistBuckets / 1024];
  __shared__ int sSegLast[kHistBuckets / 1024];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gtid = blockIdx.x * 1024 + tid, gthreads = gridDim.x * 1024;
  const int sigma = st->sigma;
  const double infeas = st->infeas;
  const int n = d.n, nm = d.nm;
  unsigned int barGen = 0u;
  if (tid == 0)
    barGen = ld_acquire_u32(d.gridBar + 1);
  if (gtid == 0) { // consumed after barrier 3 / 4
    st->harrisBits = 0x7FF0000000000000ull;
    st->chuzcKey = 0ull;
  }
  if (tid == 0)
    sHot = 0ull;
  if (tid < kHistBuckets / 1024) {
    sSegTot[tid] = 0ull;
    sSegLast[tid] = -1;
  }
  __syncthreads();

  // ---------------------------------------------------------------- P0 finalize + histogram
  double alpha[E], aabs[E], dtil[E], range[E];
  unsigned flags[E];
#pragma unroll
  for (int e = 0; e < E; e++) {
    const int j = gtid + e * gthreads; // gthreads is a multiple of 32: warp-uniform validity pattern
    flags[e] = 0u;
    alpha[e] = 0.0;
    aabs[e] = 1.0;
    dtil[e] = 0.0;
    range[e] = 0.0;
    bool cand = false, boxed = false;
    if (j < nm) {
      flags[e] = F_VALID;
      const unsigned char s = d.status[j];
      double al;
      if (j < n)
        al = (s == basic || s == isFixed) ? 0.0 : d.alphaRow[j];
      else
        al = (s == basic || s == isFixed) ? 0.0 : -d.rho[j - n];
      if (fabs(al) < d.zeroTolerance)
        al = 0.0;
      d.alphaRow[j] = al;
      alpha[e] = al;
      cand = al != 0.0 && candidate(d, j, al, sigma, aabs[e], dtil[e], boxed, range[e]);
      if (cand)
        flags[e] |= F_CAND | (boxed ? F_BOXED : 0u);
    }
    const int bkt = cand ? ratio_bucket(dtil[e] / aabs[e]) : 0;
    const unsigned long long w = cand ? slope_weight(aabs[e], boxed, range[e], infeas) : 0ull;
    hist_add_aggregated(d.histWeight, hist1_slot(bkt), w, cand, &sHot);
    // per-segment totals / last non-empty bucket of this CTA (warp-aggregated shared-memory atomics)
    hist_add_aggregated(sSegTot, bkt >> 10, w, cand);
    max_aggregated(sSegLast, bkt >> 10, bkt, cand);
  }
  __syncthreads();
  if (tid == 0 && sHot != 0ull)
    atomicAdd(d.histWeight, sHot);
  if (tid < kHistBuckets / 1024 && sSegLast[tid] >= 0) {
    atomicAdd(d.segTotal + tid, sSegTot[tid]);
    atomicMax(d.segLast + tid, sSegLast[tid]);
  }
  grid_barrier(d.gridBar, barGen);

  // ---------------------------------------------------------------- P1 crossing bucket (every CTA)
  constexpr int NSEG = kHistBuckets / 1024; // 32: one lane per segment
  if (warp == 0) {
    const unsigned long long t = __ldcg(d.segTotal + lane);
    int lastAll = __ldcg(d.segLast + lane);
    unsigned long long inc = t;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      unsigned long long u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o)
        inc += u;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      lastAll = max(lastAll, __shfl_xor_sync(0xffffffffu, lastAll, o));
    const unsigned long long excl = inc - t;
    const bool cross = excl < kFixOne && inc >= kFixOne; // first segment where the total reaches 1
    const unsigned cm = __ballot_sync(0xffffffffu, cross);
    if (lane == 0) {
      sSeg = cm ? __ffs(cm) - 1 : -1;
      sLastAll = lastAll;
      sBucket1 = -1;
      sResidual = 0xFFFFFFFFFFFFFFFFull;
    }
    if (cross)
      sPrefix = excl;
  }
  __syncthreads();
  if (sLastAll < 0) { // no candidate at all
    if (gtid == 0) {
      st->stop = STOP_NO_COLUMN;
      st->bucket1 = -1;
    }
    return;
  }
  if (sSeg < 0) {
    // slope never exhausted: stop at the last break point group
    if (tid == 0)
      sBucket1 = sLastAll;
    __syncthreads();
  } else {
    const int b = sSeg * 1024 + tid;
    const unsigned long long w = __ldcg(d.histWeight + hist1_slot(b));
    unsigned long long inc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o)
        inc += t;
    }
    if (lane == 31)
      sU64[warp] = inc;
    __syncthreads();
    unsigned long long base = sPrefix;
    for (int q = 0; q < warp; q++)
      base += sU64[q];
    const unsigned long long excl = base + inc - w;
    if (excl < kFixOne && excl + w >= kFixOne) { // exactly one thread
      sBucket1 = b;
      sResidual = kFixOne - excl;
    }
    __syncthreads();
  }
  const int bucket1 = sBucket1;
  const unsigned long long residual = sResidual;
  if (gtid == 0) {
    st->bucket1 = bucket1;
    st->residual = residual;
  }

  // ---------------------------------------------------------------- P2 level-2 histogram
  if (tid == 0) {
    sHot = 0ull;
    sHotMin = kSentinel;
  }
  __syncthreads();
#pragma unroll
  for (int e = 0; e < E; e++) {
    bool in = false;
    unsigned long long bits = 0ull;
    if (flags[e] & F_CAND) {
      bits = (unsigned long long)__double_as_longlong(dtil[e] / aabs[e]);
      in = ((int)(bits >> 48) & (kHistBuckets - 1)) == bucket1;
    }
    const int sb = (int)(bits >> 36) & (kHist2Buckets - 1);
    hist_add_aggregated(d.hist2Weight, sb,
                        in ? slope_weight(aabs[e], (flags[e] & F_BOXED) != 0u, range[e], infeas) : 0ull, in, &sHot);
    hist_min_aggregated(d.hist2Min, sb, bits, in, &sHotMin);
    // candidates of the crossing bucket and the next one: the short list every CTA scans for the
    // Harris bound and the pivot (see P4/P5) -- unordered, min/max do not care
    {
      // one atomic per warp (the candidates of the window are hundreds to thousands: one same-address
      // atomic each would serialise in L2)
      const int bk = (int)(bits >> 48) & (kHistBuckets - 1);
      const bool inWin = (flags[e] & F_CAND) && bk >= bucket1 && bk <= bucket1 + kWindowBuckets;
      const unsigned wm = __ballot_sync(0xffffffffu, inWin);
      if (wm) {
        int base = 0;
        const int leader = __ffs(wm) - 1;
        if (lane == leader)
          base = atomicAdd(d.candCount, __popc(wm));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (inWin) {
          const int at = base + __popc(wm & ((1u << lane) - 1u));
          if (at < kListCap) {
            d.candA[at] = aabs[e];
            d.candD[at] = dtil[e];
            d.candJ[at] = gtid + e * gthreads;
          }
        }
      }
    }
  }
  __syncthreads();
  if (tid == 0 && sHot != 0ull) {
    atomicAdd(d.hist2Weight, sHot);
    atomicMin(d.hist2Min, sHotMin);
  }
  grid_barrier(d.gridBar, barGen);

  // ---------------------------------------------------------------- P3 theta* (every CTA)
  {
    unsigned long long w[4], mn[4], tot = 0;
    int last = -1;
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const int b = tid * 4 + q;
      w[q] = __ldcg(d.hist2Weight + b);
      mn[q] = __ldcg(d.hist2Min + b);
      tot += w[q];
      if (mn[q] != kSentinel)
        last = b;
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
    if (lane == 31)
      sU64[warp] = inc;
    if (lane == 0)
      sI32[warp] = wl;
    if (tid == 0)
      sCross = -1;
    __syncthreads();
    unsigned long long base = 0;
    for (int q = 0; q < warp; q++)
      base += sU64[q];
    const unsigned long long excl = base + inc - tot;
    if (excl < residual && excl + tot >= residual) {
      unsigned long long c = excl;
      int found = -1;
#pragma unroll
      for (int q = 0; q < 4; q++) {
        c += w[q];
        if (found < 0 && c >= residual)
          found = q;
      }
      sCross = tid * 4 + found;
      sThetaBits = mn[found];
    }
    __syncthreads();
    if (sCross < 0 && tid == 0) {
      // numerically possible only through fixed-point truncation: take the last sub-bucket
      int lastAll = -1;
      for (int q = 0; q < 32; q++)
        lastAll = max(lastAll, sI32[q]);
      sThetaBits = __ldcg(d.hist2Min + lastAll);
    }
    __syncthreads();
  }
  const double thetaStar = __longlong_as_double((long long)sThetaBits);
  if (blockIdx.x == 0) {
    // ||rho||^2 in a fixed order (DSE weight of the pivot row)
    double nrm = 0.0;
    for (int i = tid; i < d.m; i += 1024) {
      const double r = d.rho[i];
      nrm = fma(r, r, nrm);
    }
    nrm = warp_sum(nrm);
    if (lane == 0)
      sF64[warp] = nrm;
    __syncthreads();
    if (tid == 0) {
      double nsum = 0.0;
      for (int q = 0; q < 32; q++)
        nsum += sF64[q];
      st->rhoNorm2 = nsum;
      st->thetaStar = thetaStar;
    }
  }

  // ---------------------------------------------------------------- P4/P5 Harris bound and pivot
  // Fast path (no barrier): every CTA scans the short list of the candidates whose ratio lies in
  // the crossing level-1 bucket or the next kWindowBuckets.  If the Harris bound found there is
  // below the upper edge U of that window it is the global one -- a candidate outside the list has
  // ratio >= U (or < theta*), so its own bound (d~+tol)/|alpha| >= U cannot be the minimum -- and
  // every candidate of [theta*, harris] is in the list, so the largest |alpha| is found there too.
  // Otherwise (uniform decision) the two global reductions with their grid barriers run.
  unsigned long long harrisBits, key;
  {
    const int cntAll = __ldcg(d.candCount);
    const int cnt = cntAll <= kListCap ? cntAll : 0;
    unsigned long long best = 0x7FF0000000000000ull;
    for (int i = tid; i < cnt; i += 1024) {
      const double a = __ldcg(d.candA + i), dt = __ldcg(d.candD + i);
      if (a >= st->acceptablePivot && dt / a >= thetaStar)
        best = min(best, (unsigned long long)__double_as_longlong((dt + d.dualTolerance) / a));
    }
    best = block_min_u64(best, sU64);
    const unsigned long long windowEnd = (unsigned long long)(bucket1 + kWindowBuckets + 1) << 48;
    if (cntAll <= kListCap && best < windowEnd && best != 0x7FF0000000000000ull) {
      harrisBits = best;
      const double harrisL = __longlong_as_double((long long)best);
      unsigned long long bk = 0ull;
      for (int i = tid; i < cnt; i += 1024) {
        const double a = __ldcg(d.candA + i), dt = __ldcg(d.candD + i);
        const double ratio = dt / a;
        if (a >= st->acceptablePivot && ratio >= thetaStar && ratio <= harrisL)
          bk = max(bk, ((unsigned long long)__double_as_longlong(a) & ~0xFFFFFull) |
                           (unsigned long long)(0xFFFFF - __ldcg(d.candJ + i)));
      }
      key = block_max_u64(bk, sU64);
    } else {
      // ---- global Harris bound
      unsigned long long gb = 0x7FF0000000000000ull;
#pragma unroll
      for (int e = 0; e < E; e++)
        if ((flags[e] & F_CAND) && aabs[e] >= st->acceptablePivot && dtil[e] / aabs[e] >= thetaStar)
          gb = min(gb, (unsigned long long)__double_as_longlong((dtil[e] + d.dualTolerance) / aabs[e]));
      gb = block_min_u64(gb, sU64);
      if (tid == 0 && gb != 0x7FF0000000000000ull)
        atomicMin(&st->harrisBits, gb);
      grid_barrier(d.gridBar, barGen);
      harrisBits = __ldcg(&st->harrisBits);
      const double harrisG = __longlong_as_double((long long)harrisBits);
      // ---- global largest |alpha| in [theta*, harris]
      unsigned long long bk = 0ull;
#pragma unroll
      for (int e = 0; e < E; e++) {
        if (!(flags[e] & F_CAND) || aabs[e] < st->acceptablePivot)
          continue;
        const double ratio = dtil[e] / aabs[e];
        if (ratio < thetaStar || ratio > harrisG)
          continue;
        const int j = gtid + e * gthreads;
        bk = max(bk, ((unsigned long long)__double_as_longlong(aabs[e]) & ~0xFFFFFull) |
                         (unsigned long long)(0xFFFFF - j));
      }
      bk = block_max_u64(bk, sU64);
      if (tid == 0 && bk != 0ull)
        atomicMax(&st->chuzcKey, bk);
      grid_barrier(d.gridBar, barGen);
      key = __ldcg(&st->chuzcKey);
    }
  }
  const double harris = __longlong_as_double((long long)harrisBits);

  // ---------------------------------------------------------------- P6 winner, dual update, flips
  if (key == 0ull) {
    if (gtid == 0) {
      st->stop = STOP_NO_COLUMN;
      *d.candCount = 0;
    }
    return; // uniform
  }
  const int seqIn = 0xFFFFF - (int)(key & 0xFFFFFull);
  const double alphaQ = __ldcg(d.alphaRow + seqIn);
  double theta = d.dj[seqIn] / (sigma * alphaQ); // dj[seqIn] is not touched below
  theta = theta > 0.0 ? theta : 0.0;
  if (gtid == 0) {
    st->seqIn = seqIn;
    st->alphaRow = alphaQ;
    st->thetaDual = theta;
    st->harrisTheta = harris;
  }
  {
    const double tol = d.dualTolerance;
    unsigned long long maxRange = 0ull;
#pragma unroll
    for (int e = 0; e < E; e++) {
      const int j = gtid + e * gthreads;
      const double al = alpha[e];
      if (!(flags[e] & F_VALID) || al == 0.0 || j == seqIn)
        continue;
      const unsigned char s = d.status[j];
      if (s == basic || s == isFixed)
        continue;
      double dnew = d.dj[j] - theta * (sigma * al);
      const bool wrong = (s == atLowerBound && dnew < -tol) || (s == atUpperBound && dnew > tol);
      if (wrong) {
        const double lo = d.lower[j], up = d.upper[j];
        if (up - lo < 1.0e29) {
          if (s == atLowerBound) {
            d.status[j] = atUpperBound;
            d.sol[j] = up;
          } else {
            d.status[j] = atLowerBound;
            d.sol[j] = lo;
          }
          d.flipList[atomicAdd(&st->numFlips, 1)] = j; // order is irrelevant: fixed-point sums
          maxRange = max(maxRange, (unsigned long long)__double_as_longlong(up - lo));
        } else {
          d.cost[j] -= dnew;
          dnew = 0.0;
          atomicAdd(&st->costShifts, 1);
        }
      } else if ((s == isFree || s == superBasic) && fabs(dnew) > tol) {
        d.cost[j] -= dnew;
        dnew = 0.0;
        atomicAdd(&st->costShifts, 1);
      }
      d.dj[j] = dnew;
    }
    maxRange = block_max_u64(maxRange, sU64);
    if (tid == 0 && maxRange != 0ull)
      atomicMax(&st->flipMaxBits, maxRange);
  }
  grid_barrier(d.gridBar, barGen);

  // ---------------------------------------------------------------- P8 scatter flips + entering column
  // every contribution |a_ij * delta_j| <= amax * maxRange < 2^Ex, at most nf < 2^bitsN of them per
  // row: with Q = 62 - bitsN fractional bits the int64 sums cannot overflow (same in every CTA)
  const int nf = __ldcg(&st->numFlips);
  double scale = 0.0, invScale = 0.0;
  if (nf > 0) {
    const double bound = d.amax * __longlong_as_double((long long)__ldcg(&st->flipMaxBits));
    int Ex = 0;
    frexp(bound, &Ex);
    const int Q = 62 - (32 - __clz(nf));
    scale = ldexp(1.0, Q - Ex);
    invScale = ldexp(1.0, Ex - Q);
  }
  if (nf > 0) {
    unsigned long long *acc = reinterpret_cast<unsigned long long *>(d.flipAcc);
    const int gw = gtid >> 5, GW = gthreads >> 5;
    for (int f = gw; f < nf; f += GW) {
      const int j = __ldcg(d.flipList + f);
      const double rg = d.upper[j] - d.lower[j];
      const double delta = __ldcg(d.status + j) == atUpperBound ? rg : -rg;
      if (j >= n) {
        if (lane == 0)
          atomicAdd(acc + (j - n), (unsigned long long)__double2ll_rn(delta * scale));
      } else {
        const int e1 = d.colStart[j + 1];
        for (int e = d.colStart[j] + lane; e < e1; e += 32)
          atomicAdd(acc + d.rowIdx[e], (unsigned long long)__double2ll_rn(-delta * d.val[e] * scale));
      }
    }
  }
  if (seqIn < n && (int)blockIdx.x == (int)gridDim.x - 1) { // entering column -> aqBuf (zero when idle)
    const int e1 = d.colStart[seqIn + 1];
    for (int e = d.colStart[seqIn] + tid; e < e1; e += 1024)
      d.aqBuf[d.rowIdx[e]] = d.val[e];
  }
  grid_barrier(d.gridBar, barGen);

  // ---------------------------------------------------------------- P9 rhs3 and its nucleus gather
  {
    const double inv = invScale;
    if (gtid == 0) {
      st->flipMaxBits = 0ull; // every CTA read it before the last barrier
      *d.candCount = 0;       // the list was last read before barrier 6
    }
    const int ldk = d.fd->ldk, k = d.fd->k;
    const int maxk8 = (d.m + 7) / 8 * 8;
    double *xg = d.ywork + (size_t)3 * maxk8;
    for (int p = gtid; p < d.m; p += gthreads) {
      double aq;
      if (seqIn >= n) {
        aq = (p == seqIn - n) ? -1.0 : 0.0;
      } else {
        aq = __ldcg(d.aqBuf + p);
        if (aq != 0.0)
          d.aqBuf[p] = 0.0;
      }
      double fl = 0.0;
      if (nf > 0) {
        const long long a = __ldcg(d.flipAcc + p);
        if (a != 0ll) {
          fl = (double)a * inv;
          d.flipAcc[p] = 0ll;
        }
      }
      const double rh = d.rho[p];
      d.rhs3[p] = aq;
      d.rhs3[(size_t)d.m + p] = rh;
      d.rhs3[(size_t)2 * d.m + p] = fl;
      const int ni = d.posToNuc[p];
      if (ni >= 0) {
        xg[ni] = aq;
        xg[(size_t)ldk + ni] = rh;
        xg[(size_t)2 * ldk + ni] = fl;
      }
    }
    for (int j = k + gtid; j < ldk; j += gthreads) { // zero padding so the GEMV can run over ldk
      xg[j] = 0.0;
      xg[(size_t)ldk + j] = 0.0;
      xg[(size_t)2 * ldk + j] = 0.0;
    }
  }
}

// Launch; returns false (and says why on stderr) when the row does not fit: at most 8 entries per
// thread of one 1024-thread CTA per SM, i.e. n+m <= 8 x SMs x 1024, and at least one CTA per level-1
// histogram segment (32 SMs).  Nothing else runs the ratio test.
bool launch_row_pass(const DeviceModel &d, cudaStream_t s)
{
  const int numSMs = device_sm_count();
  const long gthreads = (long)numSMs * 1024;
  const int need = (int)((d.nm + gthreads - 1) / gthreads);
  if (need > 8 || numSMs < kHistBuckets / 1024) {
    fprintf(stderr, "clp_b200: the row pass needs n+m <= 8 x SMs x 1024 = %ld and at least %d SMs; n+m = %d, SMs = %d\n",
            8 * gthreads, kHistBuckets / 1024, d.nm, numSMs);
    return false;
  }
  DeviceModel dm = d;
  void *args[] = {&dm};
  cudaError_t rc;
  if (need <= 1)
    rc = cudaLaunchCooperativeKernel((void *)row_pass_kernel<1>, dim3(numSMs), dim3(1024), args, 0, s);
  else if (need <= 2)
    rc = cudaLaunchCooperativeKernel((void *)row_pass_kernel<2>, dim3(numSMs), dim3(1024), args, 0, s);
  else if (need <= 4)
    rc = cudaLaunchCooperativeKernel((void *)row_pass_kernel<4>, dim3(numSMs), dim3(1024), args, 0, s);
  else
    rc = cudaLaunchCooperativeKernel((void *)row_pass_kernel<8>, dim3(numSMs), dim3(1024), args, 0, s);
  return rc == cudaSuccess;
}

} // namespace clpb
