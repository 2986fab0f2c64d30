// kernels_common.cuh -- device helpers shared by solve.cu / price.cu / rowpass.cu / update.cu.
#pragma once
#include "engine.cuh"

namespace clpb {

__device__ __forceinline__ bool iter_active(const IterState *st) { return st->stop == 0; }

__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// indices into DeviceModel::tailCounter
enum : int { TAIL_ITER_UPDATE = 0, TAIL_PFI_APPLY = 1, TAIL_SPREAD = 2 };

// "last block done": returns true in exactly one CTA of a 1-D grid, after every other CTA of the
// grid has passed this point (and hence finished the work before it).  What the tail then reads
// of other CTAs' results must bypass L1 (__ldcg / atomics): L1 is not coherent inside a kernel.
__device__ __forceinline__ bool last_block_done(unsigned int *counter)
{
  __shared__ int sIsLast;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int ticket = atomicAdd(counter, 1u);
    const int last = (ticket == gridDim.x - 1);
    if (last)
      *counter = 0u; // ready for the next launch
    sIsLast = last;
  }
  __syncthreads();
  if (sIsLast)
    __threadfence();
  return sIsLast != 0;
}

// Row t of Ginv (and column t of its transposed copy) for the eta that is being appended:
//   Ginv[t][j] = -nu_j / alpha_r (j < t),  Ginv[t][t] = 1 / alpha_r,
// where nu = Ginv^T W[r][0..t) is exactly what the BTRAN of this iteration computed for the same
// pivot row r and the same t (eta_rowvec_kernel mode 0), so nothing is recomputed here.
// Grid-stride over j by the calling threads (jt = linear thread index, jn = number of threads).
__device__ __forceinline__ void eta_append_row(const DeviceModel &d, int jt, int jn)
{
  const int t = d.st->numEtas;
  const double dinv = 1.0 / d.st->alphaCol;
  for (int j = jt; j <= t; j += jn) {
    const double v = j < t ? -d.nu[j] * dinv : dinv;
    d.Ginv[(size_t)t * d.tmax + j] = v;
    d.GinvT[(size_t)j * d.tmax + t] = v;
  }
}

// packed (score, position) key of the dual steepest edge row choice; 0 = primal feasible
__device__ __forceinline__ unsigned long long chuzr_key(double x, double lo, double up, double weight,
                                                        double tol, int p)
{
  double inf = 0.0;
  if (x < lo - tol)
    inf = lo - x;
  else if (x > up + tol)
    inf = x - up;
  if (!(inf > 0.0))
    return 0ull;
  const double score = inf * inf / weight;
  return ((unsigned long long)__double_as_longlong(score) & ~0xFFFFFull) | (unsigned long long)(0xFFFFF - p);
}

// accuracy gate (ClpSimplexDual.cpp:1447-1501) and primal step length.  Runs as the tail of the
// eta-panel kernel of the FTRAN (solve.cu), i.e. single thread, results of other CTAs via L2.
__device__ __forceinline__ void pivot_scalars_body(const DeviceModel &d)
{
  IterState *st = d.st;
  const int r = st->pivotRow;
  const double ac = __ldcg(d.rhs3 + r);
  st->alphaCol = ac;
  const double ar = st->alphaRow;
  const double err = fabs(ar - ac) / (1.0 + fabs(ac));
  const bool bad = !(fabs(ac) >= 1.0e-9) || !(err <= 1.0e-6);
  if (bad) {
    if (st->numEtas > 0) {
      st->stop = STOP_INACCURATE; // the host refactorizes, recomputes and retries
      return;
    }
    if (!(fabs(ac) >= 1.0e-11) || !(err <= 1.0e-3)) {
      st->stop = STOP_TINY_PIVOT; // fresh factors and still no usable pivot
      return;
    }
  }
  const int seqOut = st->seqOut;
  double valueOut = d.sol[seqOut];
  if (st->numFlips > 0)
    valueOut += __ldcg(d.rhs3 + (size_t)2 * d.m + r);
  const double bound = st->sigma < 0 ? d.lower[seqOut] : d.upper[seqOut];
  st->thetaPrimal = (valueOut - bound) / ac;
}

// ---- ratio test (CHUZC) helpers of rowpass.cu
constexpr unsigned long long kFixOne = 1ull << 40; // fixed-point 1.0 (== infeasibility)
constexpr unsigned long long kFixCap = 1ull << 41;
constexpr unsigned long long kSentinel = 0xFFFFFFFFFFFFFFFFull;

__device__ __forceinline__ int ratio_bucket(double r)
{
  return (int)((unsigned long long)__double_as_longlong(r) >> 48) & (kHistBuckets - 1);
}
// Storage slot of level-1 bucket b.  The candidates of one iteration fall into a few hundred
// CONSECUTIVE buckets (ratios within ~20 octaves); stored consecutively those are ~20 cache lines,
// i.e. ~20 L2 slices serialising tens of thousands of atomics.  Consecutive buckets are therefore
// stored 128 bytes apart (bijection on 15 bits; slot 0 = bucket 0).
__device__ __forceinline__ int hist1_slot(int b) { return ((b & 2047) << 4) | (b >> 11); }

// Ratio-test candidate test for nonbasic variable j with tableau entry alpha.
// Returns false if j cannot bound the dual step.  abar = sigma*alpha.
__device__ __forceinline__ bool candidate(const DeviceModel &d, int j, double alpha, int sigma,
                                          double &a, double &dtil, bool &boxed, double &range)
{
  const unsigned char st = d.status[j];
  if (st == basic || st == isFixed)
    return false;
  const double ab = sigma * alpha;
  a = fabs(ab);
  if (a <= 1.0e-12)
    return false;
  const double dj = d.dj[j];
  boxed = false;
  range = 0.0;
  if (st == atLowerBound) {
    if (ab <= 0.0)
      return false;
    dtil = dj > 0.0 ? dj : 0.0;
  } else if (st == atUpperBound) {
    if (ab >= 0.0)
      return false;
    dtil = dj < 0.0 ? -dj : 0.0;
  } else {
    dtil = 0.0;
    return true;
  }
  range = d.upper[j] - d.lower[j];
  boxed = range < 1.0e29;
  return true;
}

// slope contribution of a candidate in 2^-40 fixed point relative to the primal infeasibility
__device__ __forceinline__ unsigned long long slope_weight(double a, bool boxed, double range, double infeas)
{
  unsigned long long w = kFixCap;
  if (boxed) {
    double v = a * range / infeas * 1099511627776.0;
    w = v >= 2199023255552.0 ? kFixCap : (unsigned long long)v;
    if (w == 0ull)
      w = 1ull; // a bucket with a candidate is never "empty"
  }
  return w;
}


// order independent histogram add with warp aggregation: lanes of a warp that hit the same bucket
// are summed first (one atomic per distinct bucket and warp).  Degenerate LPs put thousands of
// candidates into the ratio-0 bucket; without aggregation those atomics serialise in L2.
// Must be called by all 32 lanes of a converged warp; w < 2^42.
// sHot (optional): shared-memory accumulator of the CTA for bucket 0 (ratio exactly 0: the dual
// degenerate candidates); the caller flushes it with one global atomic per CTA.
__device__ __forceinline__ void hist_add_aggregated(unsigned long long *hist, int bucket,
                                                    unsigned long long w, bool valid,
                                                    unsigned long long *sHot = nullptr)
{
  const unsigned act = __ballot_sync(0xffffffffu, valid);
  if (!valid)
    return;
  const unsigned peers = __match_any_sync(act, bucket);
  const unsigned lo = (unsigned)(w & 0xFFFFFull), hi = (unsigned)(w >> 20);
  const unsigned slo = __reduce_add_sync(peers, lo), shi = __reduce_add_sync(peers, hi);
  if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) {
    const unsigned long long sum = ((unsigned long long)shi << 20) + (unsigned long long)slo;
    if (sHot != nullptr && bucket == 0)
      atomicAdd(sHot, sum);
    else
      atomicAdd(hist + bucket, sum);
  }
}
// warp-aggregated atomicMax of an int per bucket (all 32 lanes call it; valid lanes take part)
__device__ __forceinline__ void max_aggregated(int *arr, int bucket, int value, bool valid)
{
  const unsigned act = __ballot_sync(0xffffffffu, valid);
  if (!valid)
    return;
  const unsigned peers = __match_any_sync(act, bucket);
  const int mx = __reduce_max_sync(peers, value);
  if ((int)(threadIdx.x & 31) == __ffs(peers) - 1)
    atomicMax(arr + bucket, mx);
}
// same for atomicMin of 64-bit keys (called by the lanes with valid == true of the call above)
__device__ __forceinline__ void hist_min_aggregated(unsigned long long *hist, int bucket,
                                                    unsigned long long key, bool valid,
                                                    unsigned long long *sHotMin = nullptr)
{
  const unsigned act = __ballot_sync(0xffffffffu, valid);
  if (!valid)
    return;
  const unsigned peers = __match_any_sync(act, bucket);
  const unsigned hi = (unsigned)(key >> 32);
  const unsigned mh = __reduce_min_sync(peers, hi);
  const unsigned lo = hi == mh ? (unsigned)key : 0xFFFFFFFFu;
  const unsigned ml = __reduce_min_sync(peers, lo);
  if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) {
    const unsigned long long mn = ((unsigned long long)mh << 32) | (unsigned long long)ml;
    if (sHotMin != nullptr && bucket == 0)
      atomicMin(sHotMin, mn);
    else
      atomicMin(hist + bucket, mn);
  }
}

} // namespace clpb
