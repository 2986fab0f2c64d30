// ranging.cu -- batched sensitivity analysis (ClpSimplex::dualRanging / primalRanging,
// src/ClpSimplexOther.cpp:50-374, :770-1001) on the fresh factors a status-0 dual() leaves behind.
//
// The reference ranges one variable at a time: a BTRAN + a full transposeTimes per basic variable, an
// FTRAN + an m-long ratio test per nonbasic one.  Here kRangeBatch (16) of them share one pass, and the
// factors' block structure (DESIGN.md "Basis factors") removes the GEMVs:
//   row r of B0^-1:  nucleus position -> row posToNuc[r] of Ninv, scattered by nucRow, 0 on C;
//                    slack position   -> -e_r on C, sum_j S1[r,j] Ninv[j,:] on N
//   B0^-1 a:         y = sum_{i in supp(a), posToNuc[i] >= 0} a_i NinvT[posToNuc[i],:];  x_C = S1 y - a_C
// Every ratio test keeps the best (ratio, sequence) per CTA and right-hand side; a second kernel reduces
// the CTAs in a fixed order.  Comparisons are exact (no packed key), so the result does not depend on
// the order in which CTAs finish.
#include "engine.hpp"
#include "kernels_common.cuh"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <map>
#include <stdexcept>

namespace clpb {

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr double kDualNone = 1.0e31;   // checkDualRatios starts thetaUp / thetaDown here (:277-278)
constexpr double kPrimalNone = 1.0e30; // checkPrimalRatios starts theta_ here (:970)

struct Best {
  double r;
  int s;
};

// smaller ratio wins; equal ratios go to the smaller sequence (columns before rows)
__device__ __forceinline__ void take(Best &b, double r, int s)
{
  if (r < b.r || (r == b.r && s < b.s)) {
    b.r = r;
    b.s = s;
  }
}

__device__ __forceinline__ Best shfl_best(Best b, int mask)
{
  Best o;
  o.r = __shfl_xor_sync(kFull, b.r, mask);
  o.s = __shfl_xor_sync(kFull, b.s, mask);
  return o;
}

// checkDualRatios (:301-361) for one candidate: alpha is the tableau-row entry in the reference's sign
// (alpha_j = -rho^T a_j), dj / status the working values of sequence j.
__device__ __forceinline__ void dual_candidate(double alpha, double dj, unsigned char st, int j, double tol,
                                               Best &up, Best &down)
{
  if (fabs(alpha) < 1.0e-9 || st == basic || st == isFixed)
    return;
  double ru = kDualNone, rd = kDualNone;
  if (st == isFree || st == superBasic) {
    ru = rd = 0.0;
  } else if (st == atUpperBound) {
    if (alpha > 0.0)
      ru = (tol - dj) / alpha;
    else
      rd = -(tol - dj) / alpha;
  } else { // atLowerBound
    if (alpha < 0.0)
      ru = -(tol + dj) / alpha;
    else
      rd = (tol + dj) / alpha;
  }
  if (ru < kDualNone)
    take(up, ru, j);
  if (rd < kDualNone)
    take(down, rd, j);
}

// ---- 1. rows of B0^-1 for the positions w.seq[b]: rho[i][b] (thread per nucleus row, blockIdx.y = b)
__global__ void __launch_bounds__(256) range_rho_kernel(DeviceModel d, RangeWork w)
{
  const int b = blockIdx.y;
  const int p = w.seq[b];
  const int nuc = d.posToNuc[p];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (nuc < 0 && i == 0)
    w.rho[(size_t)p * kRangeBatch + b] = -1.0; // -e_p on C
  if (i >= d.k)
    return;
  double v;
  if (nuc >= 0) {
    v = d.Ninv[(size_t)nuc * d.ldk + i];
  } else {
    v = 0.0;
    for (int e = d.s1RowStart[p]; e < d.s1RowStart[p + 1]; e++)
      v = fma(d.s1Val[e], d.Ninv[(size_t)d.s1Col[e] * d.ldk + i], v);
  }
  w.rho[(size_t)d.nucRow[i] * kRangeBatch + b] = v;
}

// ---- 2. multi-right-hand-side PRICE fused with the two-sided dual ratio test.
// Columns: one warp per column, lanes over its entries, 16 accumulators per lane (one 128-byte rho row
// per entry); after the warp sum lane b owns right-hand side b.  Rows: thread per (row, b) entry of rho,
// alpha_{n+i} = rho_i.  Lane b and lane b+16 then hold bests of the same b and are merged.
__global__ void __launch_bounds__(256) range_dual_price_kernel(DeviceModel d, RangeWork w, int nb, double tol)
{
  __shared__ Best sUp[8][kRangeBatch], sDown[8][kRangeBatch];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gwarp = blockIdx.x * 8 + warp, nwarps = gridDim.x * 8;
  Best up{kDualNone, -1}, down{kDualNone, -1};
  for (int j = gwarp; j < d.n; j += nwarps) {
    const unsigned char st = d.status[j];
    if (st == basic || st == isFixed)
      continue;
    double acc[kRangeBatch];
#pragma unroll
    for (int b = 0; b < kRangeBatch; b++)
      acc[b] = 0.0;
    for (int e = d.colStart[j] + lane; e < d.colStart[j + 1]; e += 32) {
      const double a = d.val[e];
      const double2 *row = reinterpret_cast<const double2 *>(w.rho + (size_t)d.rowIdx[e] * kRangeBatch);
#pragma unroll
      for (int q = 0; q < kRangeBatch / 2; q++) {
        const double2 r2 = row[q];
        acc[2 * q] = fma(a, r2.x, acc[2 * q]);
        acc[2 * q + 1] = fma(a, r2.y, acc[2 * q + 1]);
      }
    }
    double alpha = 0.0;
#pragma unroll
    for (int b = 0; b < kRangeBatch; b++) {
      const double sum = warp_sum(acc[b]);
      if (lane == b)
        alpha = -sum; // transposeTimes(-1.0, ...) at :117
    }
    if (lane < nb)
      dual_candidate(alpha, d.dj[j], st, j, tol, up, down);
  }
  // slack part: the stride is a multiple of 32, so every thread keeps the same b = lane & 15
  const int b = lane & (kRangeBatch - 1);
  if (b < nb) {
    for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < (size_t)d.m * kRangeBatch;
         idx += (size_t)gridDim.x * blockDim.x) {
      const int seq = d.n + (int)(idx / kRangeBatch);
      dual_candidate(w.rho[idx], d.dj[seq], d.status[seq], seq, tol, up, down);
    }
  }
  {
    const Best u2 = shfl_best(up, 16), d2 = shfl_best(down, 16);
    take(up, u2.r, u2.s);
    take(down, d2.r, d2.s);
  }
  if (lane < kRangeBatch) {
    sUp[warp][lane] = up;
    sDown[warp][lane] = down;
  }
  __syncthreads();
  if (threadIdx.x < 2 * kRangeBatch) {
    const int dir = threadIdx.x / kRangeBatch, bb = threadIdx.x % kRangeBatch;
    Best best{kDualNone, -1};
    for (int q = 0; q < 8; q++) {
      const Best o = dir == 0 ? sUp[q][bb] : sDown[q][bb];
      take(best, o.r, o.s);
    }
    const size_t slot = ((size_t)dir * kRangeBatch + bb) * kRangeBlocks + blockIdx.x;
    w.partRatio[slot] = best.r;
    w.partSeq[slot] = best.s;
  }
}

// ---- fixed-order reduction of the per-CTA bests: one thread per (direction, b)
__global__ void range_final_kernel(RangeWork w, int blocks, double none)
{
  const int t = threadIdx.x; // dir * kRangeBatch + b
  if (t >= 2 * kRangeBatch)
    return;
  Best best{none, -1};
  for (int q = 0; q < blocks; q++)
    take(best, w.partRatio[(size_t)t * kRangeBlocks + q], w.partSeq[(size_t)t * kRangeBlocks + q]);
  w.outRatio[t] = best.r;
  w.outSeq[t] = best.s;
}

// ---- 3. FTRAN of the sparse columns w.seq[b] (column of [A | -I], ClpSimplex::unpackPacked):
// y[b][i] = sum over the column's nucleus rows of a * NinvT[posToNuc[row]][i]  (thread per i)
__global__ void __launch_bounds__(256) range_ftran_y_kernel(DeviceModel d, RangeWork w, int ldy)
{
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d.k)
    return;
  const int seq = w.seq[b];
  double v = 0.0;
  if (seq < d.n) {
    for (int e = d.colStart[seq]; e < d.colStart[seq + 1]; e++) {
      const int p = d.posToNuc[d.rowIdx[e]];
      if (p >= 0)
        v = fma(d.val[e], d.NinvT[(size_t)p * d.ldk + i], v);
    }
  } else {
    const int p = d.posToNuc[seq - d.n];
    if (p >= 0)
      v = -d.NinvT[(size_t)p * d.ldk + i]; // the slack column is -e_i
  }
  w.y[(size_t)b * ldy + i] = v;
}

// x[b][p] = y[b][posToNuc[p]] on N; sum_j S1[p,j] y[b][j] on C (thread per position)
__global__ void __launch_bounds__(256) range_ftran_x_kernel(DeviceModel d, RangeWork w, int ldy)
{
  const int b = blockIdx.y;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= d.m)
    return;
  const double *y = w.y + (size_t)b * ldy;
  const int nuc = d.posToNuc[p];
  double v;
  if (nuc >= 0) {
    v = y[nuc];
  } else {
    v = 0.0;
    for (int e = d.s1RowStart[p]; e < d.s1RowStart[p + 1]; e++)
      v = fma(d.s1Val[e], y[d.s1Col[e]], v);
  }
  w.x[(size_t)b * d.m + p] = v;
}

// x_C -= a_C (one CTA per right-hand side; distinct rows, no races)
__global__ void __launch_bounds__(256) range_ftran_rhs_kernel(DeviceModel d, RangeWork w)
{
  const int b = blockIdx.x;
  const int seq = w.seq[b];
  double *x = w.x + (size_t)b * d.m;
  if (seq >= d.n) {
    const int r = seq - d.n;
    if (threadIdx.x == 0 && d.posToNuc[r] < 0)
      x[r] += 1.0;
    return;
  }
  for (int e = d.colStart[seq] + threadIdx.x; e < d.colStart[seq + 1]; e += blockDim.x) {
    const int r = d.rowIdx[e];
    if (d.posToNuc[r] < 0)
      x[r] -= d.val[e];
  }
}

// ---- 4. primal ratio over the positions, both directions at once (way +1 and -1 of checkPrimalRatios):
// theta = max(0, (x - bound) / alpha), smallest theta wins, ties to the smallest sequence; infinite
// bounds never block.  The position of w.other[b] is left out and its entry reported (primalRanging1).
__global__ void __launch_bounds__(256) range_primal_ratio_kernel(DeviceModel d, RangeWork w)
{
  __shared__ Best sUp[8], sDown[8];
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int other = w.other[b];
  const double *x = w.x + (size_t)b * d.m;
  Best up{kPrimalNone, -1}, down{kPrimalNone, -1};
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < d.m; p += gridDim.x * blockDim.x) {
    const int seq = d.pivotVariable[p];
    const double raw = x[p];
    if (seq == other) {
      w.alphaOther[b] = raw;
      continue;
    }
    if (!(fabs(raw) > 1.0e-7))
      continue;
    const double v = d.sol[seq], lo = d.lower[seq], hi = d.upper[seq];
#pragma unroll
    for (int way = 1; way >= -1; way -= 2) {
      const double alpha = raw * way;
      const double bound = alpha > 0.0 ? lo : hi; // towards the lower bound when alpha > 0
      if (bound <= -kInf || bound >= kInf)
        continue;
      const double theta = fmax(0.0, (v - bound) / alpha);
      if (theta < kPrimalNone)
        take(way > 0 ? up : down, theta, seq);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const Best u2 = shfl_best(up, o), d2 = shfl_best(down, o);
    take(up, u2.r, u2.s);
    take(down, d2.r, d2.s);
  }
  if (lane == 0) {
    sUp[warp] = up;
    sDown[warp] = down;
  }
  __syncthreads();
  if (threadIdx.x < 2) {
    Best best{kPrimalNone, -1};
    for (int q = 0; q < 8; q++) {
      const Best o = threadIdx.x == 0 ? sUp[q] : sDown[q];
      take(best, o.r, o.s);
    }
    const size_t slot = ((size_t)threadIdx.x * kRangeBatch + b) * kRangeBlocks + blockIdx.x;
    w.partRatio[slot] = best.r;
    w.partSeq[slot] = best.s;
  }
}

inline int grid_for(long long work, int perBlock)
{
  long long g = (work + perBlock - 1) / perBlock;
  const long long cap = std::min<long long>(kRangeBlocks, 4ll * device_sm_count());
  return (int)std::max(1ll, std::min(g, cap));
}

} // namespace

void launch_range_dual(const DeviceModel &d, const RangeWork &w, int nb, double dualTolerance, cudaStream_t s)
{
  cudaMemsetAsync(w.rho, 0, sizeof(double) * (size_t)d.m * kRangeBatch, s);
  range_rho_kernel<<<dim3((std::max(d.k, 1) + 255) / 256, nb), 256, 0, s>>>(d, w);
  const int blocks = grid_for(std::max<long long>((long long)d.n * 32, (long long)d.m * kRangeBatch), 256);
  range_dual_price_kernel<<<blocks, 256, 0, s>>>(d, w, nb, dualTolerance);
  range_final_kernel<<<1, 2 * kRangeBatch, 0, s>>>(w, blocks, kDualNone);
}

void launch_range_primal(const DeviceModel &d, const RangeWork &w, int nb, cudaStream_t s)
{
  const int ldy = (d.m + 7) / 8 * 8;
  cudaMemsetAsync(w.alphaOther, 0, sizeof(double) * kRangeBatch, s);
  if (d.k > 0)
    range_ftran_y_kernel<<<dim3((d.k + 255) / 256, nb), 256, 0, s>>>(d, w, ldy);
  range_ftran_x_kernel<<<dim3((d.m + 255) / 256, nb), 256, 0, s>>>(d, w, ldy);
  range_ftran_rhs_kernel<<<nb, 256, 0, s>>>(d, w);
  const int blocks = grid_for((long long)d.m, 256);
  range_primal_ratio_kernel<<<dim3(blocks, nb), 256, 0, s>>>(d, w);
  range_final_kernel<<<1, 2 * kRangeBatch, 0, s>>>(w, blocks, kPrimalNone);
}

// ---------------------------------------------------------------------------------------------
// host side: Engine::dualRanging / primalRanging

#define RANGE_CUDA_OK(call)                                                                       \
  do {                                                                                            \
    cudaError_t e__ = (call);                                                                     \
    if (e__ != cudaSuccess) {                                                                     \
      fprintf(stderr, "clp_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__,    \
              __LINE__);                                                                          \
      throw std::runtime_error("CUDA error");                                                     \
    }                                                                                             \
  } while (0)

// working-units copy of what the ratio tests read, taken once per call
struct Engine::RangeSnapshot {
  std::vector<double> sol, dj;
  std::vector<unsigned char> st;
  std::vector<int> backPivot; // position of each basic sequence, -1 for nonbasics
  // ClpSimplexOther.cpp:215-227 (costs) and :824-840 (values); the engine has no objective / rhs scale
  const Engine *e;
  double costScale(int seq) const
  {
    return e->rowScale.empty() ? 1.0 : seq < e->n ? 1.0 / e->columnScale[seq] : e->rowScale[seq - e->n];
  }
  double valueScale(int seq) const
  {
    return e->rowScale.empty() ? 1.0 : seq < e->n ? e->columnScale[seq] : 1.0 / e->rowScale[seq - e->n];
  }
};

int Engine::rangingSnapshot(RangeSnapshot &r)
{
  if (!optimalOnDevice || !deviceReady || !factorsValid || d.shardW > 1 || deviceSignature() != readySignature)
    return 1;
  fetchState();
  if (hState->numEtas != 0) {
    // dual() reports status 0 only on fresh factors, so this does not happen; should it ever, the batched
    // kernels (which read B0^-1 only) get fresh factors of the same basis instead of wrong ranges
    fprintf(stderr, "clp_b200: ranging found %d updates on the optimal factors; refactorizing\n", hState->numEtas);
    if (refactor() != 0)
      return 1;
  }
  r.e = this;
  r.sol.resize(nm);
  r.dj.resize(nm);
  r.st.resize(nm);
  std::vector<int> pivot(m);
  RANGE_CUDA_OK(cudaMemcpyAsync(r.sol.data(), d.sol, sizeof(double) * nm, cudaMemcpyDeviceToHost, stream));
  RANGE_CUDA_OK(cudaMemcpyAsync(r.dj.data(), d.dj, sizeof(double) * nm, cudaMemcpyDeviceToHost, stream));
  RANGE_CUDA_OK(cudaMemcpyAsync(r.st.data(), d.status, nm, cudaMemcpyDeviceToHost, stream));
  RANGE_CUDA_OK(cudaMemcpyAsync(pivot.data(), d.pivotVariable, sizeof(int) * m, cudaMemcpyDeviceToHost, stream));
  RANGE_CUDA_OK(cudaStreamSynchronize(stream));
  r.backPivot.assign(nm, -1);
  for (int p = 0; p < m; p++)
    r.backPivot[pivot[p]] = p;
  return 0;
}

// One batch of up to kRangeBatch right-hand sides.  ratio / seq: [2][kRangeBatch] (up, down);
// alphaOther: [kRangeBatch] (primal passes only).
void Engine::rangePass(bool dual, const int *seqs, const int *others, int nb, double *ratio, int *seq,
                       double *alphaOther)
{
  RANGE_CUDA_OK(cudaMemcpyAsync(rw.seq, seqs, sizeof(int) * nb, cudaMemcpyHostToDevice, stream));
  if (dual) {
    launch_range_dual(d, rw, nb, dualTolerance, stream);
  } else {
    RANGE_CUDA_OK(cudaMemcpyAsync(rw.other, others, sizeof(int) * nb, cudaMemcpyHostToDevice, stream));
    launch_range_primal(d, rw, nb, stream);
  }
  RANGE_CUDA_OK(cudaGetLastError());
  RANGE_CUDA_OK(cudaMemcpyAsync(ratio, rw.outRatio, sizeof(double) * 2 * kRangeBatch, cudaMemcpyDeviceToHost, stream));
  RANGE_CUDA_OK(cudaMemcpyAsync(seq, rw.outSeq, sizeof(int) * 2 * kRangeBatch, cudaMemcpyDeviceToHost, stream));
  if (!dual)
    RANGE_CUDA_OK(cudaMemcpyAsync(alphaOther, rw.alphaOther, sizeof(double) * kRangeBatch, cudaMemcpyDeviceToHost,
                                  stream));
  RANGE_CUDA_OK(cudaStreamSynchronize(stream));
}

namespace {

struct RangeResult {
  double up = 0.0, down = 0.0, alphaOther = 0.0;
  int seqUp = -1, seqDown = -1;
};

// Runs every distinct key through batches of kRangeBatch.  Dual keys: (basic sequence, -1); primal keys:
// (entering sequence, excluded sequence or -1).
template <class Pass>
void run_batches(std::map<std::pair<int, int>, RangeResult> &jobs, Pass pass)
{
  std::vector<std::map<std::pair<int, int>, RangeResult>::iterator> batch;
  auto flush = [&]() {
    if (batch.empty())
      return;
    int seqs[kRangeBatch], others[kRangeBatch], seqOut[2 * kRangeBatch];
    double ratio[2 * kRangeBatch], alphaOther[kRangeBatch];
    const int nb = (int)batch.size();
    for (int b = 0; b < nb; b++) {
      seqs[b] = batch[b]->first.first;
      others[b] = batch[b]->first.second;
    }
    pass(seqs, others, nb, ratio, seqOut, alphaOther);
    for (int b = 0; b < nb; b++) {
      RangeResult &res = batch[b]->second;
      res.up = ratio[b];
      res.seqUp = seqOut[b];
      res.down = ratio[kRangeBatch + b];
      res.seqDown = seqOut[kRangeBatch + b];
      res.alphaOther = alphaOther[b];
    }
    batch.clear();
  };
  for (auto it = jobs.begin(); it != jobs.end(); ++it) {
    batch.push_back(it);
    if ((int)batch.size() == kRangeBatch)
      flush();
  }
  flush();
}

} // namespace

// ClpSimplexOther::dualRanging (:50-260) with checkDualRatios (:266-374); the value pass is primalRanging1
// (:848-953).  Restated with one rule per side: the smallest ratio wins and ties go to the smallest
// sequence, so the answer does not depend on the order in which the device visits the candidates.
int Engine::dualRanging(int numberCheck, const int *which, double *costIncrease, int *sequenceIncrease,
                        double *costDecrease, int *sequenceDecrease, double *valueIncrease, double *valueDecrease)
{
  for (int i = 0; i < numberCheck; i++)
    if (which[i] >= nm)
      return -1;
  RangeSnapshot r;
  if (rangingSnapshot(r) != 0)
    return 1;
  const bool values = valueIncrease != nullptr && valueDecrease != nullptr;
  // tableau rows of the basic variables asked for
  std::map<std::pair<int, int>, RangeResult> dualJobs, primalJobs;
  for (int i = 0; i < numberCheck; i++)
    if (which[i] >= 0 && r.st[which[i]] == basic)
      dualJobs[{which[i], -1}];
  const int *backPivot = r.backPivot.data();
  run_batches(dualJobs, [&](const int *seqs, const int *, int nb, double *ratio, int *seq, double *) {
    int pos[kRangeBatch];
    for (int b = 0; b < nb; b++)
      pos[b] = backPivot[seqs[b]];
    rangePass(true, pos, nullptr, nb, ratio, seq, nullptr);
  });
  // primalRanging1(whichIn, whichOther): FTRAN of whichIn, ratio test without whichOther's position
  auto atBound = [&](int seq) { return seq >= 0 && (r.st[seq] == atLowerBound || r.st[seq] == atUpperBound); };
  if (values) {
    for (int i = 0; i < numberCheck; i++) {
      const int j = which[i];
      if (j < 0)
        continue;
      if (r.st[j] == basic) {
        const RangeResult &res = dualJobs[{j, -1}];
        // a free or superbasic entering variable keeps the current value (the reference asserts there, :857)
        if (atBound(res.seqUp))
          primalJobs[{res.seqUp, j}];
        if (atBound(res.seqDown))
          primalJobs[{res.seqDown, j}];
      } else if (atBound(j)) {
        primalJobs[{j, j}];
      }
    }
    run_batches(primalJobs, [&](const int *seqs, const int *others, int nb, double *ratio, int *seq, double *ao) {
      rangePass(false, seqs, others, nb, ratio, seq, ao);
    });
  }
  auto userValue = [&](int seq) { return r.sol[seq] * r.valueScale(seq); };
  auto primalRanging1 = [&](int whichIn, int whichOther) {
    const RangeResult &res = primalJobs[{whichIn, whichOther}];
    const int wayIn = r.st[whichIn] == atLowerBound ? 1 : -1;
    const double theta = wayIn > 0 ? res.up : res.down;
    const double alphaOther = res.alphaOther * wayIn;
    double v = r.sol[whichOther];
    if (whichIn != whichOther)
      v = theta < 1.0e30 ? v - theta * alphaOther : (alphaOther > 0.0 ? -1.0e30 : 1.0e30);
    else
      v += theta * wayIn;
    if (v >= 1.0e29)
      return DBL_MAX;
    if (v <= -1.0e29)
      return -DBL_MAX;
    return v * r.valueScale(whichOther);
  };
  for (int i = 0; i < numberCheck; i++) {
    const int j = which[i];
    if (j < 0) { // :85-91
      costIncrease[i] = 0.0;
      sequenceIncrease[i] = -1;
      costDecrease[i] = 0.0;
      sequenceDecrease[i] = -1;
      continue;
    }
    double up = DBL_MAX, down = DBL_MAX;
    int seqUp = -1, seqDown = -1;
    double vUp = 0.0, vDown = 0.0;
    if (values)
      vUp = vDown = userValue(j);
    switch (r.st[j]) {
    case basic: {
      const RangeResult &res = dualJobs[{j, -1}];
      if (res.seqUp >= 0) {
        up = res.up;
        seqUp = res.seqUp;
        if (values && atBound(seqUp))
          vUp = primalRanging1(seqUp, j);
      }
      if (res.seqDown >= 0) {
        down = res.down;
        seqDown = res.seqDown;
        if (values && atBound(seqDown))
          vDown = primalRanging1(seqDown, j);
      }
    } break;
    case isFixed:
      break;
    case isFree:
    case superBasic:
      up = down = 0.0;
      seqUp = seqDown = j;
      break;
    case atUpperBound:
      up = std::max(0.0, -r.dj[j]);
      seqUp = j;
      if (values)
        vUp = primalRanging1(j, j);
      break;
    case atLowerBound:
      down = std::max(0.0, r.dj[j]);
      seqDown = j;
      if (values)
        vDown = primalRanging1(j, j);
      break;
    }
    const double scale = r.costScale(j);
    if (up < 1.0e30)
      up *= scale;
    if (down < 1.0e30)
      down *= scale;
    costIncrease[i] = up;
    sequenceIncrease[i] = seqUp;
    costDecrease[i] = down;
    sequenceDecrease[i] = seqDown;
    if (values) {
      valueIncrease[i] = vUp;
      valueDecrease[i] = vDown;
    }
  }
  return 0;
}

// ClpSimplexOther::primalRanging (:770-846) with checkPrimalRatios (:958-1001).  For basic, free and
// superbasic variables the reference's own assignment is kept literally (:792-793):
// valueDecrease = max(0, upper - x) and valueIncrease = max(0, x - lower), although the names read swapped.
int Engine::primalRanging(int numberCheck, const int *which, double *valueIncrease, int *sequenceIncrease,
                          double *valueDecrease, int *sequenceDecrease)
{
  for (int i = 0; i < numberCheck; i++)
    if (which[i] < 0 || which[i] >= nm)
      return -1;
  RangeSnapshot r;
  if (rangingSnapshot(r) != 0)
    return 1;
  auto easy = [&](int seq) { return r.st[seq] == basic || r.st[seq] == isFree || r.st[seq] == superBasic; };
  std::map<std::pair<int, int>, RangeResult> jobs;
  for (int i = 0; i < numberCheck; i++)
    if (!easy(which[i]))
      jobs[{which[i], -1}];
  run_batches(jobs, [&](const int *seqs, const int *others, int nb, double *ratio, int *seq, double *ao) {
    rangePass(false, seqs, others, nb, ratio, seq, ao);
  });
  // working bounds of the basic / free variables (the nonbasic ones are only read on the device)
  std::vector<double> lo(nm), hi(nm);
  RANGE_CUDA_OK(cudaMemcpyAsync(lo.data(), d.lower, sizeof(double) * nm, cudaMemcpyDeviceToHost, stream));
  RANGE_CUDA_OK(cudaMemcpyAsync(hi.data(), d.upper, sizeof(double) * nm, cudaMemcpyDeviceToHost, stream));
  RANGE_CUDA_OK(cudaStreamSynchronize(stream));
  for (int i = 0; i < numberCheck; i++) {
    const int j = which[i];
    double up = DBL_MAX, down = DBL_MAX;
    int seqUp = -1, seqDown = -1;
    if (easy(j)) {
      down = std::max(0.0, hi[j] - r.sol[j]);
      up = std::max(0.0, r.sol[j] - lo[j]);
      seqUp = seqDown = j;
    } else {
      const RangeResult &res = jobs[{j, -1}];
      if (res.seqUp >= 0) {
        up = res.up;
        seqUp = res.seqUp;
      }
      if (res.seqDown >= 0) {
        down = res.down;
        seqDown = res.seqDown;
      }
    }
    const double scale = r.valueScale(j);
    up = up < 1.0e30 ? up * scale : DBL_MAX;
    down = down < 1.0e30 ? down * scale : DBL_MAX;
    valueIncrease[i] = up;
    sequenceIncrease[i] = seqUp;
    valueDecrease[i] = down;
    sequenceDecrease[i] = seqDown;
  }
  return 0;
}

} // namespace clpb
