// update.cu -- CHUZR, dual/primal/weight updates and the refresh (recompute-from-scratch) kernels.
//
// Replaces, with device-resident state,
//   ClpDualRowSteepest::pivotRow            /root/reference/src/ClpDualRowSteepest.cpp:179
//   ClpDualRowSteepest::updateWeights       src/ClpDualRowSteepest.cpp:375 (recurrence :501-538)
//   ClpDualRowSteepest::updatePrimalSolution src/ClpDualRowSteepest.cpp:630
//   ClpSimplex::housekeeping                src/ClpSimplex.cpp:2065 (status / pivotVariable swap)
//   ClpSimplexDual::changeBounds            src/ClpSimplexDual.cpp:3148 (fake bounds)
//   ClpSimplex::computePrimals / computeDuals  src/ClpSimplex.cpp:914 / :1164
// All reductions are order independent (packed-key atomicMax/Min, integer atomics) or done
// in a fixed order, so replicated ranks of a column-sharded run stay bit-identical.  The dual
// update and the bound flips run in the row pass (rowpass.cu).
#include "kernels_common.cuh"

namespace clpb {

// ------------------------------------------------------------------ CHUZR
// Stand-alone row choice: used at the start of a batch of iterations (after a refresh the primal
// values are new).  Inside a batch the row of the next iteration is chosen by the update kernel
// of the previous one (iteration_update_kernel), which has every x_B and weight in registers.
__global__ void chuzr_kernel(DeviceModel d)
{
  if (!iter_active(d.st))
    return;
  const double tol = d.primalTolerance;
  unsigned long long best = 0ull;
  // clear the ratio-test histograms for this iteration (the previous scans are complete)
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < kHistBuckets; b += gridDim.x * blockDim.x) {
    d.histWeight[b] = 0ull;
    if (b < kHist2Buckets) {
      d.hist2Weight[b] = 0ull;
      d.hist2Min[b] = 0xFFFFFFFFFFFFFFFFull;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x < kHistBuckets / 1024) {
    d.segTotal[threadIdx.x] = 0ull;
    d.segLast[threadIdx.x] = -1;
  }
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < d.m; p += gridDim.x * blockDim.x) {
    const int seq = d.pivotVariable[p];
    if (!d.flagged[p])
      best = max(best, chuzr_key(d.sol[seq], d.lower[seq], d.upper[seq], d.dantzig ? 1.0 : d.weights[p], tol, p));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best != 0ull)
    atomicMax(&d.st->chuzrKey, best);
}

// decode the packed argmax into pivotRow / seqOut / sigma / infeas (single thread).
// coherentSol: the caller runs as the tail of a kernel that wrote d.sol in other CTAs.
__device__ __forceinline__ void chuzr_finish_body(const DeviceModel &d, unsigned long long key, bool coherentSol)
{
  IterState *st = d.st;
  if (st->numEtas >= d.tmax) {
    st->stop = STOP_ETAS_FULL;
    return;
  }
  if (key == 0ull) {
    st->stop = STOP_NO_ROW;
    return;
  }
  const int r = 0xFFFFF - (int)(key & 0xFFFFFull);
  const int seq = d.pivotVariable[r];
  const double v = coherentSol ? __ldcg(d.sol + seq) : d.sol[seq];
  st->pivotRow = r;
  st->seqOut = seq;
  if (v < d.lower[seq]) {
    st->sigma = -1;
    st->infeas = d.lower[seq] - v;
  } else {
    st->sigma = +1;
    st->infeas = v - d.upper[seq];
  }
  st->numFlips = 0;
  st->seqIn = -1;
}

__global__ void chuzr_finish_kernel(DeviceModel d)
{
  IterState *st = d.st;
  if (!iter_active(st))
    return;
  const unsigned long long key = st->chuzrKey;
  st->chuzrKey = 0ull;
  chuzr_finish_body(d, key, false);
}

void launch_chuzr(const DeviceModel &d, cudaStream_t s)
{
  int blocks = (d.m + 255) / 256;
  if (blocks > device_sm_count() * 4)
    blocks = device_sm_count() * 4;
  if (blocks < 32)
    blocks = 32; // also clears the ratio-test histograms
  chuzr_kernel<<<blocks, 256, 0, s>>>(d);
  chuzr_finish_kernel<<<1, 1, 0, s>>>(d);
}

// ------------------------------------------------------------------ after the FTRANs
// status / pivotVariable swap and per-iteration record (ClpSimplex::housekeeping), single thread
__device__ __forceinline__ void pivot_fixup_body(const DeviceModel &d)
{
  IterState *st = d.st;
  IterRecord &rec = d.rec[st->iterations % d.recCap];
  const int r = st->pivotRow, q = st->seqIn, out = st->seqOut;
  const double bound = st->sigma < 0 ? d.lower[out] : d.upper[out];
  d.sol[q] += st->thetaPrimal;
  d.sol[out] = bound;
  d.dj[q] = 0.0;
  d.dj[out] = -st->sigma * st->thetaDual;
  d.status[q] = basic;
  d.lower[q] = d.lowerTrue[q];
  d.upper[q] = d.upperTrue[q];
  d.fake[q] = 0;
  d.status[out] = (d.lower[out] == d.upper[out]) ? isFixed
                  : (st->sigma < 0 ? atLowerBound : atUpperBound);
  d.pivotVariable[r] = q;
  const int t = st->numEtas;
  d.etaPos[t] = r;
  d.etaPrevSame[t] = d.etaLastOfPos[r];
  d.etaLastOfPos[r] = t;
  st->numEtas = t + 1;
  rec.stop = 0;
  rec.pivotRow = r;
  rec.seqIn = q;
  rec.seqOut = out;
  rec.sigma = st->sigma;
  rec.numFlips = st->numFlips;
  rec.thetaDual = st->thetaDual;
  rec.thetaPrimal = st->thetaPrimal;
  rec.alphaRow = st->alphaRow;
  rec.alphaCol = st->alphaCol;
  rec.infeas = st->infeas;
  st->iterations += 1;
}

// End of an iteration in one kernel:
//   CTAs [0, etaBlocks)      : new row of Ginv / column of GinvT from the BTRAN's nu (eta_append_row)
//   CTAs [etaBlocks, grid)   : x_B, DSE weights (ClpDualRowSteepest.cpp:501-538) and the new eta
//                              column, one thread per position; clear the ratio-test histograms;
//                              score every position for the NEXT iteration's CHUZR
//   tail (last CTA, thread 0): housekeeping of this iteration, then decode the next pivot row.
__global__ void __launch_bounds__(256) iteration_update_kernel(DeviceModel d, int etaBlocks)
{
  IterState *st = d.st;
  if (!iter_active(st)) {
    if (blockIdx.x == 0 && threadIdx.x == 0)
      d.rec[st->iterations % d.recCap].stop = st->stop;
    return;
  }
  if ((int)blockIdx.x < etaBlocks) {
    eta_append_row(d, blockIdx.x * 256 + threadIdx.x, etaBlocks * 256);
  } else {
    const int posBlocks = gridDim.x - etaBlocks;
    const int gtid = (blockIdx.x - etaBlocks) * 256 + threadIdx.x;
    const int gthreads = posBlocks * 256;
    for (int b = gtid; b < kHistBuckets; b += gthreads) {
      d.histWeight[b] = 0ull;
      if (b < kHist2Buckets) {
        d.hist2Weight[b] = 0ull;
        d.hist2Min[b] = 0xFFFFFFFFFFFFFFFFull;
      }
    }
    if (gtid < kHistBuckets / 1024) {
      d.segTotal[gtid] = 0ull;
      d.segLast[gtid] = -1;
    }
    unsigned long long best = 0ull;
    const int p = gtid;
    if (p < d.m) {
      const int r = st->pivotRow;
      const int t = st->numEtas;
      const double a = d.rhs3[p];
      const double alphaR = st->alphaCol;
      // eta column W_t = alpha_q with (alpha_r - 1) on the pivot position
      d.W[(size_t)p * d.tmax + t] = (p == r) ? a - 1.0 : a;
      if (p != r) {
        const int seq = d.pivotVariable[p];
        double x = d.sol[seq];
        if (st->numFlips > 0)
          x += d.rhs3[(size_t)2 * d.m + p];
        x -= st->thetaPrimal * a;
        d.sol[seq] = x;
        double w = d.dantzig ? 1.0 : d.weights[p];
        if (a != 0.0 && !d.dantzig) {
          // w_i += (a_i/a_r) * ((a_i/a_r) * w_r - 2 tau_i)   clipped at DEVEX_TRY_NORM
          const double ratio = a / alphaR;
          w += ratio * (ratio * st->rhoNorm2 - 2.0 * d.rhs3[(size_t)d.m + p]);
          w = w < kDevexTryNorm ? kDevexTryNorm : w;
          d.weights[p] = w;
        }
        if (!d.flagged[p])
          best = chuzr_key(x, d.lower[seq], d.upper[seq], w, d.primalTolerance, p);
      } else {
        double w = st->rhoNorm2 / (alphaR * alphaR);
        w = w < kDevexTryNorm ? kDevexTryNorm : w;
        if (d.dantzig)
          w = 1.0;
        else
          d.weights[p] = w;
        const int q = st->seqIn; // becomes basic at this position (housekeeping in the tail)
        d.flagged[p] = 0; // a new variable at this position
        best = chuzr_key(d.sol[q] + st->thetaPrimal, d.lowerTrue[q], d.upperTrue[q], w, d.primalTolerance, p);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
      best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
    if ((threadIdx.x & 31) == 0 && best != 0ull)
      atomicMax(&st->chuzrKey, best);
  }
  if (!last_block_done(d.tailCounter + TAIL_ITER_UPDATE))
    return;
  if (threadIdx.x == 0) {
    pivot_fixup_body(d);
    const unsigned long long key = atomicExch(&st->chuzrKey, 0ull);
    chuzr_finish_body(d, key, true);
  }
}

void launch_pivot_updates(const DeviceModel &d, cudaStream_t s)
{
  const int etaBlocks = (d.tmax + 1023) / 1024;
  const int posBlocks = (d.m + 255) / 256;
  iteration_update_kernel<<<etaBlocks + posBlocks, 256, 0, s>>>(d, etaBlocks);
}

// ------------------------------------------------------------------ refresh kernels
// choose a dual feasible bound for every nonbasic variable, fake bounds of width dualBound
// where the needed bound is infinite (ClpSimplexDual::changeBounds :3148)
__global__ void make_dual_feasible_kernel(DeviceModel d, double dualBound, int *counters)
{
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= d.nm)
    return;
  double lo = d.lowerTrue[j], up = d.upperTrue[j];
  unsigned char st = d.status[j];
  if (st == basic) {
    d.lower[j] = lo;
    d.upper[j] = up;
    d.fake[j] = 0;
    return;
  }
  const double dj = d.dj[j];
  const double tol = d.dualTolerance;
  const double old = d.sol[j];
  unsigned char f = 0;
  double x;
  if (lo == up) {
    st = isFixed;
    x = lo;
  } else if (dj > tol) {
    if (lo <= -kInf) {
      lo = (up < kInf ? up : 0.0) - dualBound;
      f = 1;
    }
    st = atLowerBound;
    x = lo;
  } else if (dj < -tol) {
    if (up >= kInf) {
      up = (lo > -kInf ? lo : 0.0) + dualBound;
      f = 2;
    }
    st = atUpperBound;
    x = up;
  } else {
    if (st == atUpperBound && up < kInf && !(d.fake[j] & 2)) {
      x = up;
    } else if (lo > -kInf) {
      st = atLowerBound;
      x = lo;
    } else if (up < kInf) {
      st = atUpperBound;
      x = up;
    } else {
      st = isFree;
      x = 0.0;
    }
  }
  d.lower[j] = lo;
  d.upper[j] = up;
  d.fake[j] = f;
  d.status[j] = st;
  d.sol[j] = x;
  if (f)
    atomicAdd(counters + 0, 1);
  if (x != old)
    atomicAdd(counters + 1, 1);
}

// xn[j] = nonbasic structural value (0 for basic)
__global__ void nonbasic_x_kernel(DeviceModel d, double *__restrict__ xn)
{
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < d.n)
    xn[j] = d.status[j] == basic ? 0.0 : d.sol[j];
}
// rhs[i] += value of nonbasic row variable
__global__ void primal_rhs_slack_kernel(DeviceModel d, double *__restrict__ rhs)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < d.m && d.status[d.n + i] != basic)
    rhs[i] += d.sol[d.n + i];
}
// sol[pivotVariable[p]] = x[p]
__global__ void scatter_basic_kernel(DeviceModel d, const double *__restrict__ x)
{
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < d.m)
    d.sol[d.pivotVariable[p]] = x[p];
}
// rhs[i] += value of the row variable (basic or not): residual y - A x
__global__ void primal_residual_rows_kernel(DeviceModel d, double *__restrict__ rhs)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < d.m)
    rhs[i] += d.sol[d.n + i];
}
// sol[pivotVariable[p]] += dx[p]
__global__ void add_basic_kernel(DeviceModel d, const double *__restrict__ dx)
{
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < d.m)
    d.sol[d.pivotVariable[p]] += dx[p];
}
// cB[p] = cost[pivotVariable[p]]
__global__ void gather_basic_cost_kernel(DeviceModel d, double *__restrict__ cb)
{
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < d.m)
    cb[p] = d.cost[d.pivotVariable[p]];
}
// dj = cost - z for columns, cost + pi for rows; 0 for basics
__global__ void reduced_cost_kernel(DeviceModel d, const double *__restrict__ z,
                                    const double *__restrict__ pi)
{
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= d.nm)
    return;
  double v = 0.0;
  if (d.status[j] != basic)
    v = j < d.n ? d.cost[j] - z[j] : d.cost[j] + pi[j - d.n];
  d.dj[j] = v;
}

// out[0] = sum costTrue*sol (fixed order, single CTA) ; out[1] = sum primal infeasibility of basics
__global__ void __launch_bounds__(1024) objective_kernel(DeviceModel d, double *out)
{
  __shared__ double s1[32], s2[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double a = 0.0, b = 0.0;
  for (int j = tid; j < d.nm; j += 1024)
    a = fma(d.costTrue[j], d.sol[j], a);
  for (int p = tid; p < d.m; p += 1024) {
    int seq = d.pivotVariable[p];
    double v = d.sol[seq];
    if (v < d.lower[seq] - d.primalTolerance)
      b += d.lower[seq] - v;
    else if (v > d.upper[seq] + d.primalTolerance)
      b += v - d.upper[seq];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if (lane == 0) {
    s1[warp] = a;
    s2[warp] = b;
  }
  __syncthreads();
  if (tid == 0) {
    double x = 0.0, y = 0.0;
    for (int w = 0; w < 32; w++) {
      x += s1[w];
      y += s2[w];
    }
    out[0] = x;
    out[1] = y;
  }
}

// weightsNew[p] = srcPos[p] >= 0 ? weightsOld[srcPos[p]] : 1
__global__ void permute_weights_kernel(const double *__restrict__ wOld, double *__restrict__ wNew,
                                       const int *__restrict__ srcPos, int m)
{
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < m)
    wNew[p] = srcPos[p] >= 0 ? wOld[srcPos[p]] : 1.0;
}

// dense nucleus gather into a zeroed N: N[i][j] (row-major k x ld) = A[nucRow[i], nucCol[j]].  Entries of
// a column that name the same row are added, as PRICE, times and S1 add them (loadProblem keeps them apart).
__global__ void gather_nucleus_matrix_kernel(DeviceModel d, double *__restrict__ N, int ld)
{
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (j >= d.k)
    return;
  const int col = d.nucCol[j];
  for (int e = d.colStart[col] + lane; e < d.colStart[col + 1]; e += 32) {
    int ni = d.posToNuc[d.rowIdx[e]];
    if (ni >= 0)
      atomicAdd(&N[(size_t)ni * ld + j], d.val[e]);
  }
}

__global__ void count_fake_kernel(DeviceModel d, int *counter)
{
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < d.nm && d.fake[j] && d.status[j] != basic)
    atomicAdd(counter, 1);
}
void launch_count_fake(const DeviceModel &d, int *counter, cudaStream_t s)
{
  count_fake_kernel<<<(d.nm + 255) / 256, 256, 0, s>>>(d, counter);
}

// out[m] = column seq of [A | -I]   (ClpPackedMatrix::unpack :4803)
__global__ void unpack_column_kernel(DeviceModel d, int seq, double *__restrict__ out)
{
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (seq >= d.n) {
    if (i < d.m)
      out[i] = (i == seq - d.n) ? -1.0 : 0.0;
    return;
  }
  // zero fill; unpack_scatter_kernel then writes the entries
  if (i < d.m)
    out[i] = 0.0;
}
// grid-stride over the entries: a column may hold up to m entries
__global__ void unpack_scatter_kernel(DeviceModel d, int seq, double *__restrict__ out)
{
  const int e1 = d.colStart[seq + 1];
  for (int e = d.colStart[seq] + blockIdx.x * blockDim.x + threadIdx.x; e < e1; e += gridDim.x * blockDim.x)
    out[d.rowIdx[e]] = d.val[e];
}
void launch_unpack_column(const DeviceModel &d, int seq, double *out, cudaStream_t s)
{
  unpack_column_kernel<<<(d.m + 255) / 256, 256, 0, s>>>(d, seq, out);
  if (seq < d.n)
    unpack_scatter_kernel<<<64, 256, 0, s>>>(d, seq, out);
}

// Product-form update outside the simplex loop (replaceColumn entry point / parity tests):
// rhs3[0] holds B^-1 a_q ; append it as eta for position pivotRow.
__global__ void eta_append_prepare_kernel(DeviceModel d, int pivotRow)
{
  d.st->pivotRow = pivotRow;
  d.st->alphaCol = d.rhs3[pivotRow];
}
__global__ void eta_append_column_kernel(DeviceModel d)
{
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= d.m)
    return;
  const int r = d.st->pivotRow, t = d.st->numEtas;
  const double a = d.rhs3[p];
  d.W[(size_t)p * d.tmax + t] = (p == r) ? a - 1.0 : a;
}
__global__ void eta_append_finish_kernel(DeviceModel d, int seqIn)
{
  IterState *st = d.st;
  const int r = st->pivotRow, t = st->numEtas;
  d.etaPos[t] = r;
  d.etaPrevSame[t] = d.etaLastOfPos[r];
  d.etaLastOfPos[r] = t;
  st->numEtas = t + 1;
  const int out = d.pivotVariable[r];
  d.status[out] = atLowerBound;
  d.status[seqIn] = basic;
  d.pivotVariable[r] = seqIn;
}
__global__ void eta_append_row_kernel(DeviceModel d)
{
  eta_append_row(d, blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
}
void launch_eta_append_test(const DeviceModel &d, int pivotRow, int seqIn, cudaStream_t s)
{
  eta_append_prepare_kernel<<<1, 1, 0, s>>>(d, pivotRow);
  launch_eta_rowvec(d, 0, false, s); // nu for this pivot row
  eta_append_row_kernel<<<(d.tmax + 255) / 256, 256, 0, s>>>(d);
  eta_append_column_kernel<<<(d.m + 255) / 256, 256, 0, s>>>(d);
  eta_append_finish_kernel<<<1, 1, 0, s>>>(d, seqIn);
}

// largest relative change of a basic value between the recurrence-updated solution (xold) and the one
// recomputed from scratch: out[0] = max_p |x - xold| / (1 + |x|) as double bits (positive => ordered)
__global__ void primal_drift_kernel(DeviceModel d, const double *__restrict__ xold, unsigned long long *out)
{
  double worst = 0.0;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < d.m; p += gridDim.x * blockDim.x) {
    const int seq = d.pivotVariable[p];
    const double x = d.sol[seq];
    const double r = fabs(x - xold[seq]) / (1.0 + fabs(x));
    worst = r > worst ? r : worst; // NaN never wins
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    worst = fmax(worst, __shfl_xor_sync(0xffffffffu, worst, o));
  if ((threadIdx.x & 31) == 0 && worst > 0.0)
    atomicMax(out, (unsigned long long)__double_as_longlong(worst));
}
void launch_primal_drift(const DeviceModel &d, const double *xold, unsigned long long *out, cudaStream_t s)
{
  int blocks = (d.m + 255) / 256;
  primal_drift_kernel<<<blocks > device_sm_count() * 4 ? device_sm_count() * 4 : blocks, 256, 0, s>>>(d, xold, out);
}

// ---- host wrappers used by engine.cu
void launch_make_dual_feasible(const DeviceModel &d, double dualBound, int *counters, cudaStream_t s)
{
  make_dual_feasible_kernel<<<(d.nm + 255) / 256, 256, 0, s>>>(d, dualBound, counters);
}
void launch_compute_primals(const DeviceModel &d, double *xn, double *rhs, cudaStream_t s, bool withEtas)
{
  // rhs = -A x_N + (nonbasic row values) ; x_B = B0^-1 rhs   (no etas: fresh factorization)
  if (d.n > 0)
    nonbasic_x_kernel<<<(d.n + 255) / 256, 256, 0, s>>>(d, xn);
  launch_times_rows(d, xn, rhs, -1.0, s);
  primal_rhs_slack_kernel<<<(d.m + 255) / 256, 256, 0, s>>>(d, rhs);
  launch_ftran_buffer(d, rhs, 1, withEtas, s);
  scatter_basic_kernel<<<(d.m + 255) / 256, 256, 0, s>>>(d, rhs);
  // one step of iterative refinement (ClpSimplex::computePrimals, src/ClpSimplex.cpp:1057-1110):
  // r = y - A x over ALL variables, x_B += B0^-1 r
  launch_times_rows(d, d.sol, rhs, -1.0, s);
  primal_residual_rows_kernel<<<(d.m + 255) / 256, 256, 0, s>>>(d, rhs);
  launch_ftran_buffer(d, rhs, 1, withEtas, s);
  add_basic_kernel<<<(d.m + 255) / 256, 256, 0, s>>>(d, rhs);
}
void launch_compute_duals(const DeviceModel &d, double *pi, double *z, cudaStream_t s)
{
  // right after a refactorization: no etas
  gather_basic_cost_kernel<<<(d.m + 255) / 256, 256, 0, s>>>(d, pi);
  launch_btran_dense(d, pi, false, s);
  launch_transpose_times(d, pi, z, 1.0, s);
  reduced_cost_kernel<<<(d.nm + 255) / 256, 256, 0, s>>>(d, z, pi);
}
void launch_objective(const DeviceModel &d, double *out, cudaStream_t s)
{
  objective_kernel<<<1, 1024, 0, s>>>(d, out);
}
void launch_permute_weights(const double *wOld, double *wNew, const int *srcPos, int m,
                            cudaStream_t s)
{
  permute_weights_kernel<<<(m + 255) / 256, 256, 0, s>>>(wOld, wNew, srcPos, m);
}
void launch_gather_nucleus_matrix(const DeviceModel &d, double *N, int ld, cudaStream_t s)
{
  if (d.k > 0)
    gather_nucleus_matrix_kernel<<<(d.k + 7) / 8, 256, 0, s>>>(d, N, ld);
}

} // namespace clpb
