// stream_variants.cu -- micro-benchmarks behind the design choices of the two HBM-streaming
// kernels (PRICE over the CSC arrays, GEMV over the nucleus inverse).  Not part of the product;
// built and run by hand:   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o sv stream_variants.cu
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
  for (int o = 16; o > 0; o >>= 1)
    v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------- V0: plain LDG stream (upper bound)
__global__ void __launch_bounds__(512) v0_ldg(const int *__restrict__ idx, const double *__restrict__ val, long n,
                                            double *out)
{
  double acc = 0.0;
  long stride = (long)gridDim.x * blockDim.x * 2;
  for (long e = ((long)blockIdx.x * blockDim.x + threadIdx.x) * 2; e + 1 < n; e += stride) {
    int2 i2 = __ldcs(reinterpret_cast<const int2 *>(idx + e));
    double2 v2 = __ldcs(reinterpret_cast<const double2 *>(val + e));
    acc += v2.x * (i2.x & 1) + v2.y * (i2.y & 1);
  }
  if (acc == 123.456)
    out[0] = acc;
}

// ---------------------------------------------------------------- TMA pipeline variants
// mode 0: load only ; 1: + products with smem rho ; 2: + per-"column" sums (fixed 96-entry columns)
template <int STAGES, int TILE>
__global__ void __launch_bounds__(1024, 1)
    v_tma(const int *__restrict__ idx, const double *__restrict__ val, long n, const double *__restrict__ rho, int m,
          double *__restrict__ out, int mode, int alignShift)
{
  extern __shared__ __align__(128) unsigned char raw[];
  unsigned long long *full = reinterpret_cast<unsigned long long *>(raw);
  int *sidx = reinterpret_cast<int *>(raw + 128);
  double *sval = reinterpret_cast<double *>(sidx + STAGES * TILE);
  double *srho = sval + STAGES * TILE;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long ntiles = n / TILE;
  auto issue = [&](long t, int stage) {
    long ea = t * TILE + alignShift; // alignShift=4 entries -> 16 B aligned only (not 128 B)
    mbar_expect_tx(&full[stage], TILE * 12u);
    bulk_g2s(sidx + stage * TILE, idx + ea, TILE * 4u, &full[stage]);
    bulk_g2s(sval + stage * TILE, val + ea, TILE * 8u, &full[stage]);
  };
  if (tid == 0) {
    for (int q = 0; q < STAGES; q++)
      mbar_init(&full[q], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    for (int q = 0; q < STAGES; q++)
      if (blockIdx.x + (long)q * gridDim.x < ntiles - 1)
        issue(blockIdx.x + (long)q * gridDim.x, q);
  }
  if (mode >= 1)
    for (int i = tid; i < m; i += 1024)
      srho[i] = rho[i];
  __syncthreads();
  double keep = 0.0;
  int it = 0;
  for (long t = blockIdx.x; t < ntiles - 1; t += gridDim.x, it++) {
    const int stage = it % STAGES;
    mbar_wait(&full[stage], (unsigned)((it / STAGES) & 1));
    double *v = sval + stage * TILE;
    const int *ix = sidx + stage * TILE;
    if (mode == 0) {
      keep += v[tid] + ix[tid];
    } else {
      for (int e = tid; e < TILE; e += 1024)
        v[e] *= srho[ix[e]];
      __syncthreads();
      if (mode >= 2) {
        for (int c = warp; c < TILE / 96; c += 32) {
          double acc = 0.0;
          for (int e = c * 96 + lane; e < c * 96 + 96; e += 32)
            acc += v[e];
          acc = warp_sum(acc);
          if (lane == 0)
            out[(t * (TILE / 96) + c) & 0xFFFFF] = acc;
        }
      }
    }
    __syncthreads();
    if (tid == 0) {
      long next = t + (long)STAGES * gridDim.x;
      if (next < ntiles - 1) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        issue(next, stage);
      }
    }
  }
  if (keep == 123.456)
    out[0] = keep;
}

// ---------------------------------------------------------------- LDG-to-register tile variant (no TMA)
// each CTA (512 thr, 2/SM) handles tiles of 2048 entries: loads 4 entries/thread to registers,
// multiplies by smem rho, warp-level segmented sum over fixed 96-entry columns via smem
__global__ void __launch_bounds__(512, 2)
    v_ldg_tile(const int *__restrict__ idx, const double *__restrict__ val, long n, const double *__restrict__ rho,
               int m, double *__restrict__ out)
{
  extern __shared__ __align__(16) unsigned char raw2[];
  double *srho = reinterpret_cast<double *>(raw2);
  double *sprod = srho + m; // 2 x 2048
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < m; i += 512)
    srho[i] = rho[i];
  __syncthreads();
  const long ntiles = n / 2048;
  int buf = 0;
  for (long t = blockIdx.x; t < ntiles; t += gridDim.x, buf ^= 1) {
    const long e0 = t * 2048 + tid * 4;
    int4 i4 = __ldcs(reinterpret_cast<const int4 *>(idx + e0));
    double2 va = __ldcs(reinterpret_cast<const double2 *>(val + e0));
    double2 vb = __ldcs(reinterpret_cast<const double2 *>(val + e0 + 2));
    double *p = sprod + buf * 2048 + tid * 4;
    p[0] = va.x * srho[i4.x];
    p[1] = va.y * srho[i4.y];
    p[2] = vb.x * srho[i4.z];
    p[3] = vb.y * srho[i4.w];
    __syncthreads();
    for (int c = warp; c < 21; c += 16) {
      double acc = 0.0;
      const double *q = sprod + buf * 2048 + c * 96;
      for (int e = lane; e < 96; e += 32)
        acc += q[e];
      acc = warp_sum(acc);
      if (lane == 0)
        out[(t * 21 + c) & 0xFFFFF] = acc;
    }
  }
}

// TMA with each tile fetched as NSPLIT smaller bulk copies per array (more requests in flight)
template <int STAGES, int TILE, int NSPLIT>
__global__ void __launch_bounds__(1024, 1)
    v_tma_split(const int *__restrict__ idx, const double *__restrict__ val, long n, double *__restrict__ out)
{
  extern __shared__ __align__(128) unsigned char raw[];
  unsigned long long *full = reinterpret_cast<unsigned long long *>(raw);
  int *sidx = reinterpret_cast<int *>(raw + 128);
  double *sval = reinterpret_cast<double *>(sidx + STAGES * TILE);
  const int tid = threadIdx.x;
  const long ntiles = n / TILE;
  auto issue = [&](long t, int stage) {
    long ea = t * TILE;
    mbar_expect_tx(&full[stage], TILE * 12u);
    constexpr int PART = TILE / NSPLIT;
    for (int q = 0; q < NSPLIT; q++) {
      bulk_g2s(sidx + stage * TILE + q * PART, idx + ea + q * PART, PART * 4u, &full[stage]);
      bulk_g2s(sval + stage * TILE + q * PART, val + ea + q * PART, PART * 8u, &full[stage]);
    }
  };
  if (tid == 0) {
    for (int q = 0; q < STAGES; q++)
      mbar_init(&full[q], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    for (int q = 0; q < STAGES; q++)
      if (blockIdx.x + (long)q * gridDim.x < ntiles - 1)
        issue(blockIdx.x + (long)q * gridDim.x, q);
  }
  __syncthreads();
  double keep = 0.0;
  int it = 0;
  for (long t = blockIdx.x; t < ntiles - 1; t += gridDim.x, it++) {
    const int stage = it % STAGES;
    mbar_wait(&full[stage], (unsigned)((it / STAGES) & 1));
    keep += sval[stage * TILE + tid] + sidx[stage * TILE + tid];
    __syncthreads();
    if (tid == 0) {
      long next = t + (long)STAGES * gridDim.x;
      if (next < ntiles - 1) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        issue(next, stage);
      }
    }
  }
  if (keep == 123.456)
    out[0] = keep;
}

// LDG with register prefetch: CTA of 512 threads, tiles of 2048 entries (4 per thread); the loads
// of tile i+1 are issued before tile i is consumed.  Products go through smem, half-warp sums.
template <int CTAS_PER_SM>
__global__ void __launch_bounds__(512, CTAS_PER_SM)
    v_ldg_prefetch(const int *__restrict__ idx, const double *__restrict__ val, long n,
                   const double *__restrict__ rho, int m, double *__restrict__ out, int mode)
{
  extern __shared__ __align__(16) unsigned char raw2[];
  double *srho = reinterpret_cast<double *>(raw2);
  double *sprod = srho + m; // 2048
  const int tid = threadIdx.x;
  for (int i = tid; i < m; i += 512)
    srho[i] = rho[i];
  __syncthreads();
  const long ntiles = n / 2048;
  long t = blockIdx.x;
  int4 i4 = make_int4(0, 0, 0, 0);
  double2 va = make_double2(0, 0), vb = va;
  if (t < ntiles) {
    const long e0 = t * 2048 + tid * 4;
    i4 = __ldcs(reinterpret_cast<const int4 *>(idx + e0));
    va = __ldcs(reinterpret_cast<const double2 *>(val + e0));
    vb = __ldcs(reinterpret_cast<const double2 *>(val + e0 + 2));
  }
  double keep = 0.0;
  const int half = tid >> 4, l16 = tid & 15;
  for (; t < ntiles; t += gridDim.x) {
    const int4 ci = i4;
    const double2 ca = va, cb = vb;
    const long tn = t + gridDim.x;
    if (tn < ntiles) {
      const long e0 = tn * 2048 + tid * 4;
      i4 = __ldcs(reinterpret_cast<const int4 *>(idx + e0));
      va = __ldcs(reinterpret_cast<const double2 *>(val + e0));
      vb = __ldcs(reinterpret_cast<const double2 *>(val + e0 + 2));
    }
    if (mode == 0) {
      keep += ca.x + cb.y + ci.x;
      continue;
    }
    double *p = sprod + tid * 4;
    p[0] = ca.x * srho[ci.x];
    p[1] = ca.y * srho[ci.y];
    p[2] = cb.x * srho[ci.z];
    p[3] = cb.y * srho[ci.w];
    __syncthreads();
    if (half < 21) {
      double acc = 0.0;
      const double *q = sprod + half * 96;
      for (int e = l16; e < 96; e += 16)
        acc += q[e];
      const unsigned hm = 0xFFFFu << (tid & 16);
      acc += __shfl_xor_sync(hm, acc, 8);
      acc += __shfl_xor_sync(hm, acc, 4);
      acc += __shfl_xor_sync(hm, acc, 2);
      acc += __shfl_xor_sync(hm, acc, 1);
      if (l16 == 0)
        out[(t * 21 + half) & 0xFFFFF] = acc;
    }
    __syncthreads();
  }
  if (keep == 123.456)
    out[0] = keep;
}

// ---------------------------------------------------------------- GEMV variants
template <int DEPTH>
__global__ void __launch_bounds__(256)
    gemv_cta_row(const double *__restrict__ M, int k, int ldk, const double *__restrict__ x, double *__restrict__ out)
{
  __shared__ double part[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int half = ldk >> 1;
  for (int i = blockIdx.x; i < k; i += gridDim.x) {
    const double2 *row = reinterpret_cast<const double2 *>(M + (size_t)i * ldk);
    const double2 *xv = reinterpret_cast<const double2 *>(x);
    double acc = 0.0;
    for (int j = threadIdx.x; j < half; j += 256 * DEPTH) {
      double2 a[DEPTH];
#pragma unroll
      for (int q = 0; q < DEPTH; q++)
        a[q] = (j + 256 * q < half) ? __ldcs(row + j + 256 * q) : make_double2(0.0, 0.0);
#pragma unroll
      for (int q = 0; q < DEPTH; q++) {
        double2 b = (j + 256 * q < half) ? __ldg(xv + j + 256 * q) : make_double2(0.0, 0.0);
        acc = fma(a[q].x, b.x, acc);
        acc = fma(a[q].y, b.y, acc);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0)
      part[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0;
      for (int w = 0; w < 8; w++)
        s += part[w];
      out[i] = s;
    }
    __syncthreads();
  }
}

// GEMV with x in shared memory, warp per row, DEPTH loads in flight per lane
template <int DEPTH>
__global__ void __launch_bounds__(512)
    gemv_warp_row_smemx(const double *__restrict__ M, int k, int ldk, const double *__restrict__ x,
                        double *__restrict__ out)
{
  extern __shared__ __align__(16) unsigned char raw3[];
  double2 *sx = reinterpret_cast<double2 *>(raw3);
  const int half = ldk >> 1;
  for (int j = threadIdx.x; j < half; j += 512)
    sx[j] = reinterpret_cast<const double2 *>(x)[j];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = blockIdx.x * 16 + warp; i < k; i += gridDim.x * 16) {
    const double2 *row = reinterpret_cast<const double2 *>(M + (size_t)i * ldk);
    double acc = 0.0;
    for (int j = lane; j < half; j += 32 * DEPTH) {
      double2 a[DEPTH];
#pragma unroll
      for (int q = 0; q < DEPTH; q++)
        a[q] = (j + 32 * q < half) ? __ldcs(row + j + 32 * q) : make_double2(0.0, 0.0);
#pragma unroll
      for (int q = 0; q < DEPTH; q++) {
        double2 b = (j + 32 * q < half) ? sx[j + 32 * q] : make_double2(0.0, 0.0);
        acc = fma(a[q].x, b.x, acc);
        acc = fma(a[q].y, b.y, acc);
      }
    }
    acc = warp_sum(acc);
    if (lane == 0)
      out[i] = acc;
  }
}

template <class F> float timeit(F f, int reps = 10)
{
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  f();
  CK(cudaDeviceSynchronize());
  float best = 1e30f;
  for (int r = 0; r < reps; r++) {
    cudaEventRecord(a);
    f();
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    float ms;
    cudaEventElapsedTime(&ms, a, b);
    if (ms < best)
      best = ms;
  }
  CK(cudaGetLastError());
  return best;
}

int main()
{
  const long n = 10001920; // entries per window
  const int NWIN = 8;      // rotate over 8 windows (960 MB) so that L2 (126 MB) cannot help
  const int m = 10000;
  int *idx;
  double *val, *rho, *out;
  CK(cudaMalloc(&idx, (NWIN * n + 8192) * 4));
  CK(cudaMalloc(&val, (NWIN * n + 8192) * 8));
  CK(cudaMalloc(&rho, m * 8));
  CK(cudaMalloc(&out, (1 << 20) * 8 + 64));
  std::vector<int> hi(NWIN * n + 8192);
  std::vector<double> hv(NWIN * n + 8192, 0.5), hr(m, 1.0);
  for (long i = 0; i < NWIN * n + 8192; i++)
    hi[i] = (int)((i * 2654435761u) % m);
  CK(cudaMemcpy(idx, hi.data(), (NWIN * n + 8192) * 4, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(val, hv.data(), (NWIN * n + 8192) * 8, cudaMemcpyHostToDevice));
  const int *idx0 = idx;
  const double *val0 = val;
  int win = 0;
#define NEXTWIN() do { win = (win + 1) % NWIN; idx = const_cast<int *>(idx0) + (long)win * n; val = const_cast<double *>(val0) + (long)win * n; } while (0)
  CK(cudaMemcpy(rho, hr.data(), m * 8, cudaMemcpyHostToDevice));
  // a 256 MB buffer to flush L2 between runs is unnecessary: 120 MB stream > L2 reuse window
  const double bytes = 12.0 * n;
  auto rep = [&](const char *name, float ms) { printf("%-46s %8.1f us  %7.1f GB/s\n", name, ms * 1000, bytes / ms / 1e6); fflush(stdout); };

  rep("V0 plain LDG stream SMSx8x512", timeit([&] { NEXTWIN(); v0_ldg<<<numSms() * 8, 512>>>(idx, val, n, out); }));
  rep("V0 plain LDG stream SMSx4x512", timeit([&] { NEXTWIN(); v0_ldg<<<numSms() * 4, 512>>>(idx, val, n, out); }));
#define RUN_TMA(ST, TL, MODE, AL, NAME)                                                            \
  {                                                                                                \
    size_t sm = 128 + (size_t)ST * TL * 12 + (MODE >= 1 ? m * 8 : 0);                              \
    CK(cudaFuncSetAttribute(v_tma<ST, TL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); \
    rep(NAME, timeit([&] { NEXTWIN(); v_tma<ST, TL><<<numSms(), 1024, sm>>>(idx, val, n, rho, m, out, MODE, AL); })); \
  }
  RUN_TMA(3, 3072, 0, 0, "TMA 3x3072 load only, 128B aligned");
  RUN_TMA(3, 3072, 0, 4, "TMA 3x3072 load only, 16B aligned");
  RUN_TMA(2, 6144, 0, 0, "TMA 2x6144 load only, aligned");
  RUN_TMA(4, 3072, 0, 0, "TMA 4x3072 load only, aligned");
  RUN_TMA(6, 2048, 0, 0, "TMA 6x2048 load only, aligned");
  RUN_TMA(8, 1024, 0, 0, "TMA 8x1024 load only, aligned");
  RUN_TMA(3, 3072, 1, 0, "TMA 3x3072 + products");
  RUN_TMA(3, 3072, 2, 0, "TMA 3x3072 + products + col sums");
  RUN_TMA(3, 3072, 2, 4, "TMA 3x3072 full, 16B aligned");
  RUN_TMA(4, 2048, 2, 0, "TMA 4x2048 full");
  {
    size_t sm = (size_t)m * 8 + 2 * 2048 * 8;
    CK(cudaFuncSetAttribute(v_ldg_tile, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    rep("LDG tile 2048 (512 thr, 2 CTA/SM) full", timeit([&] { NEXTWIN(); v_ldg_tile<<<numSms() * 2, 512, sm>>>(idx, val, n, rho, m, out); }));
  }

  {
    CK(cudaFuncSetAttribute(v_tma_split<3, 3072, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    CK(cudaFuncSetAttribute(v_tma_split<3, 3072, 12>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    CK(cudaFuncSetAttribute(v_tma_split<6, 3072, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    size_t sm3 = 128 + 3 * 3072 * 12, sm6 = 128 + 6 * 3072 * 12;
    rep("TMA 3x3072 load only, 4 sub-copies", timeit([&] { NEXTWIN(); v_tma_split<3, 3072, 4><<<numSms(), 1024, sm3>>>(idx, val, n, out); }));
    rep("TMA 3x3072 load only, 12 sub-copies", timeit([&] { NEXTWIN(); v_tma_split<3, 3072, 12><<<numSms(), 1024, sm3>>>(idx, val, n, out); }));
    rep("TMA 6x3072 load only, 4 sub-copies", timeit([&] { NEXTWIN(); v_tma_split<6, 3072, 4><<<numSms(), 1024, sm6>>>(idx, val, n, out); }));
  }
  {
    size_t sm = (size_t)m * 8 + 2048 * 8;
    CK(cudaFuncSetAttribute(v_ldg_prefetch<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024));
    CK(cudaFuncSetAttribute(v_ldg_prefetch<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024));
    rep("LDG prefetch 512thr 2CTA/SM load only", timeit([&] { NEXTWIN(); v_ldg_prefetch<2><<<numSms() * 2, 512, sm>>>(idx, val, n, rho, m, out, 0); }));
    rep("LDG prefetch 512thr 2CTA/SM full", timeit([&] { NEXTWIN(); v_ldg_prefetch<2><<<numSms() * 2, 512, sm>>>(idx, val, n, rho, m, out, 1); }));
  }

  // ---- GEMV: k = 4682
  const int k = 4682, ldk = 4688;
  double *M, *x;
  CK(cudaMalloc(&M, (size_t)k * ldk * 8));
  CK(cudaMalloc(&x, ldk * 8));
  CK(cudaMemset(M, 0, (size_t)k * ldk * 8));
  CK(cudaMemset(x, 0, ldk * 8));
  const double gbytes = 8.0 * k * ldk;
  auto repg = [&](const char *name, float ms) { printf("%-46s %8.1f us  %7.1f GB/s\n", name, ms * 1000, gbytes / ms / 1e6); fflush(stdout); };
  repg("GEMV cta-per-row depth4 grid 888", timeit([&] { gemv_cta_row<4><<<888, 256>>>(M, k, ldk, x, out); }));
  repg("GEMV cta-per-row depth8 grid 888", timeit([&] { gemv_cta_row<8><<<888, 256>>>(M, k, ldk, x, out); }));
  repg("GEMV cta-per-row depth4 grid 1184", timeit([&] { gemv_cta_row<4><<<1184, 256>>>(M, k, ldk, x, out); }));
  repg("GEMV cta-per-row depth8 grid 592", timeit([&] { gemv_cta_row<8><<<592, 256>>>(M, k, ldk, x, out); }));
  {
    CK(cudaFuncSetAttribute(gemv_warp_row_smemx<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    CK(cudaFuncSetAttribute(gemv_warp_row_smemx<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    size_t sm = (size_t)ldk * 8;
    repg("GEMV warp-per-row smem x depth4 SMSx4x512", timeit([&] { gemv_warp_row_smemx<4><<<numSms() * 4, 512, sm>>>(M, k, ldk, x, out); }));
    repg("GEMV warp-per-row smem x depth8 SMSx4x512", timeit([&] { gemv_warp_row_smemx<8><<<numSms() * 4, 512, sm>>>(M, k, ldk, x, out); }));
    repg("GEMV warp-per-row smem x depth8 SMSx2x512", timeit([&] { gemv_warp_row_smemx<8><<<numSms() * 2, 512, sm>>>(M, k, ldk, x, out); }));
  }
  // plain copy-like read of M for reference
  rep("(ref) V0 LDG stream again", timeit([&] { NEXTWIN(); v0_ldg<<<numSms() * 8, 512>>>(idx, val, n, out); }));
  return 0;
}
