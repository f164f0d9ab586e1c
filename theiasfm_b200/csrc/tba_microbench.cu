// tba_microbench.cu -- three tiny device micro-benchmarks that give the roofline denominators MEASURED_PEAKS.json
// does not have (SURVEY 8d: "fp64 peak is not in that file -- builder must measure a DFMA microbenchmark"):
//   out[0] fp64 FMA throughput, TFLOP/s (8 independent DFMA chains per thread)
//   out[1] fp64 RED.ADD throughput to 60 000 spread addresses (the matvec's camera vector at 10k cameras), G ops/s
//   out[2] 48-byte gather throughput from the same vector (3 x LDG.128 per lane, 32 distinct rows per warp), G rows/s
// Built into its own library (libtheia_microbench_b200.so) and run by bench.py in a separate process, so that nothing
// here can disturb the measured solve.
#include <cuda_runtime.h>

#include <cstdio>

namespace {

__global__ void k_dfma(double* out, int iters) {
  double a0 = threadIdx.x * 1e-3, a1 = a0 + 1.0, a2 = a0 + 2.0, a3 = a0 + 3.0, a4 = a0 + 4.0, a5 = a0 + 5.0, a6 = a0 + 6.0, a7 = a0 + 7.0;
  const double b = 1.0000001, c = 1e-9;
  for (int i = 0; i < iters; ++i) {
    a0 = fma(a0, b, c); a1 = fma(a1, b, c); a2 = fma(a2, b, c); a3 = fma(a3, b, c);
    a4 = fma(a4, b, c); a5 = fma(a5, b, c); a6 = fma(a6, b, c); a7 = fma(a7, b, c);
  }
  out[(size_t)blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

__global__ void k_red(double* y, unsigned n, int reps) {
  const unsigned gid = blockIdx.x * blockDim.x + threadIdx.x;
  for (int k = 0; k < reps; ++k) {
    const unsigned idx = (gid * 2654435761u + (unsigned)k * 40503u) % n;
    atomicAdd(y + idx, 1.0);
  }
}

__global__ void k_gather(const double* __restrict__ x, unsigned n_rows, int reps, double* out) {
  const unsigned gid = blockIdx.x * blockDim.x + threadIdx.x;
  double acc = 0.0;
  for (int k = 0; k < reps; ++k) {
    const unsigned row = (gid * 2654435761u + (unsigned)k * 40503u) % n_rows;
    const double2* p = reinterpret_cast<const double2*>(x + (size_t)row * 6);
    const double2 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2);
    acc += a.x + a.y + b.x + b.y + c.x + c.y;
  }
  out[gid] = acc;
}

// Design questions, measured by every bench run before the timed solve (tba_microbench_ex):
// k_red_rows: the element-major ("transposed", TBA_TRED) emission -- lanes 6q..6q+5 of a warp add to the 6 consecutive doubles
// of one random 48-byte row (2 sectors), i.e. 32 elements cover ~11 sectors instead of 32.  G elements/s, comparable to k_red.
__global__ void k_red_rows(double* y, unsigned n_rows, int reps) {
  const unsigned gid = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned lane = threadIdx.x & 31u, warp = gid >> 5;
  const unsigned q = lane / 6u, j = lane - q * 6u;  // lanes 30, 31: a sixth row (2 of its elements)
  for (int k = 0; k < reps; ++k) {
    const unsigned row = ((warp * 6u + q) * 2654435761u + (unsigned)k * 40503u) % n_rows;
    atomicAdd(y + (size_t)row * 6 + j, 1.0);
  }
}
// k_smem_atomic: shared-memory fp64 atomicAdd (compiles to a CAS loop) to random slots of a 2048-double window per CTA,
// flushed once at the end: would a shared-memory camera-window accumulator beat global REDs?  G ops/s.
__global__ void k_smem_atomic(double* out, int reps) {
  __shared__ double win[2048];
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) win[i] = 0.0;
  __syncthreads();
  const unsigned gid = blockIdx.x * blockDim.x + threadIdx.x;
  for (int k = 0; k < reps; ++k) {
    const unsigned idx = (gid * 2654435761u + (unsigned)k * 40503u) & 2047u;
    atomicAdd(&win[idx], 1.0);
  }
  __syncthreads();
  double acc = 0.0;
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) acc += win[i];
  out[gid] = acc;
}
// k_red_win: the same global REDs as k_red but every CTA confined to a window of 1200 rows x 6 doubles that slides with
// the CTA index (TBA_PACK_SORT locality: concurrent CTAs hit the same few thousand addresses).  G ops/s.
__global__ void k_red_win(double* y, unsigned n, int reps) {
  const unsigned gid = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned win = 7200u, base = (unsigned)(((unsigned long long)blockIdx.x * (n - win)) / gridDim.x);
  for (int k = 0; k < reps; ++k) {
    const unsigned idx = base + (gid * 2654435761u + (unsigned)k * 40503u) % win;
    atomicAdd(y + idx, 1.0);
  }
}

// Gather strategies for the matvec's 48-byte camera rows (k_gather above = the shipped one: 3 x LDG.128 per lane, lane-per-row).
// k_gather_coop: chunk-major -- lane l of load k fetches 16-byte chunk 32k + l of the warp's 32 rows (3 lanes cover one row: ~21 sectors
// per instruction instead of 32), transposed back through shared memory (3 x STS.128 + 3 x LDS.128 per lane).
__global__ void k_gather_coop(const double* __restrict__ x, unsigned n_rows, int reps, double* out) {
  __shared__ __align__(16) double s_rows[8][32 * 6];
  __shared__ unsigned s_row[8][32];
  const unsigned gid = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  double acc = 0.0;
  for (int k = 0; k < reps; ++k) {
    s_row[w][lane] = (gid * 2654435761u + (unsigned)k * 40503u) % n_rows;
    __syncwarp();
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const unsigned e = c * 32u + lane, o = e / 3u, part = e - o * 3u;
      const double2 v = __ldg(reinterpret_cast<const double2*>(x + (size_t)s_row[w][o] * 6) + part);
      *reinterpret_cast<double2*>(&s_rows[w][e * 2]) = v;
    }
    __syncwarp();
    const double2* r = reinterpret_cast<const double2*>(&s_rows[w][lane * 6]);
    const double2 a = r[0], b = r[1], c2 = r[2];
    acc += a.x + a.y + b.x + b.y + c2.x + c2.y;
    __syncwarp();
  }
  out[gid] = acc;
}
// k_gather_64: rows padded to 64 bytes (8 doubles, 64-byte aligned): three 128-bit loads per lane (sm_90 has no 256-bit load),
// 2 sectors of ONE 128-byte line per row.
__global__ void k_gather_64(const double* __restrict__ x8, unsigned n_rows, int reps, double* out) {
  const unsigned gid = blockIdx.x * blockDim.x + threadIdx.x;
  double acc = 0.0;
  for (int k = 0; k < reps; ++k) {
    const unsigned row = (gid * 2654435761u + (unsigned)k * 40503u) % n_rows;
    const double* p = x8 + (size_t)row * 8;
    const double2 a = __ldg(reinterpret_cast<const double2*>(p)), b = __ldg(reinterpret_cast<const double2*>(p + 2));
    const double2 e = __ldg(reinterpret_cast<const double2*>(p + 4));
    acc += a.x + a.y + b.x + b.y + e.x + e.y;
  }
  out[gid] = acc;
}
// k_gather_elem: element-major 64-bit loads (6 x LDG.64: lane l of load k fetches double 32k + l of the warp's 32 rows), no transposition
// back (the sum does not need it): isolates the load side of the chunk-major idea.
__global__ void k_gather_elem(const double* __restrict__ x, unsigned n_rows, int reps, double* out) {
  __shared__ unsigned s_row[8][32];
  const unsigned gid = blockIdx.x * blockDim.x + threadIdx.x, lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  double acc = 0.0;
  for (int k = 0; k < reps; ++k) {
    s_row[w][lane] = (gid * 2654435761u + (unsigned)k * 40503u) % n_rows;
    __syncwarp();
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      const unsigned e = c * 32u + lane, o = e / 6u;
      acc += __ldg(x + (size_t)s_row[w][o] * 6 + (e - o * 6u));
    }
    __syncwarp();
  }
  out[gid] = acc;
}

float time_ms(cudaEvent_t e0, cudaEvent_t e1) { float ms = 0; cudaEventElapsedTime(&ms, e0, e1); return ms; }

}  // namespace

extern "C" int tba_microbench(int device, double* out3) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return -5;
  if (cudaSetDevice(device) != cudaSuccess) return -3;
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const int blocks = sms * 16, threads = 256;
  const size_t nthreads = (size_t)blocks * threads;
  const unsigned n_y = 60000;
  double *d_out = nullptr, *d_y = nullptr;
  if (cudaMalloc(&d_out, nthreads * sizeof(double)) != cudaSuccess || cudaMalloc(&d_y, (size_t)n_y * sizeof(double)) != cudaSuccess) return -3;
  cudaMemset(d_y, 0, (size_t)n_y * sizeof(double));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int iters = 4096, reps = 64;
  double best[3] = {0, 0, 0};
  for (int rep = 0; rep < 6; ++rep) {  // first repetition is the warm-up
    cudaEventRecord(e0); k_dfma<<<blocks, threads>>>(d_out, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
    const double t0 = time_ms(e0, e1) * 1e-3;
    cudaEventRecord(e0); k_red<<<blocks, threads>>>(d_y, n_y, reps); cudaEventRecord(e1); cudaEventSynchronize(e1);
    const double t1 = time_ms(e0, e1) * 1e-3;
    cudaEventRecord(e0); k_gather<<<blocks, threads>>>(d_y, n_y / 6, reps, d_out); cudaEventRecord(e1); cudaEventSynchronize(e1);
    const double t2 = time_ms(e0, e1) * 1e-3;
    if (rep == 0) continue;
    const double v0 = (double)nthreads * iters * 8 * 2 / t0 * 1e-12, v1 = (double)nthreads * reps / t1 * 1e-9, v2 = (double)nthreads * reps / t2 * 1e-9;
    if (v0 > best[0]) best[0] = v0;
    if (v1 > best[1]) best[1] = v1;
    if (v2 > best[2]) best[2] = v2;
  }
  const cudaError_t err = cudaDeviceSynchronize();
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(d_out); cudaFree(d_y);
  if (err != cudaSuccess || cudaGetLastError() != cudaSuccess) return -3;
  out3[0] = best[0]; out3[1] = best[1]; out3[2] = best[2];
  return 0;
}

// out[0] = element-major RED rate (k_red_rows), out[1] = shared-memory fp64 atomicAdd rate (k_smem_atomic),
// out[2] = windowed global RED rate (k_red_win), all in G operations/s; out[3..5] = 48-byte row gather rates in G rows/s of
// k_gather_coop / k_gather_64 / k_gather_elem (compare with tba_microbench's out[2]); best of 5 after a warm-up.  Diagnostics only.
extern "C" int tba_microbench_ex(int device, double* out6) {
  double* out3 = out6;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return -5;
  if (cudaSetDevice(device) != cudaSuccess) return -3;
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const int blocks = sms * 16, threads = 256;
  const size_t nthreads = (size_t)blocks * threads;
  const unsigned n_y = 60000;
  double *d_out = nullptr, *d_y = nullptr;
  if (cudaMalloc(&d_out, nthreads * sizeof(double)) != cudaSuccess || cudaMalloc(&d_y, (size_t)n_y * sizeof(double)) != cudaSuccess) return -3;
  cudaMemset(d_y, 0, (size_t)n_y * sizeof(double));
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int reps = 64;
  double best[6] = {0, 0, 0, 0, 0, 0};
  double* d_x8 = nullptr;
  if (cudaMalloc(&d_x8, (size_t)(n_y / 6) * 8 * sizeof(double)) != cudaSuccess) return -3;
  cudaMemset(d_x8, 0, (size_t)(n_y / 6) * 8 * sizeof(double));
  for (int rep = 0; rep < 6; ++rep) {
    cudaEventRecord(e0); k_gather_coop<<<blocks, threads>>>(d_y, n_y / 6, reps, d_out); cudaEventRecord(e1); cudaEventSynchronize(e1);
    const double g0 = time_ms(e0, e1) * 1e-3;
    cudaEventRecord(e0); k_gather_64<<<blocks, threads>>>(d_x8, n_y / 6, reps, d_out); cudaEventRecord(e1); cudaEventSynchronize(e1);
    const double g1 = time_ms(e0, e1) * 1e-3;
    cudaEventRecord(e0); k_gather_elem<<<blocks, threads>>>(d_y, n_y / 6, reps, d_out); cudaEventRecord(e1); cudaEventSynchronize(e1);
    const double g2 = time_ms(e0, e1) * 1e-3;
    if (rep > 0) {
      const double w0 = (double)nthreads * reps / g0 * 1e-9, w1 = (double)nthreads * reps / g1 * 1e-9, w2 = (double)nthreads * reps / g2 * 1e-9;
      if (w0 > best[3]) best[3] = w0;
      if (w1 > best[4]) best[4] = w1;
      if (w2 > best[5]) best[5] = w2;
    }
    cudaEventRecord(e0); k_red_rows<<<blocks, threads>>>(d_y, n_y / 6, reps); cudaEventRecord(e1); cudaEventSynchronize(e1);
    const double t0 = time_ms(e0, e1) * 1e-3;
    cudaEventRecord(e0); k_smem_atomic<<<blocks, threads>>>(d_out, reps); cudaEventRecord(e1); cudaEventSynchronize(e1);
    const double t1 = time_ms(e0, e1) * 1e-3;
    cudaEventRecord(e0); k_red_win<<<blocks, threads>>>(d_y, n_y, reps); cudaEventRecord(e1); cudaEventSynchronize(e1);
    const double t2 = time_ms(e0, e1) * 1e-3;
    if (rep == 0) continue;
    const double v0 = (double)nthreads * reps / t0 * 1e-9, v1 = (double)nthreads * reps / t1 * 1e-9, v2 = (double)nthreads * reps / t2 * 1e-9;
    if (v0 > best[0]) best[0] = v0;
    if (v1 > best[1]) best[1] = v1;
    if (v2 > best[2]) best[2] = v2;
  }
  const cudaError_t err = cudaDeviceSynchronize();
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(d_out); cudaFree(d_y); cudaFree(d_x8);
  if (err != cudaSuccess || cudaGetLastError() != cudaSuccess) return -3;
  for (int i = 0; i < 6; ++i) out3[i] = best[i];
  return 0;
}

// ---- launch-gap microbenchmark: what does a CG iteration pay for alternating a persistent 220 KB-shared-memory kernel (the matvec)
// with small vector kernels?  All kernels are empty (one store by one thread), queued back to back on the default stream.
// out[0] = us per launch, small kernel alone (64 x 256, no shared memory);  out[1] = us per launch, big kernel alone (one CTA per SM,
// 384 threads, 220 KB dynamic shared memory, every CTA spinning for 40000 cycles ~ 20 us so that the host stays ahead);  out[2] = us per PAIR big + small;  out[3] = the same pair with the small kernel hinted
// to the maximum shared-memory carve-out (cudaFuncAttributePreferredSharedMemoryCarveout = 100: no L1 / shared reconfiguration between
// the two);  out[4] = the same pair with the small kernel itself launched with 220 KB of dynamic shared memory.
namespace {
__global__ void k_gap_small(double* out) { if (blockIdx.x == 0 && threadIdx.x == 0) out[0] = 1.0; }
__global__ void k_gap_small_hint(double* out) { if (blockIdx.x == 0 && threadIdx.x == 0) out[1] = 1.0; }
__global__ void k_gap_small_dyn(double* out) { extern __shared__ double sm_dyn[]; if (blockIdx.x == 0 && threadIdx.x == 0) { sm_dyn[0] = 2.0; out[2] = sm_dyn[0]; } }
__global__ void k_gap_big(double* out, long long spin) {  // every CTA stays for `spin` cycles: the host stays ahead of the GPU with its launches
  extern __shared__ double sm_big[];
  if (threadIdx.x == 0) {
    sm_big[0] = (double)blockIdx.x;
    const long long t0 = clock64();
    while (clock64() - t0 < spin) {}
    if (blockIdx.x == 0) out[3] = sm_big[0];
  }
}
}  // namespace

extern "C" int tba_microbench_gaps(int device, double* out5) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || device < 0 || device >= ndev) return -5;
  if (cudaSetDevice(device) != cudaSuccess) return -3;
  int sms = 132;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const int big_smem = 220 * 1024;
  if (cudaFuncSetAttribute(k_gap_big, cudaFuncAttributeMaxDynamicSharedMemorySize, big_smem) != cudaSuccess ||
      cudaFuncSetAttribute(k_gap_small_dyn, cudaFuncAttributeMaxDynamicSharedMemorySize, big_smem) != cudaSuccess ||
      cudaFuncSetAttribute(k_gap_small_hint, cudaFuncAttributePreferredSharedMemoryCarveout, 100) != cudaSuccess) return -3;
  double* d = nullptr;
  if (cudaMalloc(&d, 64) != cudaSuccess) return -3;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int N = 2000;
  double best[5] = {1e30, 1e30, 1e30, 1e30, 1e30};
  for (int rep = 0; rep < 4; ++rep) {
    for (int mode = 0; mode < 5; ++mode) {
      cudaEventRecord(e0);
      for (int i = 0; i < N; ++i) {
        if (mode != 0) k_gap_big<<<sms, 384, big_smem>>>(d, 40000);
        if (mode == 0 || mode == 2) k_gap_small<<<64, 256>>>(d);
        if (mode == 3) k_gap_small_hint<<<64, 256>>>(d);
        if (mode == 4) k_gap_small_dyn<<<64, 256, big_smem>>>(d);
      }
      cudaEventRecord(e1);
      cudaEventSynchronize(e1);
      const double us = time_ms(e0, e1) * 1e3 / N;
      if (rep > 0 && us < best[mode]) best[mode] = us;
    }
  }
  const cudaError_t err = cudaDeviceSynchronize();
  cudaEventDestroy(e0); cudaEventDestroy(e1);
  cudaFree(d);
  if (err != cudaSuccess || cudaGetLastError() != cudaSuccess) return -3;
  for (int i = 0; i < 5; ++i) out5[i] = best[i];
  return 0;
}
