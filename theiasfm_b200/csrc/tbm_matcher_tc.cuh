// tbm_matcher_tc.cuh -- tensor-core path of the brute-force matcher (SURVEY 8 row a16; sm_90a: wgmma + TMA + mbarrier).
//
// Replaces the hot loop of BruteForceFeatureMatcher::MatchImagePair
// (src/theia/matching/brute_force_feature_matcher.cc:64-82 forward, :93-112 reverse; L2::operator() distance.h:52-56):
// for every descriptor of one image the two nearest descriptors of the other image in squared L2.
//
// Two passes per (image pair, direction):
//   1. k_nn_candidates (this file): ||x - y||^2 = ||x||^2 + ||y||^2 - 2 x.y with the 128-dimensional dot products as a TF32
//      wgmma GEMM -- a 128-query block of image A (resident in shared memory) against 64-candidate tiles of image B streamed
//      by TMA (cp.async.bulk.tensor, 128-byte swizzle, NSTAGE-deep ring) -- and a fused epilogue on the fp32 accumulator
//      registers that keeps, per query row, the candidates whose score interval (||y||^2 - 2 x.y widened by its TF32 and float
//      error bounds) reaches below the runner-up's (branch-free, lists in shared memory).
//      Warp roles: warpgroup 0 = TMA producer (one thread), warpgroups 1 and 2 = consumers: each issues the m64n64k8 wgmmas
//      of its 64 query rows and scans its accumulators.  Persistent CTAs over a list of work items.
//   2. k_exact_top2: the KC candidates of every query are re-evaluated EXACTLY -- float, term by term in the reference's
//      order without fused multiply-add, like the round-1 kernel k_nn2 -- and the best two (ties: lower index) are kept.
// TF32 only ranks candidates; every distance that leaves the GPU, every ratio test and every tie-break is computed from
// the exact values, so the match lists equal the CPU oracle's: the reference's nearest and second-nearest neighbours always reach
// the exact pass (see the epilogue comment; tests/test_xx_matcher_gpu_adversarial.py checks it at the inputs where it is tightest).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>

#include <cstdint>

#include "tbm_exact.cuh"  // DIM, KC, ET, kOverflow + the exact re-evaluation kernel (plain CUDA, shared with the emulation build)

namespace tbm_tc {

constexpr int BM = 128;        // query rows per work item (two consumer warpgroups x 64 rows)
constexpr int BN = 64;         // candidate rows per tile (= accumulator columns of one m64n64 wgmma)
constexpr int WG_ROWS = 64;    // query rows of one consumer warpgroup
constexpr int CAP = 15;        // list slots per (query, column quarter) in shared memory: 11 usable (a list that reaches slot 11 => exact full scan of that query) + 4 spare behind them (pointer clamped once per four appends)
constexpr int PANEL_BYTES = 64 * 128;             // one 64-row x 128-byte swizzle-atom panel (32 floats of 64 rows)
constexpr int A_BYTES = 2 * 4 * PANEL_BYTES;      // 64 KB: the 128 x 128 float query block, [warpgroup][atom panel]
constexpr int B_BYTES = 4 * PANEL_BYTES;          // 32 KB: a 64 x 128 float candidate tile
constexpr int NSTAGE = 3;
constexpr int THREADS = 3 * 128;
constexpr int NLISTS = 2 * 256;                   // candidate lists: two query rows per consumer thread

struct WorkItem {
  int a_row0;    // global row of the first query of this block
  int a_rows;    // valid query rows (1..128)
  int b_row0;    // global row of the first candidate of image B
  int b_rows;    // number of candidates
  long long out_row0;  // first row of this block in the candidate-index output
};

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(uint64_t* b, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void bar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_addr(b)) : "memory");
}
__device__ __forceinline__ bool bar_try(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_addr(b)), "r"(parity) : "memory");
  return ok != 0;
}
// (no printf on the timeout: a function call anywhere in the kernel makes ptxas serialise the wgmma pipeline)
__device__ __forceinline__ void bar_wait(uint64_t* b, uint32_t parity) {
  if (bar_try(b, parity)) return;
  const long long t0 = clock64();
  while (!bar_try(b, parity)) {
    if (clock64() - t0 > 4000000000ll) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_addr(dst)), "l"(map), "r"(smem_addr(bar)), "r"(c0), "r"(c1) : "memory");
}
// Shared-memory matrix descriptor of wgmma (sm_90): K-major operand, 128-byte swizzle, 8-row groups 1024 bytes apart.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);        // start address, 16-byte units
  d |= (uint64_t)1 << 16;                        // leading byte offset (unused with swizzled K-major layouts): 1
  d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset: 8 rows x 128 bytes
  d |= (uint64_t)1 << 62;                        // layout type SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 64] (+)= A[smem, 64 x 8] * B[smem, 64 x 8]^T, both operands K-major, TF32 inputs, fp32 accumulation in registers
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t desc_a, uint64_t desc_b, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
        "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
        "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(desc_a), "l"(desc_b), "r"(accumulate)
      : "memory");
}
// keeps the compiler from moving accumulator reads above the wait of the asynchronous wgmma
__device__ __forceinline__ void acc_fence(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

struct __align__(8) Ctl {
  uint64_t a_full, a_empty, b_full[NSTAGE], b_empty[NSTAGE];
};

// ------------------------------------------------------------------ pass 1: TF32 candidates
// desc_map: the concatenated descriptor matrix [total_rows][128] float as a 2-D tensor map, box = 32 floats x 64 rows, SWIZZLE_128B.
// nrm[r] = ||descriptor r||^2 (float).  cand[(out_row0 + m) * KC + k] = global row of the k-th candidate of query m (-1: none).
template <bool NONNEG>
__global__ void __launch_bounds__(THREADS, 1) k_nn_candidates(const __grid_constant__ CUtensorMap desc_map, const WorkItem* __restrict__ items,
                                                              int n_items, const float* __restrict__ nrm, int* __restrict__ cand) {
  extern __shared__ uint8_t smem_raw[];
  // 128-byte-swizzled operand panels must start on 1024-byte boundaries (of the shared-memory address)
  uint8_t* smem = smem_raw + ((1024u - (smem_addr(smem_raw) & 1023u)) & 1023u);
  uint8_t* sA = smem;                                  // [2 warpgroups][4 atom panels] of the query block
  uint8_t* sB = smem + A_BYTES;                        // NSTAGE x 4 atom panels of candidate tiles
  uint2* sC = reinterpret_cast<uint2*>(smem + A_BYTES + (size_t)NSTAGE * B_BYTES);  // [CAP][NLISTS] provisional candidates (score bits, row)
  Ctl* ctl = reinterpret_cast<Ctl*>(smem + A_BYTES + (size_t)NSTAGE * B_BYTES + (size_t)CAP * NLISTS * sizeof(uint2));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    bar_init(&ctl->a_full, 1); bar_init(&ctl->a_empty, 8);
    for (int s = 0; s < NSTAGE; ++s) { bar_init(&ctl->b_full[s], 1); bar_init(&ctl->b_empty[s], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      uint32_t bt = 0, itc = 0;
      for (int it = blockIdx.x; it < n_items; it += gridDim.x, ++itc) {
        const WorkItem w = items[it];
        bar_wait(&ctl->a_empty, (itc & 1) ^ 1);          // the wgmmas of the previous item have read sA
        bar_expect_tx(&ctl->a_full, A_BYTES);
        for (int g = 0; g < 2; ++g)
          for (int a = 0; a < 4; ++a) tma_load_2d(sA + (g * 4 + a) * PANEL_BYTES, &desc_map, a * 32, w.a_row0 + g * WG_ROWS, &ctl->a_full);
        const int n_tiles = (w.b_rows + BN - 1) / BN;
        for (int t = 0; t < n_tiles; ++t, ++bt) {
          const int s = bt % NSTAGE;
          bar_wait(&ctl->b_empty[s], ((bt / NSTAGE) & 1) ^ 1);
          bar_expect_tx(&ctl->b_full[s], B_BYTES);
          for (int a = 0; a < 4; ++a) tma_load_2d(sB + (size_t)s * B_BYTES + a * PANEL_BYTES, &desc_map, a * 32, w.b_row0 + t * BN, &ctl->b_full[s]);
        }
      }
    }
  } else {
    // ===================== consumers: wgmma + epilogue on the accumulator registers =====================
    // Accumulator layout of m64n64 (per warp w of the warpgroup, lane l): d[4j + 2i + c] = row 16w + l/4 + 8i, column 8j + 2(l%4) + c.
    // A thread therefore owns two query rows (i = 0, 1) and one column quarter (l % 4) of each: 16 of the 64 columns of every tile.
    //
    // Branch-free streaming selection.  Every element n of the row (query x, candidate y_n) gets an interval [lo_n, up_n] of
    // float scores that must contain the reference's distance D_n = fl(sum_k (x_k - y_nk)^2) minus ||x||^2, and an element can only be
    // among the two nearest when lo_n <= the second smallest up of the row: were lo_n > up_c1, up_c2 for two other elements, both
    // would be strictly nearer than n in the reference's own arithmetic.  Per (row, quarter) the thread keeps the running two smallest
    // up, m1 <= m2 (three min/max per element), and appends an element to its candidate list in shared memory -- one predicated
    // 8-byte store, no branch, no divergence -- whenever lo_n <= m2 (m2 only decreases, so a true top-2 element passes when it is
    // seen and at every later compaction).  lo and up are the computed score ||y_n||^2 - 2 acc_n minus / plus the bound of its
    // distance from D_n - ||x||^2 (X = ||x||^2, Y = ||y_n||^2, A = sum_k |x_k y_nk|, p = x.y_n, d = X + Y - 2p):
    //   * TF32 operands: wgmma .tf32 uses the top 10 mantissa bits of each fp32 operand and ignores the low 13 -- truncation toward
    //     zero, which an H100 does (tests/test_xx_matcher_gpu_adversarial.py::test_tf32_operands_are_truncated pins it): an operand
    //     loses < 2^-10 of itself.  The products are exact in fp32; the fp32 accumulation of 128 of them errs <= 2^-16 A either way.
    //     With non-negative data every product only shrinks: acc - p lies in [-2^-9 A (1 + 2^-7), +2^-16 A], i.e. the score
    //     ||y||^2 - 2 acc errs by at most 2^-8 A (1 + 2^-7) upward and 2^-15 A downward; with signed data by 2^-8 A either way;
    //   * the float norm nrm[n] (k_row_norms' order) differs from Y by <= 2^-19 Y, the reference's sum D_n from d by <= 2^-17 d (a
    //     left-to-right sum of 128 rounded squares), and the roundings of lo / up add <= 2^-22 (X + Y + A): <= 2^-16 (X + Y) with d <= X + Y;
    //   * NONNEG (every descriptor component >= 0: SIFT, RootSIFT, any histogram descriptor): A = p = acc (1 + 2^-9), d <= X + Y:
    //       lo = Y (1 - 2^-16) - acc (2 + 2^-8 + 2^-14) - 2^-16 X,   up = Y (1 + 2^-16) - acc (2 - 2^-14) + 2^-16 X;
    //   * otherwise A <= ||x|| ||y|| <= (X + Y) / 2 and d <= 2 (X + Y):
    //       lo = Y (1 - b) - 2 acc - b X,   up = Y (1 + b) - 2 acc + b X,   b = 2^-9 (1 + 2^-4).
    // The norm terms keep the interval open where the TF32 term vanishes (a zero query or candidate, disjoint supports: x.y = 0),
    // and since lo_n <= up_n always, the comparison "<=" keeps the runner-up itself and every exact tie.  The kernel keeps lo and up
    // scaled (lo', up' below: one FMA each off the plain norm, as cheap as a bare score) and compares lo' with the running limit
    // kK m2' + kX X (one more FMA per element).  m1', m2' start at 2^126 instead of +inf, so the limit stays finite: out-of-range
    // columns of the last tile (lo' = up' = +inf) are never appended.
    // At the end of an item the four quarters of a row merge their (m1, m2) by shuffles; the entries within the row's own limit are
    // written to the KC slots of the query for the exact pass.  A list that fills up, or a row with more than KC such entries (a dense
    // cluster of near-identical candidates), flags the row: the exact pass then scans every candidate of that query.
    // The first tile is scanned twice: once only to establish m1, m2 (otherwise every element of it would be appended).
    const int g = warp / 4 - 1;              // consumer warpgroup: query rows [64 g, 64 g + 64) of the block
    const int wl = warp & 3;
    const int et = threadIdx.x - 128;        // 0..255 among the consumer threads
    const int cq = lane & 3;                 // column quarter
    const float kInf = __int_as_float(0x7f800000), kBig = 0x1p126f;
    // the interval scaled per side so that both ends are one FMA off the plain norm: lo' = (lo + b X) / (1 - b) = fmaf(kLo, acc, nrm),
    // up' = (up - b X) / (1 + b) = fmaf(kUp, acc, nrm); lo <= up_2 + b X  <=>  lo' <= kK up'_2 + kX X  (kK = (1 + b) / (1 - b),
    // kX = 2 b / (1 - b)).  Each constant is rounded away from the tighter side (|kLo|, kK, kX up; |kUp| down).
    // NONNEG: b = 2^-16, lo / up TF32 coefficients 2 + 2^-8 + 2^-14 / 2 - 2^-14;  otherwise: b = 2^-9 + 2^-13, both 2
    constexpr float kLo = NONNEG ? -0x1.0083020000000p+1f : -0x1.00884a0000000p+1f;
    constexpr float kUp = NONNEG ? -0x1.fffa000000000p+0f : -0x1.fef0900000000p+0f;
    constexpr float kK = NONNEG ? 0x1.0002020000000p+0f : 0x1.0110920000000p+0f;
    constexpr float kX = NONNEG ? 0x1.0001020000000p-15f : 0x1.1090ce0000000p-8f;
    constexpr uint32_t kStride = NLISTS * (uint32_t)sizeof(uint2);   // bytes between consecutive entries of one list
    const uint32_t a_base = smem_addr(sA + g * 4 * PANEL_BYTES);
    float acc[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) acc[k] = 0.0f;
    uint32_t bt = 0, itc = 0;
    for (int it = blockIdx.x; it < n_items; it += gridDim.x, ++itc) {
      const WorkItem w = items[it];
      int row[2];
      float m1[2], m2[2], xm[2];
      uint32_t c_base[2], c_last[2], wp[2];
      int ovf[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        row[i] = g * WG_ROWS + wl * 16 + (lane >> 2) + 8 * i;   // query row of this thread inside the block
        m1[i] = kBig; m2[i] = kBig;
        xm[i] = row[i] < w.a_rows ? kX * __ldg(nrm + w.a_row0 + row[i]) : 0.0f;  // the row term of the limit
        // wp = shared-memory address of the next append; it saturates at the last slot, and a list that reaches the last slot
        // counts as overflowed (capacity CAP - 4 entries between two maintenance points)
        c_base[i] = smem_addr(sC + i * 256 + et);
        c_last[i] = c_base[i] + (CAP - 4) * kStride;
        wp[i] = c_base[i];
        ovf[i] = 0;
      }
      bar_wait(&ctl->a_full, itc & 1);
      const int n_tiles = (w.b_rows + BN - 1) / BN;
      for (int t = 0; t < n_tiles; ++t, ++bt) {
        const int s = bt % NSTAGE;
        bar_wait(&ctl->b_full[s], (bt / NSTAGE) & 1);
        __syncwarp();   // wgmma is .sync.aligned: the warp must be converged after the spin of the wait
        const uint32_t b_base = smem_addr(sB + (size_t)s * B_BYTES);
        wg_fence();
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int k = 0; k < 4; ++k)  // K = 8 tf32 = 32 bytes inside the 128-byte swizzle atom
            wgmma_tf32(acc, make_desc(a_base + a * PANEL_BYTES + k * 32), make_desc(b_base + a * PANEL_BYTES + k * 32), (a | k) != 0);
        wg_commit();
        // squared norms of this thread's 16 columns of the tile, loaded while the wgmmas run
        float nn[8][2];
        const int jt = t * BN + 2 * cq;
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int c = 0; c < 2; ++c) nn[j][c] = jt + 8 * j + c < w.b_rows ? __ldg(nrm + w.b_row0 + jt + 8 * j + c) : kInf;
        wg_wait0();
        acc_fence(acc);
        __syncwarp();
        if (lane == 0) {
          bar_arrive(&ctl->b_empty[s]);                   // this warp's wgmmas have read the stage
          if (t == n_tiles - 1) bar_arrive(&ctl->a_empty);  // ... and the query block
        }
        const int jg = w.b_row0 + jt;   // global row of column (j = 0, c = 0)
        // one predicated 8-byte store + pointer bump per element; the pointer is clamped to the last slot once per FOUR elements
        // (TBM_CLAMP): at most four appends can happen in between, and the lists keep four spare slots behind c_last for them
#define TBM_APPEND(I, VAL, J)                                                                                           \
  asm volatile("{\n\t.reg .pred p;\n\tsetp.le.f32 p, %1, %2;\n\t@p st.shared.v2.b32 [%0], {%3, %4};\n\t@p add.u32 %0, %0, %5;\n\t}"      \
               : "+r"(wp[I]) : "f"(VAL), "f"(lim), "r"(__float_as_uint(VAL)), "r"(J), "n"(kStride) : "memory")
#define TBM_CLAMP(I) wp[I] = min(wp[I], c_last[I])
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          if (t == 0) {  // tile 0: m1, m2 first, then the appends against them (counting an element twice would turn the best into its own runner-up)
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                const float up = fmaf(kUp, acc[4 * j + 2 * i + c], nn[j][c]);
                m2[i] = fminf(m2[i], fmaxf(m1[i], up));
                m1[i] = fminf(m1[i], up);
              }
          }
          if (t == 0) {
            const float lim = fmaf(m2[i], kK, xm[i]);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                const float lo = fmaf(kLo, acc[4 * j + 2 * i + c], nn[j][c]);
                TBM_APPEND(i, lo, jg + 8 * j + c);
              }
              if (j & 1) TBM_CLAMP(i);
            }
          } else {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                const float dotv = acc[4 * j + 2 * i + c];
                const float lo = fmaf(kLo, dotv, nn[j][c]);
                const float up = fmaf(kUp, dotv, nn[j][c]);
                const float lim = fmaf(m2[i], kK, xm[i]);
                TBM_APPEND(i, lo, jg + 8 * j + c);
                m2[i] = fminf(m2[i], fmaxf(m1[i], up));
                m1[i] = fminf(m1[i], up);
              }
              if (j & 1) TBM_CLAMP(i);
            }
          }
          // list maintenance, once per tile (rare per lane; divergent, but cheap)
          ovf[i] |= wp[i] == c_last[i];
          if (wp[i] > c_base[i] + 8 * kStride) {
            const int cnt = (int)((wp[i] - c_base[i]) / kStride);
            const float lim = fmaf(m2[i], kK, xm[i]);
            uint2* myC = sC + i * 256 + et;
            int k = 0;
            for (int e = 0; e < cnt; ++e) {
              const uint2 ce = myC[e * NLISTS];
              if (__uint_as_float(ce.x) <= lim) { myC[k * NLISTS] = ce; ++k; }
            }
            wp[i] = c_base[i] + (uint32_t)k * kStride;
          }
        }
#undef TBM_APPEND
#undef TBM_CLAMP
      }
      // ---- the row's runner-up over its four quarters (lanes 4r .. 4r + 3), then the kept entries into the KC slots of the query
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float r1 = m1[i], r2 = m2[i];
#pragma unroll
        for (int o = 1; o <= 2; o <<= 1) {
          const float o1 = __shfl_xor_sync(0xffffffffu, r1, o), o2 = __shfl_xor_sync(0xffffffffu, r2, o);
          r2 = fminf(fmaxf(r1, o1), fminf(r2, o2));
          r1 = fminf(r1, o1);
        }
        const float lim = fmaf(r2, kK, xm[i]);   // the row's final limit: only entries with lo' <= it can be among the two nearest
        const uint2* myC = sC + i * 256 + et;
        const int cnt = (int)((wp[i] - c_base[i]) / kStride);
        int k = 0;
        for (int e = 0; e < cnt; ++e) k += __uint_as_float(myC[e * NLISTS].x) <= lim;
        int before = 0, total = 0, any_ovf = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int kq = __shfl_sync(0xffffffffu, k, (lane & ~3) | q);
          total += kq;
          before += q < cq ? kq : 0;
          any_ovf |= __shfl_sync(0xffffffffu, ovf[i], (lane & ~3) | q);
        }
        if (row[i] < w.a_rows) {
          int* o = cand + (size_t)(w.out_row0 + row[i]) * KC;
          if (any_ovf || total > KC) {
            if (cq == 0) o[0] = kOverflow;
          } else {
            int n = before;
            for (int e = 0; e < cnt; ++e) {
              const uint2 ce = myC[e * NLISTS];
              if (__uint_as_float(ce.x) <= lim) o[n++] = (int)ce.y;
            }
            if (cq == 3) for (int q = total; q < KC; ++q) o[q] = -1;
          }
        }
      }
    }
  }
}

// ||d||^2 of every descriptor row (float, plain left-to-right sum: only used to RANK candidates); *any_negative is set when a
// component < 0 exists anywhere (selects the general TF32 error margin instead of the tighter one of non-negative descriptors)
__global__ void k_row_norms(const float* __restrict__ d, long long n_rows, float* __restrict__ nrm, int* __restrict__ any_negative) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  const float4* p = reinterpret_cast<const float4*>(d + r * DIM);
  float s = 0.0f, mn = 0.0f;
#pragma unroll 8
  for (int k = 0; k < DIM / 4; ++k) {
    const float4 x = __ldg(p + k);
    s += x.x * x.x + x.y * x.y + x.z * x.z + x.w * x.w;
    mn = fminf(mn, fminf(fminf(x.x, x.y), fminf(x.z, x.w)));
  }
  nrm[r] = s;
  if (mn < 0.0f) *any_negative = 1;
}

// ------------------------------------------------------------------ host helpers
inline bool make_desc_map(CUtensorMap* map, const float* d_desc, long long n_rows) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) return false;
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)DIM, (cuuint64_t)n_rows};
  const cuuint64_t strides[1] = {(cuuint64_t)DIM * sizeof(float)};
  const cuuint32_t box[2] = {32u, (cuuint32_t)BN};
  const cuuint32_t estr[2] = {1u, 1u};
  return encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(d_desc), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

constexpr size_t kSmemBytes = (size_t)A_BYTES + (size_t)NSTAGE * B_BYTES + (size_t)CAP * NLISTS * sizeof(uint2) + sizeof(Ctl) + 1024;
static_assert(kSmemBytes <= 227 * 1024, "k_nn_candidates must fit the 227 KB of shared memory an H100 block can have");
static_assert(BN == WG_ROWS, "one tensor map (box 32 floats x 64 rows) serves both operands");

}  // namespace tbm_tc
