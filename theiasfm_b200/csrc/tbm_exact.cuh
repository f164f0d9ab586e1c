// tbm_exact.cuh -- pass 2 of the tensor-core matcher (tbm_matcher_tc.cuh): the exact float re-evaluation of the candidates the TF32
// pass selected, in the reference's summation order (distance.h:52-56), and the exhaustive scan of the queries whose candidate list
// overflowed.  Plain CUDA (no wgmma / TMA): also compiled by the SIMT emulation build, where tbm_debug_exact_top2 drives it with
// hand-made candidate lists (tests/test_matcher_host.py).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

namespace tbm_tc {

constexpr int DIM = 128;       // descriptor length (SIFT); 4 swizzle atoms of 32 floats
constexpr int KC = 16;         // candidate slots per query handed to the exact pass (-1 = empty; typically 2..4 are filled)
constexpr int kOverflow = -2;  // cand[q*KC] marker: the exact pass scans every candidate of this query

// ------------------------------------------------------------------ pass 2: exact top-2 among the candidates
// One thread per (query, candidate): the exact squared distance -- float, term by term, no fused multiply-add: L2::operator()
// (distance.h:52-56) as the oracle and k_nn2 evaluate it; then thread 0 of the query picks the best two (ties: lower index).
// q_row[i] = global descriptor row of query i, b_row0[i] / b_rows[i] = first row / number of rows of the candidate image (indices are
// reported relative to b_row0).  A query whose candidate ring overflowed in pass 1 (cand[i*KC] == kOverflow) is scanned exhaustively.
// exact squared distance, float, term by term in index order without fused multiply-add (128-bit loads, same arithmetic)
__device__ __forceinline__ float exact_sqdist(const float* __restrict__ a, const float* __restrict__ b) {
  const float4* a4 = reinterpret_cast<const float4*>(a);
  const float4* b4 = reinterpret_cast<const float4*>(b);
  float s = 0.0f;
#pragma unroll 8
  for (int k = 0; k < DIM / 4; ++k) {
    const float4 x = __ldg(a4 + k), y = __ldg(b4 + k);
    float df = __fsub_rn(x.x, y.x); s = __fadd_rn(s, __fmul_rn(df, df));
    df = __fsub_rn(x.y, y.y); s = __fadd_rn(s, __fmul_rn(df, df));
    df = __fsub_rn(x.z, y.z); s = __fadd_rn(s, __fmul_rn(df, df));
    df = __fsub_rn(x.w, y.w); s = __fadd_rn(s, __fmul_rn(df, df));
  }
  return s;
}
// lexicographic (distance, index) order: what MatchImagePair's partial_sort over index-ordered candidates yields
__device__ __forceinline__ void top2_take(int& bj, float& bd, int& sj, float& sd, int jj, float dd) {
  if (jj < 0) return;
  if (bj < 0 || dd < bd || (dd == bd && jj < bj)) { sj = bj; sd = bd; bj = jj; bd = dd; }
  else if (sj < 0 || dd < sd || (dd == sd && jj < sj)) { sj = jj; sd = dd; }
}
// smem_sqdist: the same sum from shared-memory rows (the term order and the roundings of exact_sqdist)
__device__ __forceinline__ float smem_sqdist(const float* a, const float* b) {
  const float4* a4 = reinterpret_cast<const float4*>(a);
  const float4* b4 = reinterpret_cast<const float4*>(b);
  float s = 0.0f;
#pragma unroll 8
  for (int k = 0; k < DIM / 4; ++k) {
    const float4 x = a4[k], y = b4[k];
    float df = __fsub_rn(x.x, y.x); s = __fadd_rn(s, __fmul_rn(df, df));
    df = __fsub_rn(x.y, y.y); s = __fadd_rn(s, __fmul_rn(df, df));
    df = __fsub_rn(x.z, y.z); s = __fadd_rn(s, __fmul_rn(df, df));
    df = __fsub_rn(x.w, y.w); s = __fadd_rn(s, __fmul_rn(df, df));
  }
  return s;
}

constexpr int XT = 64;             // candidate rows per staged tile
constexpr int XS = DIM + 4;        // padded row stride (floats): conflict-free 128-bit reads, one row per thread
constexpr int kRowLoads = XT * (DIM / 4) / 256;   // 128-bit loads per thread and tile (8)

// Tile staging in two steps so that the kRowLoads loads of a thread are in flight TOGETHER (a load-store loop would serialise them:
// each store waits for its load): fetch into registers (32 consecutive threads = one 512-byte row: coalesced), then store.
// row_of(r) -> global descriptor row of tile row r, or -1.
template <class RowOf>
__device__ __forceinline__ void tile_fetch(const float* __restrict__ d, RowOf row_of, float4 (&v)[kRowLoads]) {
#pragma unroll
  for (int u = 0; u < kRowLoads; ++u) {
    const int e = (int)threadIdx.x + u * 256, r = e / (DIM / 4), k4 = e % (DIM / 4);
    const long long j = row_of(r);
    v[u] = j >= 0 ? __ldg(reinterpret_cast<const float4*>(d + (size_t)j * DIM) + k4) : float4{0.0f, 0.0f, 0.0f, 0.0f};
  }
}
__device__ __forceinline__ void tile_store(float* s_rows, const float4 (&v)[kRowLoads]) {
#pragma unroll
  for (int u = 0; u < kRowLoads; ++u) {
    const int e = (int)threadIdx.x + u * 256, r = e / (DIM / 4), k4 = e % (DIM / 4);
    reinterpret_cast<float4*>(s_rows + r * XS)[k4] = v[u];
  }
}

// Exhaustive scan of ONE query (row `a`, already in shared memory) against candidate rows [base, base + nb) by the whole CTA: tiles of
// XT rows staged with coalesced loads, one row per thread 0 .. XT-1 in the reference's term order, then a top-2 merge of the XT
// scanners.  All 256 threads must call it; m_* are [XT] scratch arrays.
// (The scan is bound by its LSU wavefronts -- load + store + row read = 12 per row -- not by load latency: a register-staged,
// prefetching version of this loop bought nothing, so the plain loop stayed.)
__device__ __forceinline__ void exhaustive_scan(const float* __restrict__ d, const float* s_a, float* s_rows, int base, int nb, float* m_d,
                                                float* m_d2, int* m_j, int* m_j2, int* out_j, float* out_d, float* out_d2) {
  const int tid = threadIdx.x;
  int xbj = -1, xsj = -1; float xbd = 0.0f, xsd = 0.0f;
  for (int r0 = 0; r0 < nb; r0 += XT) {
    __syncthreads();  // the previous tile (or whatever used s_rows / m_* before) is consumed
    const int rows = nb - r0 < XT ? nb - r0 : XT;
    for (int e = tid; e < rows * (DIM / 4); e += 256) {
      const int r = e / (DIM / 4), k4 = e % (DIM / 4);
      reinterpret_cast<float4*>(s_rows + r * XS)[k4] = __ldg(reinterpret_cast<const float4*>(d + (size_t)(base + r0 + r) * DIM) + k4);
    }
    __syncthreads();
    if (tid < rows) top2_take(xbj, xbd, xsj, xsd, r0 + tid, smem_sqdist(s_a, s_rows + tid * XS));
  }
  __syncthreads();
  if (tid < XT) { m_d[tid] = xbd; m_j[tid] = xbj; m_d2[tid] = xsd; m_j2[tid] = xsj; }
  __syncthreads();
  if (tid == 0) {
    int fj = -1, gj = -1; float fd = 0.0f, gd = 0.0f;
    for (int k = 0; k < XT; ++k) { top2_take(fj, fd, gj, gd, m_j[k], m_d[k]); top2_take(fj, fd, gj, gd, m_j2[k], m_d2[k]); }
    *out_j = fj; *out_d = fd; *out_d2 = gj >= 0 ? gd : 0.0f;
  }
}

// k_nn_candidates marks an overflowed query in slot 0 only; slot KC / 2 is also honoured because it is part of the documented
// input format of the tbm_debug_exact_top2 test hook (include/theia_matcher_b200.h), which callers use to build candidate lists.
__device__ __forceinline__ bool list_overflowed(const int* __restrict__ cand, long long qi) {
  return cand[qi * KC] == kOverflow || cand[qi * KC + KC / 2] == kOverflow;
}

constexpr int kExactSmemBytes = (XT + 32) * XS * (int)sizeof(float);  // dynamic shared memory: [XT] candidate rows + [32] query rows

// One CTA = 32 queries, EVERY descriptor row goes through shared memory with coalesced loads.
// Per-lane row loads (32 different rows per load instruction) made the first version of this pass bound by its LSU wavefronts:
//   * the 32 query rows are staged once;
//   * the listed candidates of the 32 queries are compacted into ONE dense work list (ballot / popc per query, prefix over the queries)
//     and evaluated XT rows per tile, one row per thread; a per-query thread then picks its two best from its slice of the list;
//   * a query whose list overflowed in pass 1 is scanned exhaustively by the whole CTA afterwards (exhaustive_scan).
__global__ void __launch_bounds__(256) k_exact_top2(const float* __restrict__ d, const int* __restrict__ q_row, const int* __restrict__ b_row0,
                                                    const int* __restrict__ b_rows, const int* __restrict__ cand, long long n_q,
                                                    int* __restrict__ best_j, float* __restrict__ best_d, float* __restrict__ second_d,
                                                    unsigned long long* __restrict__ n_exhaustive) {
#ifdef TBA_EMULATE
  float* smem = emu::dyn_smem<float>();
#else
  extern __shared__ __align__(16) float smem[];
#endif
  float* s_rows = smem;             // [XT][XS]
  float* s_q = smem + XT * XS;      // [32][XS]
  __shared__ float m_d[XT], m_d2[XT];
  __shared__ int m_j[XT], m_j2[XT];
  __shared__ int s_wj[32 * KC];     // dense work list: global descriptor row ...
  __shared__ float s_wd[32 * KC];   // ... and its exact distance; the entries of query q are [s_off[q], s_off[q + 1]) in slot order
  __shared__ unsigned char s_wq[32 * KC];
  __shared__ int s_cnt[32], s_off[33];
  __shared__ int s_ovf[32];
  __shared__ int s_novf;
  const int tid = threadIdx.x, lane = tid & 31;
  const long long q0 = (long long)blockIdx.x * 32;
  const int nq_cta = (int)((n_q - q0) < 32 ? (n_q - q0) : 32);
  if (tid == 0) s_novf = 0;
  // ---- the query rows (4 loads per thread, together in flight)
  {
    float4 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int e = tid + u * 256, r = e / (DIM / 4), k4 = e % (DIM / 4);
      v[u] = r < nq_cta ? __ldg(reinterpret_cast<const float4*>(d + (size_t)q_row[q0 + r] * DIM) + k4) : float4{0.0f, 0.0f, 0.0f, 0.0f};
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int e = tid + u * 256, r = e / (DIM / 4), k4 = e % (DIM / 4);
      reinterpret_cast<float4*>(s_q + r * XS)[k4] = v[u];
    }
  }
  // ---- dense work list: entry e = (query e / 16, slot e % 16), two entries per thread; a warp covers two queries
  int my_j[2], my_rank[2];
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int e = it * 256 + tid, q = e >> 4, k = e & 15;
    int j = -1;
    if (q < nq_cta && !list_overflowed(cand, q0 + q)) j = cand[(q0 + q) * KC + k];
    const unsigned b = __ballot_sync(0xffffffffu, j >= 0);
    const unsigned m16 = (b >> (lane & 16)) & 0xFFFFu;
    my_j[it] = j;
    my_rank[it] = __popc(m16 & ((1u << (lane & 15)) - 1u));
    if ((lane & 15) == 0) s_cnt[q] = __popc(m16);
  }
  __syncthreads();  // s_q, s_cnt, s_novf = 0
  if (tid == 0) {
    int o = 0;
    for (int q = 0; q < 32; ++q) { s_off[q] = o; o += s_cnt[q]; }
    s_off[32] = o;
  }
  if (tid < nq_cta && list_overflowed(cand, q0 + tid)) {
    s_ovf[atomicAdd(&s_novf, 1)] = tid;
    if (n_exhaustive) atomicAdd(n_exhaustive, 1ull);
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int e = it * 256 + tid, q = e >> 4;
    if (my_j[it] >= 0) { const int w = s_off[q] + my_rank[it]; s_wj[w] = my_j[it]; s_wq[w] = (unsigned char)q; }
  }
  __syncthreads();
  const int n_work = s_off[32];
  {
    float4 v[kRowLoads];
    if (n_work > 0) tile_fetch(d, [&](int r) { return r < n_work ? (long long)s_wj[r] : -1ll; }, v);
    for (int w0 = 0; w0 < n_work; w0 += XT) {
      __syncthreads();  // the previous tile is consumed
      tile_store(s_rows, v);
      __syncthreads();
      const int next = w0 + XT;
      if (next < n_work) tile_fetch(d, [&](int r) { return next + r < n_work ? (long long)s_wj[next + r] : -1ll; }, v);
      if (tid < XT && w0 + tid < n_work) s_wd[w0 + tid] = smem_sqdist(s_q + (int)s_wq[w0 + tid] * XS, s_rows + tid * XS);
    }
  }
  __syncthreads();
  if (tid < nq_cta && !list_overflowed(cand, q0 + tid)) {
    const long long qi = q0 + tid;
    const int base = b_row0[qi];
    int fj = -1, gj = -1; float fd = 0.0f, gd = 0.0f;
    for (int w = s_off[tid]; w < s_off[tid + 1]; ++w) top2_take(fj, fd, gj, gd, s_wj[w] - base, s_wd[w]);
    best_j[qi] = fj; best_d[qi] = fd; second_d[qi] = gj >= 0 ? gd : 0.0f;
  }
  // ---- exhaustive scans, one overflowed query of this CTA after the other
  const int novf = s_novf;
  for (int o = 0; o < novf; ++o) {
    const int ql = s_ovf[o];
    const long long qx = q0 + ql;
    exhaustive_scan(d, s_q + ql * XS, s_rows, b_row0[qx], b_rows[qx], m_d, m_d2, m_j, m_j2, best_j + qx, best_d + qx, second_d + qx);
  }
}

}  // namespace tbm_tc
