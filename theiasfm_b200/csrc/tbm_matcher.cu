// tbm_matcher.cu -- secondary path (SURVEY 8 row a16): brute-force descriptor matching on the GPU, C-ABI of
// include/theia_matcher_b200.h.  Round-1 kernel: CUDA cores, exact float arithmetic in the reference's order (so the
// match sets are bit-identical to the CPU restatement); dim 128 takes the wgmma distance GEMM of tbm_matcher_tc.cuh.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <vector>

#include "../../include/theia_matcher_b200.h"
#include "tbm_top2.h"
#include "tbm_decide.cuh"       // MatchImagePair's decisions on the device (ratio test, early exits, IntersectMatches)
#include "tbm_exact.cuh"        // exact re-evaluation of the tensor-core path's candidates (plain CUDA: in both builds)
#ifndef TBA_EMULATE
#include "tbm_matcher_tc.cuh"   // wgmma / TMA path (sm_90a); the SIMT emulation build keeps the exact CUDA-core kernels only
#endif
#include <cstdlib>

static double g_last_timing[4] = {0, 0, 0, 0};  // ms: candidate GEMM kernel, exact re-evaluation kernel, H2D of the descriptors; [3] = queries scanned exhaustively

namespace {

constexpr int ROWS = 32;    // query descriptors per CTA (= lanes of a warp)
constexpr int SLICES = 8;   // warps per CTA; warp w scans candidate rows w, w+8, ... of every tile
constexpr int TJ = 32;      // candidate descriptors per shared-memory tile

using tbm::Top2;
using tbm::top2_push;

// For every row i of A: the nearest (squared L2, ties -> lower index) and second-nearest distance among the rows of B.
// Distances are accumulated left to right in float WITHOUT fused multiply-add: s = s + (a-b)*(a-b), exactly
// L2::operator() evaluated term by term (distance.h:52-56).
__global__ void __launch_bounds__(ROWS* SLICES) k_nn2(const float* __restrict__ A, int nA, const float* __restrict__ B, int nB, int dim,
                                                      int* __restrict__ best_j, float* __restrict__ best_d, float* __restrict__ second_d) {
#ifdef TBA_EMULATE  // CPU emulation build (tests/emu)
  float* smem = emu::dyn_smem<float>();
#else
  extern __shared__ float smem[];
#endif
  const int dimp = dim + 1;                 // padded row stride of the query tile: conflict-free column access
  float* sA = smem;                         // [ROWS][dimp]
  float* sB = smem + ROWS * dimp;           // [TJ][dim]
  __shared__ Top2 s_merge[SLICES][ROWS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int i0 = blockIdx.x * ROWS;
  for (int idx = threadIdx.x; idx < ROWS * dim; idx += ROWS * SLICES) {
    const int r = idx / dim, k = idx - r * dim;
    sA[r * dimp + k] = (i0 + r < nA) ? A[(size_t)(i0 + r) * dim + k] : 0.0f;
  }
  Top2 t;
  tbm::top2_init(t);
  for (int j0 = 0; j0 < nB; j0 += TJ) {
    __syncthreads();  // previous tile consumed (and sA written, first time)
    for (int idx = threadIdx.x; idx < TJ * dim; idx += ROWS * SLICES) {
      const int r = idx / dim, k = idx - r * dim;
      sB[idx] = (j0 + r < nB) ? B[(size_t)(j0 + r) * dim + k] : 0.0f;
    }
    __syncthreads();
    for (int jj = warp; jj < TJ; jj += SLICES) {
      const int j = j0 + jj;
      if (j >= nB) break;
      const float* a = sA + lane * dimp;
      const float* b = sB + jj * dim;
      float s = 0.0f;
      for (int k = 0; k < dim; ++k) {
        const float d = __fsub_rn(a[k], b[k]);
        s = __fadd_rn(s, __fmul_rn(d, d));
      }
      top2_push(t, s, j);
    }
  }
  s_merge[warp][lane] = t;
  __syncthreads();
  if (warp == 0 && i0 + lane < nA) {
    // merge the 8 scanners (tbm_top2.h)
    Top2 m = s_merge[0][lane];
    for (int w = 1; w < SLICES; ++w) tbm::top2_merge(m, s_merge[w][lane]);
    best_j[i0 + lane] = m.bj;
    best_d[i0 + lane] = m.bd;
    second_d[i0 + lane] = m.has2 ? m.sd : 0.0f;
  }
}

template <class T>
struct Dev {
  T* p = nullptr; size_t n = 0;
  Dev() = default;
  Dev(const Dev&) = delete;
  Dev& operator=(const Dev&) = delete;
  ~Dev() { if (p) cudaFree(p); }
  bool alloc(size_t c) {
    if (c <= n && p) return true;
    if (p) cudaFree(p);
    p = nullptr; n = 0;
    if (cudaMalloc(&p, (c ? c : 1) * sizeof(T)) != cudaSuccess) return false;
    n = c;
    return true;
  }
};
using DevF = Dev<float>;
using DevI = Dev<int>;

#ifdef TBA_EMULATE
#define TBM_LAUNCH(kern, grid, block, smem, ...) emu::launch((const void*)(kern), (unsigned)(grid), (unsigned)(block), (size_t)(smem), [&] { kern(__VA_ARGS__); })
#else
#define TBM_LAUNCH(kern, grid, block, smem, ...) kern<<<(grid), (block), (smem)>>>(__VA_ARGS__)
#endif

static_assert(sizeof(tbm_match) == 12, "k_gather_matches copies a match as three 32-bit words");

// Per-query results of the nearest-neighbour stage (what k_pair_decide consumes), copied to the host after every chunk / pair for
// tbm_debug_nn2; layout per pair: forward queries [n1], then reverse queries [n2] when matching is symmetric.  nullptr: normal call.
struct Nn2Out {
  int32_t* best_j; float* best_d; float* second_d; uint8_t* exhaustive;
};

// Device buffers of the decision stage, kept for the whole call (grown on demand).
struct DecideBuffers {
  Dev<tbm::PairSeg> segs;
  Dev<tbm_match> staged, packed;
  Dev<int> count;
  Dev<uint8_t> ok;
  Dev<long long> dst_off;
  std::vector<int> h_count;
  std::vector<uint8_t> h_ok;
  std::vector<long long> h_off;
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  double kernel_ms = 0.0;  // device time of k_pair_decide + k_gather_matches, summed over the chunks of a call
  ~DecideBuffers() { for (auto e : ev) if (e) cudaEventDestroy(e); }
};

// The pairs `segs` (results of both directions in best_j / best_d / second_d on the device, `n_fwd_queries` forward queries in
// all): decisions on the device, kept matches packed and copied to matches[*written ...], match_off / pair_ok filled for pairs
// [p0, p0 + segs.size()).  Returns 0 or a negative tbm code; *overflow is set when the caller's capacity is too small.
int decide_and_fetch(DecideBuffers& B, const std::vector<tbm::PairSeg>& segs, long long n_queries, const int* best_j, const float* best_d,
                     const float* second_d, const tbm_options* options, int64_t p0, tbm_match* matches, int64_t cap, int64_t* written,
                     int64_t* match_off, uint8_t* pair_ok, bool* overflow) {
  const int np = (int)segs.size();
  if (np == 0) return 0;
  tbm::DecideOptions o;
  o.symmetric = options->keep_only_symmetric_matches != 0; o.use_ratio = options->use_lowes_ratio != 0; o.min_matches = options->min_num_feature_matches;
  o.ratio_sq = options->lowes_ratio * options->lowes_ratio;
  const size_t nq = (size_t)(n_queries > 0 ? n_queries : 1);
  if (!B.segs.alloc((size_t)np) || !B.staged.alloc(nq) || !B.packed.alloc(nq) || !B.count.alloc((size_t)np) || !B.ok.alloc((size_t)np) || !B.dst_off.alloc((size_t)np)) return -3;
  if (cudaMemcpy(B.segs.p, segs.data(), (size_t)np * sizeof(tbm::PairSeg), cudaMemcpyHostToDevice) != cudaSuccess) return -3;
  const int grid = np < 4096 ? np : 4096;
  for (auto& e : B.ev) if (!e && cudaEventCreate(&e) != cudaSuccess) return -3;
  cudaEventRecord(B.ev[0]);
  TBM_LAUNCH(tbm::k_pair_decide, grid, tbm::kDecideThreads, 0, B.segs.p, np, best_j, best_d, second_d, o, B.staged.p, B.count.p, B.ok.p);
  if (cudaPeekAtLastError() != cudaSuccess) return -3;
  cudaEventRecord(B.ev[1]);
  B.h_count.resize((size_t)np); B.h_ok.resize((size_t)np); B.h_off.resize((size_t)np);
  if (cudaMemcpy(B.h_count.data(), B.count.p, (size_t)np * sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(B.h_ok.data(), B.ok.p, (size_t)np, cudaMemcpyDeviceToHost) != cudaSuccess) return -3;
  { float ms = 0; if (cudaEventElapsedTime(&ms, B.ev[0], B.ev[1]) == cudaSuccess) B.kernel_ms += ms; }
  long long total = 0;
  for (int k = 0; k < np; ++k) {
    B.h_off[(size_t)k] = total;
    match_off[p0 + k] = *written + total;
    pair_ok[p0 + k] = B.h_ok[(size_t)k];
    total += B.h_count[(size_t)k];
  }
  if (total > 0) {
    if (*written + total > cap || !matches) *overflow = true;
    else {
      if (cudaMemcpy(B.dst_off.p, B.h_off.data(), (size_t)np * sizeof(long long), cudaMemcpyHostToDevice) != cudaSuccess) return -3;
      cudaEventRecord(B.ev[2]);
      TBM_LAUNCH(tbm::k_gather_matches, grid, 256, 0, B.segs.p, np, B.count.p, B.dst_off.p, B.staged.p, B.packed.p);
      if (cudaPeekAtLastError() != cudaSuccess) return -3;
      cudaEventRecord(B.ev[3]);
      if (cudaMemcpy(matches + *written, B.packed.p, (size_t)total * sizeof(tbm_match), cudaMemcpyDeviceToHost) != cudaSuccess) return -3;
      float ms = 0;
      if (cudaEventElapsedTime(&ms, B.ev[2], B.ev[3]) == cudaSuccess) B.kernel_ms += ms;
    }
  }
  *written += total;
  return 0;
}

// launches the exact pass of the tensor-core path on the current stream
inline int launch_exact_top2(const float* d, const int* q_row, const int* b_row0, const int* b_rows, const int* cand, long long n_q, int* best_j,
                             float* best_d, float* second_d, unsigned long long* n_exhaustive) {
  using namespace tbm_tc;
  if (cudaFuncSetAttribute(k_exact_top2, cudaFuncAttributeMaxDynamicSharedMemorySize, kExactSmemBytes) != cudaSuccess) return -3;
  TBM_LAUNCH(k_exact_top2, (unsigned)((n_q + 31) / 32), 256, kExactSmemBytes, d, q_row, b_row0, b_rows, cand, n_q, best_j, best_d, second_d, n_exhaustive);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -3;
}

// :58-59, :78-81: keep the best match when the ratio test is off, there is no second candidate, or it passes
inline bool passes(const tbm_options* o, float best, float second, int second_valid) {
  if (!o->use_lowes_ratio || !second_valid) return true;
  const float sqf = o->lowes_ratio * o->lowes_ratio;  // FeatureMatcherOptions::lowes_ratio is a float: the product is rounded to float, then widened (:58-59)
  const double sq = (double)sqf;
  return (double)best < sq * (double)second;
}

}  // namespace

extern "C" {

void tbm_options_init(tbm_options* o) { o->keep_only_symmetric_matches = 1; o->use_lowes_ratio = 1; o->lowes_ratio = 0.8f; o->min_num_feature_matches = 30; }

void tbm_debug_last_timing(double* out4) { for (int i = 0; i < 4; ++i) out4[i] = g_last_timing[i]; }

// Test hook: the exact pass of the tensor-core path alone (k_exact_top2) on caller-made candidate lists.  descriptors [n_rows][128];
// query i = row q_row[i] against rows [b_row0[i], b_row0[i] + b_rows[i]); cand [n_q][16] global row indices, -1 = empty slot,
// cand[i][0] or cand[i][8] == -2: exhaustive scan of that query.  Returns 0 or a negative tbm code.
int tbm_debug_exact_top2(int device, const float* descriptors, int64_t n_rows, const int32_t* q_row, const int32_t* b_row0, const int32_t* b_rows,
                         const int32_t* cand, int64_t n_q, int32_t* best_j, float* best_d, float* second_d) {
  if (!descriptors || !q_row || !b_row0 || !b_rows || !cand || !best_j || !best_d || !second_d || n_rows <= 0 || n_q <= 0) return -1;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) { cudaGetLastError(); return -5; }
  if (cudaSetDevice(device) != cudaSuccess) return -3;
  using namespace tbm_tc;
  DevF d_desc, d_bd, d_sd;
  DevI d_q, d_b0, d_bn, d_cand, d_bj;
  if (!d_desc.alloc((size_t)n_rows * DIM) || !d_bd.alloc((size_t)n_q) || !d_sd.alloc((size_t)n_q) || !d_q.alloc((size_t)n_q) || !d_b0.alloc((size_t)n_q) ||
      !d_bn.alloc((size_t)n_q) || !d_cand.alloc((size_t)n_q * KC) || !d_bj.alloc((size_t)n_q)) return -3;
  if (cudaMemcpy(d_desc.p, descriptors, (size_t)n_rows * DIM * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(d_q.p, q_row, (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(d_b0.p, b_row0, (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(d_bn.p, b_rows, (size_t)n_q * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(d_cand.p, cand, (size_t)n_q * KC * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess) return -3;
  if (launch_exact_top2(d_desc.p, d_q.p, d_b0.p, d_bn.p, d_cand.p, (long long)n_q, d_bj.p, d_bd.p, d_sd.p, nullptr) != 0) return -3;
  if (cudaPeekAtLastError() != cudaSuccess) return -3;
  if (cudaMemcpy(best_j, d_bj.p, (size_t)n_q * sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(best_d, d_bd.p, (size_t)n_q * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess ||
      cudaMemcpy(second_d, d_sd.p, (size_t)n_q * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) return -3;
  return 0;
}

int tbm_debug_postprocess(const int32_t* f_best_j, const float* f_best_d, const float* f_second_d, int32_t n1, int f_second_valid,
                          const int32_t* r_best_j, const float* r_best_d, const float* r_second_d, int32_t n2, int r_second_valid,
                          const tbm_options* o, tbm_match* matches, int32_t* n_matches) {
  int n = 0;
  for (int i = 0; i < n1; ++i) {  // forward matches (:63-82)
    if (f_best_j[i] < 0) continue;
    if (passes(o, f_best_d[i], f_second_d[i], f_second_valid)) { matches[n].feature1_ind = i; matches[n].feature2_ind = f_best_j[i]; matches[n].distance = f_best_d[i]; ++n; }
  }
  *n_matches = n;
  if (n < o->min_num_feature_matches) return 0;  // :84-86
  if (o->keep_only_symmetric_matches) {          // :89-113 + IntersectMatches
    int kept = 0;
    for (int k = 0; k < n; ++k) {
      const int i = matches[k].feature1_ind, j = matches[k].feature2_ind;
      const bool rev = j >= 0 && j < n2 && r_best_j[j] == i && passes(o, r_best_d[j], r_second_d[j], r_second_valid);
      if (rev) matches[kept++] = matches[k];
    }
    n = kept;
    *n_matches = n;
  }
  return n >= o->min_num_feature_matches;  // :116
}

#ifndef TBA_EMULATE
// Tensor-core path (dim == 128): all pairs of a chunk in ONE launch of k_nn_candidates + ONE launch of k_exact_top2, one
// device-to-host copy per chunk, then MatchImagePair's ratio test / early exits / IntersectMatches per pair on the host.
static int match_all_tc(const float* descriptors, const int64_t* img_off, int32_t n_img, const int32_t* pairs, int64_t n_pairs,
                        const tbm_options* options, tbm_match* matches, int64_t cap, int64_t* match_off, uint8_t* pair_ok, const Nn2Out* dbg) {
  using namespace tbm_tc;
  const int64_t total = img_off[n_img];
  if (total >= (int64_t)1 << 31) return -1;
  cudaEvent_t ev[6];
  for (auto& e : ev) if (cudaEventCreate(&e) != cudaSuccess) return -3;
  struct EvGuard { cudaEvent_t* e; ~EvGuard() { for (int i = 0; i < 6; ++i) cudaEventDestroy(e[i]); } } ev_guard{ev};
  g_last_timing[0] = g_last_timing[1] = g_last_timing[2] = g_last_timing[3] = 0.0;
  cudaEventRecord(ev[0]);
  int n_sm = 132;
  { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev); }
  DevF d_desc, d_nrm, d_bd, d_sd;
  DevI d_cand, d_bj, d_qrow, d_brow0, d_brows;
  if (!d_bj.alloc(1) || !d_bd.alloc(1) || !d_sd.alloc(1)) return -3;  // (never null: chunks of pairs between empty images)
  if (!d_desc.alloc((size_t)(total > 0 ? total : 1) * DIM) || !d_nrm.alloc((size_t)(total > 0 ? total : 1))) return -3;
  if (total > 0 && cudaMemcpy(d_desc.p, descriptors, (size_t)total * DIM * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return -3;
  cudaEventRecord(ev[1]);
  int any_negative = 0;
  if (total > 0) {
    DevI d_neg;
    if (!d_neg.alloc(1) || cudaMemset(d_neg.p, 0, sizeof(int)) != cudaSuccess) return -3;
    k_row_norms<<<(unsigned)((total + 255) / 256), 256>>>(d_desc.p, total, d_nrm.p, d_neg.p);
    if (cudaPeekAtLastError() != cudaSuccess) return -3;
    if (cudaMemcpy(&any_negative, d_neg.p, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return -3;
  }
  CUtensorMap map;
  if (total > 0 && !make_desc_map(&map, d_desc.p, total)) return -3;
  unsigned long long* d_nex = nullptr;  // queries handed to the exhaustive exact scan (diagnostics: tbm_debug_last_timing)
  if (cudaMalloc(&d_nex, 8) != cudaSuccess || cudaMemset(d_nex, 0, 8) != cudaSuccess) return -3;
  struct NexGuard { unsigned long long* p; ~NexGuard() { cudaFree(p); } } nex_guard{d_nex};
  if (cudaFuncSetAttribute(k_nn_candidates<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(k_nn_candidates<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes) != cudaSuccess) return -3;
  Dev<WorkItem> d_items;
  Dev<tbm::QuerySeg> d_qsegs;
  DecideBuffers dec;
  std::vector<WorkItem> items;
  std::vector<tbm::QuerySeg> qsegs;
  std::vector<tbm::PairSeg> psegs;
  const bool sym = options->keep_only_symmetric_matches != 0;
  int64_t written = 0;
  bool overflow = false;
  const int64_t kChunkQueries = (int64_t)4 << 20;  // queries per chunk (both directions): bounds the device staging
  int64_t q_base = 0;                                // queries of the chunks before this one (tbm_debug_nn2 output offset)
  for (int64_t p0 = 0; p0 < n_pairs;) {
    // ---- chunk [p0, p1): as many pairs as fit the query budget; one (pair, direction) segment table instead of per-query host arrays
    items.clear(); qsegs.clear(); psegs.clear();
    int64_t p1 = p0, qo = 0;
    while (p1 < n_pairs) {
      const int a = pairs[2 * p1], b = pairs[2 * p1 + 1];
      if (a < 0 || a >= n_img || b < 0 || b >= n_img) return -1;
      const int n1 = (int)(img_off[a + 1] - img_off[a]), n2 = (int)(img_off[b + 1] - img_off[b]);
      const int64_t add = (int64_t)n1 + (sym ? n2 : 0);
      if (p1 > p0 && qo + add > kChunkQueries) break;
      tbm::PairSeg ps;
      ps.f0 = qo; ps.r0 = qo + n1; ps.n1 = n1; ps.n2 = n2; ps.n_rev = sym ? n2 : 0;
      psegs.push_back(ps);
      for (int dir = 0; dir < (sym ? 2 : 1); ++dir) {
        const int qa = dir == 0 ? a : b, cb = dir == 0 ? b : a;
        const int nq = dir == 0 ? n1 : n2, nc = dir == 0 ? n2 : n1;
        if (nq > 0) {
          tbm::QuerySeg g;
          g.out0 = qo; g.nq = nq; g.q_row0 = (int)img_off[qa]; g.b_row0 = (int)img_off[cb]; g.b_rows = nc;
          qsegs.push_back(g);
        }
        if (nc > 0)
          for (int m0 = 0; m0 < nq; m0 += BM) {
            WorkItem w;
            w.a_row0 = (int)img_off[qa] + m0; w.a_rows = nq - m0 < BM ? nq - m0 : BM; w.b_row0 = (int)img_off[cb]; w.b_rows = nc; w.out_row0 = qo + m0;
            items.push_back(w);
          }
        qo += nq;
      }
      ++p1;
    }
    const int64_t nq_chunk = qo;
    if (nq_chunk > 0) {
      if (!d_cand.alloc((size_t)nq_chunk * KC) || !d_bj.alloc((size_t)nq_chunk) || !d_bd.alloc((size_t)nq_chunk) || !d_sd.alloc((size_t)nq_chunk) ||
          !d_qrow.alloc((size_t)nq_chunk) || !d_brow0.alloc((size_t)nq_chunk) || !d_brows.alloc((size_t)nq_chunk) || !d_qsegs.alloc(qsegs.size())) return -3;
      if (cudaMemset(d_cand.p, 0xFF, (size_t)nq_chunk * KC * sizeof(int)) != cudaSuccess) return -3;  // -1: no candidate (empty other image)
      if (cudaMemcpy(d_qsegs.p, qsegs.data(), qsegs.size() * sizeof(tbm::QuerySeg), cudaMemcpyHostToDevice) != cudaSuccess) return -3;
      tbm::k_expand_segments<<<(unsigned)(qsegs.size() < 8192 ? qsegs.size() : 8192), 256>>>(d_qsegs.p, (int)qsegs.size(), d_qrow.p, d_brow0.p, d_brows.p);
      if (cudaPeekAtLastError() != cudaSuccess) return -3;
      if (!items.empty()) {
        if (!d_items.alloc(items.size())) return -3;
        if (cudaMemcpy(d_items.p, items.data(), items.size() * sizeof(WorkItem), cudaMemcpyHostToDevice) != cudaSuccess) return -3;
        const int grid = (int)(items.size() < (size_t)n_sm ? items.size() : (size_t)n_sm);
        cudaEventRecord(ev[2]);
        if (any_negative) k_nn_candidates<false><<<grid, THREADS, kSmemBytes>>>(map, d_items.p, (int)items.size(), d_nrm.p, d_cand.p);
        else k_nn_candidates<true><<<grid, THREADS, kSmemBytes>>>(map, d_items.p, (int)items.size(), d_nrm.p, d_cand.p);
        if (cudaPeekAtLastError() != cudaSuccess) return -3;
        cudaEventRecord(ev[3]);
      }
      cudaEventRecord(ev[4]);
      if (launch_exact_top2(d_desc.p, d_qrow.p, d_brow0.p, d_brows.p, d_cand.p, nq_chunk, d_bj.p, d_bd.p, d_sd.p, d_nex) != 0) return -3;
      cudaEventRecord(ev[5]);
      if (dbg) {
        std::vector<int> slot0((size_t)nq_chunk);  // candidate slot 0 of every query: kOverflow = scanned exhaustively
        if (cudaMemcpy(dbg->best_j + q_base, d_bj.p, (size_t)nq_chunk * sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess ||
            cudaMemcpy(dbg->best_d + q_base, d_bd.p, (size_t)nq_chunk * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess ||
            cudaMemcpy(dbg->second_d + q_base, d_sd.p, (size_t)nq_chunk * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess ||
            cudaMemcpy2D(slot0.data(), sizeof(int), d_cand.p, KC * sizeof(int), sizeof(int), (size_t)nq_chunk, cudaMemcpyDeviceToHost) != cudaSuccess) return -3;
        for (int64_t q = 0; q < nq_chunk; ++q) dbg->exhaustive[q_base + q] = slot0[(size_t)q] == kOverflow;
      }
    }
    q_base += nq_chunk;
    // ---- MatchImagePair's decisions per pair, on the device (tbm_decide.cuh); only the kept matches are copied back
    const int rc = decide_and_fetch(dec, psegs, nq_chunk, d_bj.p, d_bd.p, d_sd.p, options, p0, matches, cap, &written, match_off, pair_ok, &overflow);
    if (rc) return rc;
    if (nq_chunk > 0) {
      float ms = 0;
      if (!items.empty() && cudaEventElapsedTime(&ms, ev[2], ev[3]) == cudaSuccess) g_last_timing[0] += ms;
      if (cudaEventElapsedTime(&ms, ev[4], ev[5]) == cudaSuccess) g_last_timing[1] += ms;
    }
    p0 = p1;
  }
  if (cudaDeviceSynchronize() != cudaSuccess) return -3;
  g_last_timing[1] += dec.kernel_ms;  // the decision kernels count as device time of the "exact" stage
  { float ms = 0; if (cudaEventElapsedTime(&ms, ev[0], ev[1]) == cudaSuccess) g_last_timing[2] = ms; }
  { unsigned long long h = 0; if (cudaMemcpy(&h, d_nex, 8, cudaMemcpyDeviceToHost) == cudaSuccess) g_last_timing[3] = (double)h; }
  match_off[n_pairs] = written;
  return overflow ? -1 : 0;
}
#endif

static int match_all(int device, const float* descriptors, const int64_t* img_off, int32_t n_img, int32_t dim, const int32_t* pairs,
                     int64_t n_pairs, const tbm_options* options, tbm_match* matches, int64_t cap, int64_t* match_off, uint8_t* pair_ok,
                     const Nn2Out* dbg) {
  if (!descriptors || !img_off || !pairs || !options || !match_off || !pair_ok || n_img < 0 || dim <= 0 || dim > 512 || n_pairs < 0) return -1;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) { cudaGetLastError(); return -5; }
  if (cudaSetDevice(device) != cudaSuccess) return -3;
#ifndef TBA_EMULATE
  {
    // dim 128 (SIFT): the tensor-core path.  TBM_PATH=exact forces the CUDA-core kernel (the bit-exact checker of round 1).
    const char* e = getenv("TBM_PATH");
    for (int i = 0; i < n_img; ++i) if (img_off[i + 1] < img_off[i]) return -1;
    if (dim == tbm_tc::DIM && !(e != nullptr && e[0] == 'e')) return match_all_tc(descriptors, img_off, n_img, pairs, n_pairs, options, matches, cap, match_off, pair_ok, dbg);
  }
#endif
  const int64_t total = img_off[n_img];
  int64_t max_n = 0;
  for (int i = 0; i < n_img; ++i) { if (img_off[i + 1] < img_off[i]) return -1; max_n = img_off[i + 1] - img_off[i] > max_n ? img_off[i + 1] - img_off[i] : max_n; }
  DevF d_desc, d_bd, d_sd;
  DevI d_bj;  // results of one pair: forward queries [0, n1), reverse queries [n1, n1 + n2)
  if (!d_desc.alloc((size_t)total * dim)) return -3;
  if (!d_bd.alloc((size_t)max_n * 2) || !d_sd.alloc((size_t)max_n * 2) || !d_bj.alloc((size_t)max_n * 2)) return -3;
  if (cudaMemcpy(d_desc.p, descriptors, (size_t)total * dim * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return -3;
  const size_t smem = ((size_t)ROWS * (dim + 1) + (size_t)TJ * dim) * sizeof(float);
  // the 48 KB a launch may use without the attribute include k_nn2's static s_merge (4 KB): dims 176..191 need it as well
  if (cudaFuncSetAttribute(k_nn2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return -3;
  DecideBuffers dec;
  std::vector<tbm::PairSeg> one(1);
  int64_t written = 0;
  bool overflow = false;
  const bool sym = options->keep_only_symmetric_matches != 0;
  int64_t q_base = 0;  // tbm_debug_nn2 output offset of the current pair
  for (int64_t p = 0; p < n_pairs; ++p) {
    const int a = pairs[2 * p], b = pairs[2 * p + 1];
    if (a < 0 || a >= n_img || b < 0 || b >= n_img) return -1;
    const int n1 = (int)(img_off[a + 1] - img_off[a]), n2 = (int)(img_off[b + 1] - img_off[b]);
    const float* A = d_desc.p + (size_t)img_off[a] * dim;
    const float* B = d_desc.p + (size_t)img_off[b] * dim;
    if (n1 + n2 > 0 && cudaMemset(d_bj.p, 0xFF, (size_t)(n1 + n2) * sizeof(int)) != cudaSuccess) return -3;  // -1: no match (empty other image)
    if (dbg && n1 + n2 > 0 && (cudaMemset(d_bd.p, 0, (size_t)(n1 + n2) * sizeof(float)) != cudaSuccess ||
                               cudaMemset(d_sd.p, 0, (size_t)(n1 + n2) * sizeof(float)) != cudaSuccess)) return -3;
    for (int dir = 0; dir < (sym ? 2 : 1); ++dir) {
      const int nq = dir == 0 ? n1 : n2, nc = dir == 0 ? n2 : n1;
      if (nq == 0 || nc == 0) continue;
      const size_t o = dir == 0 ? 0 : (size_t)n1;
      TBM_LAUNCH(k_nn2, (nq + ROWS - 1) / ROWS, ROWS * SLICES, smem, dir == 0 ? A : B, nq, dir == 0 ? B : A, nc, dim, d_bj.p + o, d_bd.p + o, d_sd.p + o);
      if (cudaPeekAtLastError() != cudaSuccess) return -3;
    }
    one[0].f0 = 0; one[0].r0 = n1; one[0].n1 = n1; one[0].n2 = n2; one[0].n_rev = sym ? n2 : 0;
    const int rc = decide_and_fetch(dec, one, (long long)n1 + n2, d_bj.p, d_bd.p, d_sd.p, options, p, matches, cap, &written, match_off, pair_ok, &overflow);
    if (rc) return rc;
    if (dbg) {
      const size_t nq = (size_t)n1 + (sym ? (size_t)n2 : 0);
      if (nq > 0 && (cudaMemcpy(dbg->best_j + q_base, d_bj.p, nq * sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess ||
                     cudaMemcpy(dbg->best_d + q_base, d_bd.p, nq * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess ||
                     cudaMemcpy(dbg->second_d + q_base, d_sd.p, nq * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess)) return -3;
      q_base += (int64_t)nq;
    }
  }
  match_off[n_pairs] = written;
  return overflow ? -1 : 0;
}

int tbm_match_all(int device, const float* descriptors, const int64_t* img_off, int32_t n_img, int32_t dim, const int32_t* pairs,
                  int64_t n_pairs, const tbm_options* options, tbm_match* matches, int64_t cap, int64_t* match_off, uint8_t* pair_ok) {
  return match_all(device, descriptors, img_off, n_img, dim, pairs, n_pairs, options, matches, cap, match_off, pair_ok, nullptr);
}

int tbm_debug_nn2(int device, const float* descriptors, const int64_t* img_off, int32_t n_img, int32_t dim, const int32_t* pairs,
                  int64_t n_pairs, int symmetric, int32_t* best_j, float* best_d, float* second_d, uint8_t* exhaustive) {
  if (!img_off || !pairs || !best_j || !best_d || !second_d || !exhaustive || n_img < 0 || n_pairs < 0) return -1;
  for (int i = 0; i < n_img; ++i) if (img_off[i + 1] < img_off[i]) return -1;
  int64_t nq = 0;
  for (int64_t p = 0; p < n_pairs; ++p) {
    const int a = pairs[2 * p], b = pairs[2 * p + 1];
    if (a < 0 || a >= n_img || b < 0 || b >= n_img) return -1;
    nq += (img_off[a + 1] - img_off[a]) + (symmetric ? img_off[b + 1] - img_off[b] : 0);
  }
  std::memset(exhaustive, 0, (size_t)nq);
  // every forward query may keep its match: no ratio test, no early exit -- the decisions are not what this hook reports
  tbm_options o;
  tbm_options_init(&o);
  o.keep_only_symmetric_matches = symmetric != 0; o.use_lowes_ratio = 0; o.min_num_feature_matches = 0;
  std::vector<tbm_match> m((size_t)nq + 1);
  std::vector<int64_t> off((size_t)n_pairs + 1);
  std::vector<uint8_t> ok((size_t)n_pairs + 1);
  const Nn2Out out{best_j, best_d, second_d, exhaustive};
  return match_all(device, descriptors, img_off, n_img, dim, pairs, n_pairs, &o, m.data(), nq + 1, off.data(), ok.data(), &out);
}

}  // extern "C"
