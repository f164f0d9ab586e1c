// tba_pack.h -- host-side packing of a flattened BA problem into the engine's tile layout (DESIGN.md section 4).
// Pure host code (no CUDA): used by tba_upload() and, for CPU-only tests of the host logic, by tba_debug_pack().
//
// Layout rules: observations sorted by point, (intrinsics group, camera, index) order inside a point; tiles of TILE
// slots = 8 warp slices of 32; in a normal tile a point never straddles a warp slice; tracks with more than 32
// observations go to "long" tiles (packed after all normal points); at most MAXP points per tile; padding slots have
// cam = -1.  Which parameter blocks take part follows bundle_adjuster.cc:102-180 as recorded by the adapter in
// ext_const / group_const_mask / pt_const, plus "blocks without residuals are not in the program".
#pragma once
#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include <unistd.h>

#include "../../include/theia_ba_b200.h"

namespace tba {

constexpr int kPackTile = 256;
constexpr int kPackMaxPoints = 256;

// ---- worker pool of the host pack.  Creating and joining 64 threads costs 1 - 2 ms per parallel loop, and an upload runs about
// twenty of them (eight for the chunked fill alone): a quarter of the upload time of a 20 M-observation problem was thread creation.
// One process-wide pool of detached workers (grown on demand, never destroyed: the process exit ends them), one job at a time; a
// caller that finds the pool busy (the rank threads of tba_solve_multi pack concurrently) or that IS a worker falls back to plain
// std::thread's.  After a fork() the child starts a fresh pool (the parent's workers do not exist there).
class PackPool {
 public:
  // runs task(0 .. n_tasks-1), the caller included, and returns when all are done; false = pool busy, nothing was run
  template <class Task>
  bool try_run(int n_tasks, Task&& task) {
    PackPool* p = instance();
    if (p == nullptr) return false;
    return p->run_impl(n_tasks, std::function<void(int)>(std::forward<Task>(task)));
  }
  static PackPool& get() { static PackPool front; return front; }  // (stateless front end; the state lives in instance())

 private:
  struct Job {
    std::function<void(int)> fn;
    int n = 0;
    std::atomic<int> next{0}, remaining{0};
  };
  std::mutex job_mu_;                  // one job at a time (try_lock by callers)
  std::mutex m_;                       // guards current_ / gen_ / n_workers_
  std::condition_variable cv_work_, cv_done_;
  std::shared_ptr<Job> current_;
  unsigned long long gen_ = 0;
  int n_workers_ = 0;
  long long pid_ = 0;
  static constexpr int kMaxWorkers = 255;

  static PackPool* instance() {
    static std::mutex im;
    static PackPool* inst = nullptr;
    std::lock_guard<std::mutex> lk(im);
    const long long pid = (long long)getpid();
    if (inst == nullptr || inst->pid_ != pid) { inst = new PackPool(); inst->pid_ = pid; }  // (a forked child leaks the parent's object on purpose)
    return inst;
  }
  static bool& is_worker() { static thread_local bool w = false; return w; }

  void worker_loop() {
    is_worker() = true;
    unsigned long long seen = 0;
    for (;;) {
      std::shared_ptr<Job> job;
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_work_.wait(lk, [&] { return gen_ != seen; });
        seen = gen_;
        job = current_;
      }
      if (job) drain(*job);
    }
  }
  void drain(Job& job) {
    for (;;) {
      const int i = job.next.fetch_add(1, std::memory_order_relaxed);
      if (i >= job.n) return;
      job.fn(i);
      if (job.remaining.fetch_sub(1, std::memory_order_acq_rel) == 1) {
        std::lock_guard<std::mutex> lk(m_);
        cv_done_.notify_all();
      }
    }
  }
  bool run_impl(int n_tasks, std::function<void(int)> fn) {
    if (n_tasks <= 0) return true;
    if (is_worker()) return false;                 // nested use: the caller runs its loop with its own threads
    std::unique_lock<std::mutex> job_lk(job_mu_, std::try_to_lock);
    if (!job_lk.owns_lock()) return false;
    auto job = std::make_shared<Job>();
    job->fn = std::move(fn); job->n = n_tasks; job->remaining.store(n_tasks);
    {
      std::lock_guard<std::mutex> lk(m_);
      const int want = std::min(kMaxWorkers, n_tasks - 1);
      while (n_workers_ < want) { std::thread([this] { worker_loop(); }).detach(); ++n_workers_; }
      current_ = job;
      ++gen_;
    }
    cv_work_.notify_all();
    drain(*job);
    {
      std::unique_lock<std::mutex> lk(m_);
      cv_done_.wait(lk, [&] { return job->remaining.load(std::memory_order_acquire) == 0; });
      current_.reset();
    }
    return true;
  }
};

// grain: least number of items worth a thread of its own (8192 for per-observation loops; per-tile loops pass a small one)
template <class F>
void parallel_for(int64_t n, int nthreads, F f, int64_t grain = 8192) {
  if (n <= 0) return;
  const int T = (int)std::min<int64_t>(nthreads, (n + grain - 1) / grain);
  if (T <= 1) { f((int64_t)0, n, 0); return; }
  const int64_t chunk = (n + T - 1) / T;
  auto task = [&](int t) {
    const int64_t b = t * chunk, e = std::min(n, b + chunk);
    if (b < e) f(b, e, t);
  };
  static const bool use_pool = getenv("TBA_PACK_POOL") == nullptr || getenv("TBA_PACK_POOL")[0] != '0';  // TBA_PACK_POOL=0: threads per loop
  if (use_pool && PackPool::get().try_run(T, task)) return;
  std::vector<std::thread> th;
  for (int t = 0; t < T; ++t) {
    if ((int64_t)t * chunk >= n) break;
    th.emplace_back([=, &task] { task(t); });
  }
  for (auto& x : th) x.join();
}

struct HostPack {  // lives in the engine context: the vectors keep their capacity (and their faulted-in pages) across uploads
  // phases A-C
  std::vector<int> cnt_pt, cnt_cam;
  std::vector<int> cam_hist;       // per-thread camera histograms of phase A
  std::vector<int64_t> cursor;     // per-point write cursors of phase C
  std::vector<int64_t> off, order;
  std::vector<uint16_t> pt_nruns;  // (point, group) runs per point: up to the track length, 256
  // scattered input (observations not grouped by point, e.g. the adapter's per-view flattening): two-level counting sort
  std::vector<int64_t> tmp_idx;    // observation indices grouped by point bucket (stable)
  std::vector<int> tmp_q, tmp_cam; // their point / camera
  std::vector<int> ocam;           // camera of order[k] (point-sorted copy: the per-point sort and the fill read it sequentially)
  std::vector<int64_t> bucket_cnt; // [thread][bucket] counts -> write offsets
  bool have_ocam = false;
  int maxlen = 0;
  int64_t bad = -1;
  // packed points
  std::vector<int> pk2caller;
  int n_long = 0;
  int64_t n_free_pt = 0, n_free_cs = 0;
  // masks + tiles
  std::vector<double> mask, blk_free;
  uint32_t union_free = 0;
  std::vector<int> tile_pt_begin, tile_nruns;
  std::vector<uint8_t> tile_flags;
  std::vector<int64_t> pt_slot;  // first slot of each packed point
  std::vector<int> pt_runbase;   // run index (inside its tile) of the point's first run
  int n_tiles = 0;
  int64_t n_slots = 0;
};

struct PackDest {
  double* xy;        // [tile][warp][2][32]
  double* pt;        // [packed point][4]
  int* slot_cam;     // -1 = padding
  int* slot_pt;      // packed point id
  int16_t* slot_run;
  uint8_t* slot_flags;
  uint8_t* pt_const;  // [packed point]
  int64_t* slot_orig; // optional (nullptr: not wanted); pre-filled with -1
};

// A: validate + per-point / per-camera counts; B: offsets; C: observations grouped by point and sorted inside a point.
// Written for both input orders that occur: grouped by point (synthetic scenes, BAL-style files) and grouped by view (the
// adapter's flattening, bundle_adjuster.cc:125-134): per-thread camera histograms instead of contended atomics, one
// atomic per RUN of equal point indices instead of one per observation, and the per-point sort works on locally
// gathered (group, camera) keys and is skipped when the run is already in order.
inline void pack_count_and_sort(const tba_problem* p, int T, HostPack* H) {
  const int nc = p->n_cam, np = p->n_pt;
  const int64_t no = p->n_obs;
  T = std::max(1, T);
  const bool trace = getenv("TBA_PACK_TRACE") != nullptr;  // sub-phase wall clock on stderr
  auto t_prev = std::chrono::steady_clock::now();
  auto lap = [&](const char* what) {
    if (!trace) return;
    const auto t = std::chrono::steady_clock::now();
    fprintf(stderr, "[pack A-C] %-22s %8.2f ms\n", what, std::chrono::duration<double, std::milli>(t - t_prev).count());
    t_prev = t;
  };
  H->cnt_pt.assign((size_t)np, 0);
  H->cnt_cam.assign((size_t)nc, 0);
  const bool use_hist = (int64_t)nc * T <= ((int64_t)1 << 24);
  if (use_hist) H->cam_hist.assign((size_t)nc * T, 0);
  std::atomic<int64_t> bad(-1);
  int* cnt_pt = H->cnt_pt.data();
  int* cnt_cam = H->cnt_cam.data();
  H->have_ocam = false;
  // ---- is the input grouped by point?  (look at the first million observations: a new point on more than a quarter of them = scattered)
  bool scattered = false;
  {
    const int64_t ns = std::min<int64_t>(no, 1 << 20);
    int64_t breaks = 0;
    for (int64_t i = 1; i < ns; ++i) breaks += p->obs_pt[i] != p->obs_pt[i - 1];
    scattered = ns >= 4096 && breaks * 4 > ns && np >= 4096;
  }
  if (scattered) {
    // Two-level counting sort without contended atomics (the run-based path below does one atomic per RUN of equal points: with
    // scattered input that is one random atomic + one random 8-byte store per observation -- 360 ms instead of 8 for 20 M observations):
    //   1. observations -> point buckets of 2^shift points (<= 256 buckets), per-thread bucket counts, then a stable scatter of
    //      (index, point, camera) into bucket-grouped temporaries (sequential streams per (thread, bucket));
    //   2. per bucket (its points' counters and its slice of `order` are cache-resident): counts, offsets, stable scatter into
    //      order / ocam.  Same `order` contents per point as the run path up to the order INSIDE a point, which phase C fixes.
    int shift = 0;
    while (((int64_t)(np - 1) >> shift) >= 256) ++shift;
    const int B = (int)(((int64_t)np - 1) >> shift) + 1;
    H->bucket_cnt.assign((size_t)(T + 1) * B, 0);
    int64_t* bc = H->bucket_cnt.data();
    // the chunks of the two passes must be identical: fixed here, independent of parallel_for's grain
    const int64_t chunk = (no + T - 1) / T;
    parallel_for(T, T, [&](int64_t t0, int64_t t1, int) {
      for (int64_t t = t0; t < t1; ++t) {
        int* hist = use_hist ? H->cam_hist.data() + (size_t)t * nc : nullptr;
        int64_t* mine = bc + (size_t)t * B;
        const int64_t b0 = t * chunk, e0 = std::min(no, b0 + chunk);
        for (int64_t i = b0; i < e0; ++i) {
          const int q = p->obs_pt[i], cam = p->obs_cam[i];
          if (q < 0 || q >= np || cam < 0 || cam >= nc) { bad.store(i); return; }
          if (hist) ++hist[cam]; else __atomic_fetch_add(&cnt_cam[cam], 1, __ATOMIC_RELAXED);
          ++mine[q >> shift];
        }
      }
    }, 1);
    H->bad = bad.load();
    lap("A count (buckets)");
    if (H->bad >= 0) return;
    if (use_hist)
      parallel_for(nc, T, [&](int64_t b0, int64_t e0, int) {
        for (int t = 0; t < T; ++t) {
          const int* hist = H->cam_hist.data() + (size_t)t * nc;
          for (int64_t i = b0; i < e0; ++i) cnt_cam[i] += hist[i];
        }
      });
    // write offsets: bucket-major, thread-minor (stable); row T = bucket begins
    std::vector<int64_t> bucket_begin((size_t)B + 1, 0);
    {
      int64_t run = 0;
      for (int b = 0; b < B; ++b) {
        bucket_begin[b] = run;
        for (int t = 0; t < T; ++t) { const int64_t c = bc[(size_t)t * B + b]; bc[(size_t)t * B + b] = run; run += c; }
      }
      bucket_begin[B] = run;
    }
    H->tmp_idx.resize((size_t)no); H->tmp_q.resize((size_t)no); H->tmp_cam.resize((size_t)no);
    parallel_for(T, T, [&](int64_t t0, int64_t t1, int) {
      for (int64_t t = t0; t < t1; ++t) {
        int64_t* mine = bc + (size_t)t * B;
        const int64_t b0 = t * chunk, e0 = std::min(no, b0 + chunk);
        for (int64_t i = b0; i < e0; ++i) {
          const int q = p->obs_pt[i];
          const int64_t dst = mine[q >> shift]++;
          H->tmp_idx[(size_t)dst] = i; H->tmp_q[(size_t)dst] = q; H->tmp_cam[(size_t)dst] = p->obs_cam[i];
        }
      }
    }, 1);
    lap("B1 bucket scatter");
    H->off.assign((size_t)np + 1, 0);
    H->order.resize((size_t)no);
    H->ocam.resize((size_t)no);
    std::atomic<int> maxlen(0);
    parallel_for(B, T, [&](int64_t bb0, int64_t bb1, int) {
      std::vector<int64_t> cur((size_t)1 << shift);
      int local_max = 0;
      for (int64_t b = bb0; b < bb1; ++b) {
        const int q0 = (int)(b << shift), q1 = (int)std::min<int64_t>(np, (b + 1) << shift);
        const int64_t s0 = bucket_begin[b], s1 = bucket_begin[b + 1];
        for (int64_t k = s0; k < s1; ++k) ++cnt_pt[H->tmp_q[(size_t)k]];
        int64_t run = s0;
        for (int q = q0; q < q1; ++q) { H->off[q] = run; cur[(size_t)(q - q0)] = run; run += cnt_pt[q]; local_max = std::max(local_max, cnt_pt[q]); }
        for (int64_t k = s0; k < s1; ++k) {
          const int64_t dst = cur[(size_t)(H->tmp_q[(size_t)k] - q0)]++;
          H->order[(size_t)dst] = H->tmp_idx[(size_t)k];
          H->ocam[(size_t)dst] = H->tmp_cam[(size_t)k];
        }
      }
      int seen = maxlen.load();
      while (local_max > seen && !maxlen.compare_exchange_weak(seen, local_max)) {}
    }, 1);
    H->off[(size_t)np] = no;
    H->maxlen = maxlen.load();
    H->have_ocam = true;
    lap("B2 per-bucket sort");
    if (H->maxlen > kPackTile) return;
  } else {
  parallel_for(no, T, [&](int64_t b0, int64_t e0, int t) {
    int* hist = use_hist ? H->cam_hist.data() + (size_t)t * nc : nullptr;
    int cur = -1, run = 0;
    for (int64_t i = b0; i < e0; ++i) {
      const int q = p->obs_pt[i], cam = p->obs_cam[i];
      if (q < 0 || q >= np || cam < 0 || cam >= nc) { bad.store(i); return; }
      if (hist) ++hist[cam]; else __atomic_fetch_add(&cnt_cam[cam], 1, __ATOMIC_RELAXED);
      if (q == cur) { ++run; continue; }
      if (run) __atomic_fetch_add(&cnt_pt[cur], run, __ATOMIC_RELAXED);
      cur = q; run = 1;
    }
    if (run) __atomic_fetch_add(&cnt_pt[cur], run, __ATOMIC_RELAXED);
  });
  H->bad = bad.load();
  lap("A count");
  if (H->bad >= 0) return;
  if (use_hist)
    parallel_for(nc, T, [&](int64_t b0, int64_t e0, int) {
      for (int t = 0; t < T; ++t) {
        const int* hist = H->cam_hist.data() + (size_t)t * nc;
        for (int64_t i = b0; i < e0; ++i) cnt_cam[i] += hist[i];
      }
    });
  H->off.resize((size_t)np + 1);
  H->maxlen = 0;
  {
    // exclusive prefix sum of the per-point counts in two parallel passes (chunk sums, then the chunks with their bases)
    const int PC = std::max(1, std::min(T, (np + 65535) / 65536));
    const int64_t pchunk = ((int64_t)np + PC - 1) / PC;
    std::vector<int64_t> csum((size_t)PC + 1, 0);
    std::vector<int> cmax((size_t)PC, 0);
    parallel_for(PC, PC, [&](int64_t c0, int64_t c1, int) {
      for (int64_t c = c0; c < c1; ++c) {
        int64_t sum = 0; int mx = 0;
        for (int64_t q = c * pchunk, e = std::min<int64_t>(np, q + pchunk); q < e; ++q) { sum += cnt_pt[q]; mx = std::max(mx, cnt_pt[q]); }
        csum[(size_t)c + 1] = sum; cmax[(size_t)c] = mx;
      }
    }, 1);
    for (int c = 0; c < PC; ++c) { csum[(size_t)c + 1] += csum[c]; H->maxlen = std::max(H->maxlen, cmax[c]); }
    parallel_for(PC, PC, [&](int64_t c0, int64_t c1, int) {
      for (int64_t c = c0; c < c1; ++c) {
        int64_t run = csum[(size_t)c];
        for (int64_t q = c * pchunk, e = std::min<int64_t>(np, q + pchunk); q < e; ++q) { H->off[(size_t)q] = run; run += cnt_pt[q]; }
      }
    }, 1);
    H->off[(size_t)np] = csum[(size_t)PC];
  }
  lap("hist merge + prefix");
  if (H->maxlen > kPackTile) return;
  H->order.resize((size_t)no);
  H->cursor.assign(H->off.begin(), H->off.end() - 1);
  {
    int64_t* cur = H->cursor.data();
    int64_t* order = H->order.data();
    parallel_for(no, T, [&](int64_t b0, int64_t e0, int) {
      int64_t i = b0;
      while (i < e0) {
        const int q = p->obs_pt[i];
        int64_t j = i + 1;
        while (j < e0 && p->obs_pt[j] == q) ++j;
        int64_t dst = __atomic_fetch_add(&cur[q], j - i, __ATOMIC_RELAXED);
        for (; i < j; ++i) order[(size_t)dst++] = i;
      }
    });
  }
  lap("B scatter (order)");
  }  // grouped input
  H->pt_nruns.assign((size_t)np, 0);
  parallel_for(np, T, [&](int64_t b0, int64_t e0, int) {
    uint64_t key[kPackTile];
    for (int64_t q = b0; q < e0; ++q) {
      int64_t* o = H->order.data() + H->off[q];
      int* oc = H->have_ocam ? H->ocam.data() + H->off[q] : nullptr;
      const int n = (int)(H->off[(size_t)q + 1] - H->off[q]);
      if (n == 0) continue;
      // key = (intrinsics group, camera); ties (a camera observing the point twice) fall back to the observation index
      bool sorted = true;
      for (int j = 0; j < n; ++j) {
        const int cam = oc ? oc[j] : p->obs_cam[o[j]];
        key[j] = ((uint64_t)(uint32_t)p->cam_group[cam] << 32) | (uint32_t)cam;
        if (j > 0 && (key[j] < key[j - 1] || (key[j] == key[j - 1] && o[j] < o[j - 1]))) sorted = false;
      }
      if (!sorted) {  // insertion sort: n <= 256, almost always <= 32
        for (int j = 1; j < n; ++j) {
          const uint64_t kj = key[j];
          const int64_t oj = o[j];
          int m = j - 1;
          while (m >= 0 && (key[m] > kj || (key[m] == kj && o[m] > oj))) { key[m + 1] = key[m]; o[m + 1] = o[m]; --m; }
          key[m + 1] = kj; o[m + 1] = oj;
        }
        if (oc) for (int j = 0; j < n; ++j) oc[j] = (int)(uint32_t)key[j];  // the camera is the low half of the key
      }
      int runs = 1;
      for (int j = 1; j < n; ++j) runs += (key[j] >> 32) != (key[j - 1] >> 32);
      H->pt_nruns[q] = (uint16_t)runs;
    }
  });
  lap("C per-point sort");
}

// Packed points = points that have observations (zero-observation points are left untouched): first the points whose
// track fits one warp slice (<= 32 observations) in caller order, then the long tracks.
inline void pack_points(const tba_problem* p, HostPack* H) {
  const int np = p->n_pt;
  // two parallel passes over fixed chunks of points: count (short, long, free) per chunk, then write at the chunk's offsets
  const int T = std::max(1, std::min<int>(16, (int)std::thread::hardware_concurrency()));
  const int PC = std::max(1, std::min(T, (np + 65535) / 65536));
  const int64_t pchunk = ((int64_t)np + PC - 1) / PC;
  std::vector<int64_t> n_short((size_t)PC + 1, 0), n_lng((size_t)PC + 1, 0), n_free((size_t)PC, 0);
  parallel_for(PC, PC, [&](int64_t c0, int64_t c1, int) {
    for (int64_t c = c0; c < c1; ++c) {
      int64_t a = 0, b = 0, f = 0;
      for (int64_t q = c * pchunk, e = std::min<int64_t>(np, q + pchunk); q < e; ++q) {
        const int n = H->cnt_pt[q];
        if (n == 0) continue;
        if (n <= 32) ++a; else ++b;
        f += p->pt_const[q] ? 0 : 1;
      }
      n_short[(size_t)c + 1] = a; n_lng[(size_t)c + 1] = b; n_free[(size_t)c] = f;
    }
  }, 1);
  H->n_free_pt = 0;
  for (int c = 0; c < PC; ++c) { n_short[(size_t)c + 1] += n_short[c]; n_lng[(size_t)c + 1] += n_lng[c]; H->n_free_pt += n_free[c]; }
  const int64_t total_short = n_short[(size_t)PC];
  H->n_long = (int)n_lng[(size_t)PC];
  H->pk2caller.resize((size_t)(total_short + H->n_long));
  parallel_for(PC, PC, [&](int64_t c0, int64_t c1, int) {
    for (int64_t c = c0; c < c1; ++c) {
      int64_t a = n_short[(size_t)c], b = total_short + n_lng[(size_t)c];
      for (int64_t q = c * pchunk, e = std::min<int64_t>(np, q + pchunk); q < e; ++q) {
        const int n = H->cnt_pt[q];
        if (n == 0) continue;
        if (n <= 32) H->pk2caller[(size_t)a++] = (int)q; else H->pk2caller[(size_t)b++] = (int)q;
      }
    }
  }, 1);
}

// Free-coordinate masks (cnt_c / cnt_g are the GLOBAL observation counts per camera / group) and phase D: tiles.
inline void pack_masks_and_tiles(const tba_problem* p, const std::vector<double>& cnt_c, const std::vector<double>& cnt_g, HostPack* H) {
  const int nc = p->n_cam, ng = p->n_group;
  const int ne = nc * 6, ncs = ne + ng * 10;
  H->mask.assign((size_t)ncs, 0.0);
  H->blk_free.assign((size_t)nc + ng, 0.0);
  H->union_free = 0;
  H->n_free_cs = 0;
  for (int i = 0; i < nc; ++i) {
    if (cnt_c[i] == 0.0) continue;
    for (int j = 0; j < 6; ++j) {
      const bool fr = j < 3 ? !(p->ext_const[i] & TBA_EXT_POSITION_CONST) : !(p->ext_const[i] & TBA_EXT_ORIENTATION_CONST);
      if (fr) { H->mask[(size_t)i * 6 + j] = 1.0; H->blk_free[i] = 1.0; H->n_free_cs++; }
    }
  }
  for (int g = 0; g < ng; ++g) {
    if (cnt_g[g] == 0.0) continue;
    const int K = TBA_MODEL_NUM_PARAMETERS(p->group_model[g]);
    for (int j = 0; j < K; ++j)
      if (!((p->group_const_mask[g] >> j) & 1u)) { H->mask[(size_t)ne + g * 10 + j] = 1.0; H->blk_free[(size_t)nc + g] = 1.0; H->union_free |= 1u << j; H->n_free_cs++; }
  }
  const int npk = (int)H->pk2caller.size();
  H->tile_pt_begin.clear(); H->tile_nruns.clear(); H->tile_flags.clear();
  H->pt_slot.resize((size_t)npk);      // (every entry is written below: no zero fill of 24 MB per upload)
  H->pt_runbase.resize((size_t)npk);
  {
    int used = kPackTile, npts_in_tile = kPackMaxPoints, run = 0;
    bool in_long = false;
    for (int k = 0; k < npk; ++k) {
      const int q = H->pk2caller[k];
      const int len = H->cnt_pt[q];
      const bool is_long = len > 32;
      int start = used;
      if (!is_long && (start % 32) + len > 32) start = (start / 32 + 1) * 32;  // next warp slice
      if (start + len > kPackTile || npts_in_tile + 1 > kPackMaxPoints || is_long != in_long) {
        if (!H->tile_pt_begin.empty()) H->tile_nruns.push_back(run);
        H->tile_pt_begin.push_back(k);
        H->tile_flags.push_back(is_long ? 1 : 0);
        in_long = is_long;
        start = 0; npts_in_tile = 0; run = 0;
      }
      H->pt_slot[k] = (int64_t)(H->tile_pt_begin.size() - 1) * kPackTile + start;
      H->pt_runbase[k] = run;
      run += H->pt_nruns[q];
      used = start + len;
      npts_in_tile++;
    }
    if (!H->tile_pt_begin.empty()) H->tile_nruns.push_back(run);
  }
  H->n_tiles = (int)H->tile_pt_begin.size();
  H->tile_pt_begin.push_back(npk);
  H->n_slots = (int64_t)H->n_tiles * kPackTile;
}

// slot -> caller observation index (-1 for padding), derived from the grouped order: what the debug read-back of
// per-observation quantities and the CPU tests need; not part of the upload.
inline void pack_slot_orig(const HostPack& H, int T, int64_t* slot_orig) {
  parallel_for(H.n_slots, T, [&](int64_t b0, int64_t e0, int) { for (int64_t s = b0; s < e0; ++s) slot_orig[s] = -1; });
  const int npk = (int)H.pk2caller.size();
  parallel_for(npk, T, [&](int64_t b0, int64_t e0, int) {
    for (int64_t k = b0; k < e0; ++k) {
      const int q = H.pk2caller[k];
      int64_t s0 = H.pt_slot[k];
      for (int64_t kk = H.off[q]; kk < H.off[(size_t)q + 1]; ++kk, ++s0) slot_orig[s0] = H.order[kk];
    }
  });
}

// E: fill the slot arrays, parallel over tiles (each tile is cleared and filled while it is in cache).
// tile_begin / tile_end: fill only that range of tiles (the upload fills and copies chunk by chunk so that the host-to-device
// copy of one chunk overlaps the filling of the next); default: everything.
inline void pack_fill(const tba_problem* p, const HostPack& H, int T, const PackDest& d, int64_t tile_begin = 0, int64_t tile_end = -1) {
  const int nc = p->n_cam;
  if (tile_end < 0) tile_end = H.n_tiles;
  parallel_for(tile_end - tile_begin, T, [&](int64_t r0, int64_t r1, int) {
    const int64_t t0 = tile_begin + r0, t1 = tile_begin + r1;
    for (int64_t t = t0; t < t1; ++t) {
      const int64_t sb = t * kPackTile;
      memset(d.slot_cam + sb, 0xFF, (size_t)kPackTile * 4);
      memset(d.slot_pt + sb, 0, (size_t)kPackTile * 4);
      memset(d.slot_run + sb, 0xFF, (size_t)kPackTile * 2);
      memset(d.slot_flags + sb, 0, (size_t)kPackTile);
      memset(d.xy + sb * 2, 0, (size_t)kPackTile * 16);
      for (int k = H.tile_pt_begin[t]; k < H.tile_pt_begin[t + 1]; ++k) {
        const int q = H.pk2caller[k];
        const bool ptc = p->pt_const[q] != 0;
        d.pt_const[k] = ptc ? 1 : 0;
        memcpy(d.pt + (size_t)k * 4, p->pt + (size_t)q * 4, 32);
        int64_t s0 = H.pt_slot[k];
        int run = H.pt_runbase[k] - 1, last_grp = -1;
        for (int64_t kk = H.off[q]; kk < H.off[(size_t)q + 1]; ++kk, ++s0) {
          const int64_t oi = H.order[kk];
          if (H.have_ocam && kk + 16 < (int64_t)H.order.size()) __builtin_prefetch(p->obs_xy + 2 * H.order[(size_t)kk + 16]);  // scattered input: random 16-byte gathers
          const int cam = H.have_ocam ? H.ocam[(size_t)kk] : p->obs_cam[oi], g = p->cam_group[cam];
          if (g != last_grp) { ++run; last_grp = g; }
          d.slot_cam[s0] = cam; d.slot_pt[s0] = k; d.slot_run[s0] = (int16_t)run;
          const bool any_free = H.blk_free[cam] != 0.0 || H.blk_free[(size_t)nc + g] != 0.0 || !ptc;
          d.slot_flags[s0] = any_free ? 0 : 1;
          const int64_t wq = s0 / 32, l = s0 % 32;  // [tile][warp][2][32]
          d.xy[(size_t)(wq * 2 + 0) * 32 + l] = p->obs_xy[2 * oi];
          d.xy[(size_t)(wq * 2 + 1) * 32 + l] = p->obs_xy[2 * oi + 1];
        }
      }
    }
  }, /*grain: tiles*/ 32);
  if (d.slot_orig && tile_begin == 0 && tile_end == H.n_tiles) pack_slot_orig(H, T, d.slot_orig);
}

}  // namespace tba
