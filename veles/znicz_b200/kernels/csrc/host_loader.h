// Host-side minibatch assembly for streaming loaders (dataset in host memory).
//
//   gather_rows()      rows by index -> a (pinned) staging buffer, fp32 -> bf16 on the fly, or
//                      raw bytes as they are (uint8 ImageNet samples, augmented on the device)
//   HostPrefetcher     a small persistent worker pool that assembles the NEXT minibatch into the
//                      next pinned slot while the current step is being enqueued / executed, so
//                      the training loop never waits for the 0.6-1.2 MB gather (the reference's
//                      loaders fill the minibatch with a python loop inside the step)
//
// No torch headers: raw pointers only (ext.cpp validates the tensors).
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

namespace znhost {

static inline uint16_t f32_to_bf16_rne(uint32_t u) {      // branch-free: vectorises
  const uint32_t rounded = (u + 0x7fffu + ((u >> 16) & 1u)) >> 16;
  const uint32_t is_nan = ((u & 0x7fffffffu) > 0x7f800000u) ? 0xffffffffu : 0u;
  return (uint16_t)((rounded & ~is_nan) | (((u >> 16) | 0x40u) & is_nan));
}
// one row; cloned per ISA and dispatched once at load time (the build has no -march flag)
#if defined(__x86_64__) && defined(__GNUC__)
__attribute__((target_clones("avx512f", "avx2", "default")))
#endif
inline void convert_row_bf16(const uint32_t* __restrict__ iu, uint16_t* __restrict__ o16, int64_t row) {
#pragma GCC ivdep
  for (int64_t j = 0; j < row; ++j) o16[j] = f32_to_bf16_rne(iu[j]);
}

struct GatherJob {
  const void* src = nullptr; int64_t rows = 0, row = 0;    // dataset [rows][row] fp32 (uint8 if raw)
  const int* idx = nullptr;                                // n valid indices
  void* dst = nullptr; int64_t n = 0, cap = 0;             // staging [cap][row], rows >= n zeroed
  bool to_bf16 = false;
  bool raw = false;                                        // copy the bytes as they are
};

inline void gather_range(const GatherJob& j, int64_t b, int64_t e) {
  const size_t isz = j.raw ? 1 : 4;
  const size_t esz = j.raw ? 1 : (j.to_bf16 ? 2 : 4);
  uint8_t* dp = reinterpret_cast<uint8_t*>(j.dst);
  for (int64_t r = b; r < e; ++r) {
    uint8_t* out = dp + (size_t)r * j.row * esz;
    if (r >= j.n) { memset(out, 0, (size_t)j.row * esz); continue; }
    int64_t k = j.idx[r];
    k = k < 0 ? 0 : (k >= j.rows ? j.rows - 1 : k);
    const uint8_t* in = reinterpret_cast<const uint8_t*>(j.src) + (size_t)k * j.row * isz;
    if (!j.to_bf16) memcpy(out, in, (size_t)j.row * esz);
    else convert_row_bf16(reinterpret_cast<const uint32_t*>(in), reinterpret_cast<uint16_t*>(out), j.row);
  }
}

class HostPrefetcher {
 public:
  // heap singleton, never destroyed: the workers block on its condition variable for the whole
  // process lifetime (a static object would be torn down under them at exit)
  static HostPrefetcher& get() { static HostPrefetcher* p = new HostPrefetcher(); return *p; }

  // Starts assembling a minibatch; the index list is copied. One job in flight at a time
  // (submit waits for the previous one). Returns a ticket for wait().
  uint64_t submit(GatherJob job) {
    wait(submitted_);
    std::unique_lock<std::mutex> lk(mu_);
    idx_.assign(job.idx, job.idx + job.n);
    job.idx = idx_.data();
    job_ = job;
    remaining_ = kWorkers;
    ++submitted_;
    lk.unlock();
    cv_work_.notify_all();
    return submitted_;
  }
  void wait(uint64_t ticket) {
    if (done_.load(std::memory_order_acquire) >= ticket) return;
    std::unique_lock<std::mutex> lk(mu_);
    cv_done_.wait(lk, [&] { return done_.load(std::memory_order_acquire) >= ticket; });
  }
  const std::vector<int>& last_indices() const { return idx_; }

 private:
  static constexpr int kWorkers = 4;
  HostPrefetcher() {
    for (int w = 0; w < kWorkers; ++w) threads_.emplace_back([this, w] { loop(w); });
    for (auto& t : threads_) t.detach();     // process-lifetime pool
  }
  void loop(int w) {
    uint64_t seen = 0;
    for (;;) {
      GatherJob j;
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_work_.wait(lk, [&] { return submitted_ > seen; });
        seen = submitted_;
        j = job_;
      }
      const int64_t per = (j.cap + kWorkers - 1) / kWorkers;
      const int64_t b = w * per, e = std::min<int64_t>(j.cap, b + per);
      if (b < e) gather_range(j, b, e);
      {
        std::unique_lock<std::mutex> lk(mu_);
        if (--remaining_ == 0) {
          done_.store(seen, std::memory_order_release);
          cv_done_.notify_all();
        }
      }
    }
  }
  std::mutex mu_;
  std::condition_variable cv_work_, cv_done_;
  std::vector<std::thread> threads_;
  std::vector<int> idx_;
  GatherJob job_;
  uint64_t submitted_ = 0;
  int remaining_ = 0;
  std::atomic<uint64_t> done_{0};
};

}  // namespace znhost
