// Minimal persistent thread pool with a blocking parallel_for (host side of libcoverm_b200).
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <exception>
#include <functional>
#include <mutex>
#include <thread>
#include <utility>
#include <vector>

namespace cmbh {

class ThreadPool {
 public:
  explicit ThreadPool(int n_threads) : n_(n_threads < 1 ? 1 : n_threads) {
    for (int i = 1; i < n_; ++i) workers_.emplace_back([this, i] { worker(i); });
  }
  ~ThreadPool() {
    {
      std::unique_lock<std::mutex> lk(mu_);
      stop_ = true;
      ++generation_;
    }
    cv_.notify_all();
    for (auto& t : workers_) t.join();
  }
  int size() const { return n_; }

  // Runs fn(index, thread_id) for index in [0, n_items); dynamic scheduling; the caller participates as thread 0.
  // The first exception fn throws is rethrown here, once every thread is done (the items not started yet are skipped).
  void parallel_for(size_t n_items, const std::function<void(size_t, int)>& fn) {
    if (n_items == 0) return;
    if (n_ == 1 || n_items == 1) {
      for (size_t i = 0; i < n_items; ++i) fn(i, 0);
      return;
    }
    {
      std::unique_lock<std::mutex> lk(mu_);
      fn_ = &fn;
      n_items_ = n_items;
      next_.store(0);
      pending_ = n_ - 1;
      ++generation_;
    }
    cv_.notify_all();
    run(0);
    std::unique_lock<std::mutex> lk(mu_);
    done_cv_.wait(lk, [this] { return pending_ == 0; });
    fn_ = nullptr;
    if (error_) std::rethrow_exception(std::exchange(error_, nullptr));
  }

 private:
  void run(int tid) {
    for (;;) {
      size_t i = next_.fetch_add(1);
      if (i >= n_items_) break;
      try {
        (*fn_)(i, tid);
      } catch (...) {
        std::lock_guard<std::mutex> lk(mu_);
        if (!error_) error_ = std::current_exception();
        next_.store(n_items_);
      }
    }
  }
  void worker(int tid) {
    uint64_t seen = 0;
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(mu_);
        cv_.wait(lk, [&] { return generation_ != seen; });
        seen = generation_;
        if (stop_) return;
      }
      run(tid);
      {
        std::unique_lock<std::mutex> lk(mu_);
        if (--pending_ == 0) done_cv_.notify_one();
      }
    }
  }
  int n_;
  std::vector<std::thread> workers_;
  std::mutex mu_;
  std::condition_variable cv_, done_cv_;
  const std::function<void(size_t, int)>* fn_ = nullptr;
  size_t n_items_ = 0;
  std::atomic<size_t> next_{0};
  int pending_ = 0;
  uint64_t generation_ = 0;
  bool stop_ = false;
  std::exception_ptr error_;
};

}  // namespace cmbh
