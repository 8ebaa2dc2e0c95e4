// The task scheduler of the region-parallel BAM decode (the block index and the record decoder it runs are in bam_source.hpp).
//
// Work items are ~1 MB of uncompressed data (whole BGZF blocks).  Three kinds of work, none of which ever blocks on
// another thread:
//   INFLATE(item)   any worker, any order: zlib-inflate the item's blocks into a pooled buffer.
//                   While the data is hot in its cache the same worker GUESSES where the first whole record of the
//                   item starts (a chain of plausible BAM record headers) and pre-walks the block_size chain from there.
//   CHAIN           whoever gets the try-lock: for every consecutive inflated item, finish the record that straddles
//                   the item boundary — which gives the exact start — and, if the guess was right (it practically
//                   always is), take the pre-walked offsets; otherwise walk the chain now.  Then assign the item a
//                   contiguous slice of a staging batch and queue it for extraction.  O(1) per item, exact always.
//   EXTRACT(item)   any worker: decode the item's records straight into the pinned SoA staging batch.
// The calling thread is the coordinator: it alone talks to the (not thread-safe) device ABI — it keeps one staging
// batch acquired ahead of the chain and submits each batch once every item assigned to it has been extracted.
#pragma once
#include <atomic>
#include <chrono>
#include <deque>
#include <exception>
#include <memory>
#include <mutex>
#include <thread>

#include "bam_source.hpp"

namespace cmbh {

struct PipelineCounts {
  uint64_t n_records = 0, primaries = 0;
  // summed over the worker threads (seconds): where the decode time goes
  double inflate_s = 0, scan_s = 0, extract_s = 0, idle_s = 0;
  uint32_t n_items = 0, n_workers = 0;
};

inline double pipeline_now() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

struct WorkCtx {  // pooled per-item scratch
  std::unique_ptr<uint8_t[]> buf;
  size_t cap = 0;
  std::vector<uint32_t> offs;
  std::vector<uint8_t> stitched;
};
// Scratch that outlives one sample: re-using the item buffers avoids re-faulting hundreds of MB of fresh pages from
// 100+ threads at once on every sample.
struct DecodeScratch {
  std::vector<WorkCtx> ctxs;
};

// Runs the whole record stream (starting at uncompressed offset `records_at`) through the device context.
// acquire()/submit() are the caller's wrappers around cmb_acquire_batch / cmb_submit_batch (called only from this thread).
template <class Acquire, class Submit>
PipelineCounts run_decode_pipeline(const BlockIndex& bx, uint64_t records_at, uint32_t n_ref, int n_threads, uint32_t cap_r,
                                   uint32_t cap_i, uint32_t n_staging, DecodeScratch& scratch, Acquire acquire, Submit submit) {
  constexpr size_t ITEM_BYTES = 1u << 20;
  struct Item {
    size_t b0 = 0, b1 = 0, usize = 0;
    std::atomic<int> inflated{0};
    int ctx = -1;
    // speculative alignment, set by the inflating worker
    int64_t guess_start = -1;
    size_t guess_tail = 0;      // offset of the incomplete last record
    uint64_t guess_ub_iv = 0;
    // set by the chain step
    bool have_stitched = false;
    uint64_t seq = 0;
    uint32_t r0 = 0, i0 = 0, ub_iv = 0, n_rec = 0;
  };
  size_t first_block = 0;
  while (first_block < bx.blocks.size() && bx.ustart[first_block + 1] <= records_at) ++first_block;
  const uint64_t skip0 = first_block < bx.blocks.size() ? records_at - bx.ustart[first_block] : 0;
  size_t n_items = 0, max_item = 0;
  for (size_t b = first_block; b < bx.blocks.size();) {
    size_t e = b;
    uint64_t sz = 0;
    while (e < bx.blocks.size() && (sz == 0 || sz + bx.blocks[e].isize <= ITEM_BYTES)) sz += bx.blocks[e++].isize;
    ++n_items;
    max_item = std::max<size_t>(max_item, sz);
    b = e;
  }
  std::unique_ptr<Item[]> items(new Item[n_items + 1]);
  {
    size_t k = 0;
    for (size_t b = first_block; b < bx.blocks.size(); ++k) {
      size_t e = b;
      uint64_t sz = 0;
      while (e < bx.blocks.size() && (sz == 0 || sz + bx.blocks[e].isize <= ITEM_BYTES)) sz += bx.blocks[e++].isize;
      items[k].b0 = b;
      items[k].b1 = e;
      items[k].usize = (size_t)sz;
      b = e;
    }
  }
  const int nt = std::max(1, std::min<int>(n_threads, (int)std::max<size_t>(1, n_items)));

  // ---- pooled contexts (bounds memory: 3 buffers per worker)
  const int n_ctx = nt * 4;
  std::vector<WorkCtx>& ctxs = scratch.ctxs;
  if ((int)ctxs.size() < n_ctx) ctxs.resize(n_ctx);
  std::mutex ctx_mu;
  std::vector<int> free_ctx;
  for (int k = 0; k < n_ctx; ++k) free_ctx.push_back(k);
  auto get_ctx = [&]() {
    std::lock_guard<std::mutex> g(ctx_mu);
    if (free_ctx.empty()) return -1;
    const int k = free_ctx.back();
    free_ctx.pop_back();
    return k;
  };
  auto put_ctx = [&](int k) {
    std::lock_guard<std::mutex> g(ctx_mu);
    free_ctx.push_back(k);
  };

  // ---- per-batch bookkeeping, indexed by batch sequence number (a batch holds >= 1 item, so n_items+1 bounds it)
  struct BatchInfo {
    std::atomic<int> closed{0};
    std::atomic<uint32_t> done{0};
    uint32_t final_r = 0, final_i = 0, final_items = 0;
  };
  std::unique_ptr<BatchInfo[]> batches(new BatchInfo[n_items + 2]);
  struct Slot {
    std::atomic<int64_t> have_seq{-1};
    cmb_read_batch ptrs{};
  };
  std::unique_ptr<Slot[]> slots(new Slot[n_staging]);
  std::atomic<int64_t> needed_seq{0};

  // ---- chain state (guarded by chain_mu)
  std::mutex chain_mu;
  std::atomic<size_t> chain_head{0};
  std::vector<uint8_t> carry;
  uint64_t cur_seq = 0;
  uint32_t used_r = 0, used_i = 0, items_in_batch = 0;

  std::mutex q_mu;
  std::deque<size_t> extract_q;
  std::atomic<size_t> next_inflate{0}, items_finished{0};
  std::atomic<bool> abort{false};
  std::atomic<int> workers_left{0};
  std::exception_ptr first_error;
  std::mutex err_mu;
  std::atomic<uint64_t> tot_records{0}, tot_primaries{0};
  std::mutex stat_mu;
  PipelineCounts stats;

  auto fail = [&](std::exception_ptr e) {
    std::lock_guard<std::mutex> g(err_mu);
    if (!first_error) first_error = e;
    abort = true;
  };

  // CHAIN step for item i (chain_mu held): alignment, block_size walk, batch assignment.
  auto chain_step = [&](size_t i) {
    Item& it = items[i];
    WorkCtx& w = ctxs[it.ctx];
    const uint8_t* buf = w.buf.get();
    const size_t usize = it.usize;
    size_t pos = i == 0 ? (size_t)skip0 : 0;
    it.have_stitched = false;
    uint64_t ub_iv = 0;
    bool swallowed = false;  // the whole item is the middle of one huge record
    if (!carry.empty()) {
      w.stitched.swap(carry);
      carry.clear();
      while (w.stitched.size() < 4 && pos < usize) w.stitched.push_back(buf[pos++]);
      if (w.stitched.size() < 4) {
        swallowed = true;
      } else {
        const size_t need = 4 + (size_t)rd_u32(w.stitched.data());
        if (need < 36) throw Panic("Error reading BAM record: corrupt block_size");
        const size_t take = std::min(need - w.stitched.size(), usize - pos);
        w.stitched.insert(w.stitched.end(), buf + pos, buf + pos + take);
        pos += take;
        if (w.stitched.size() < need) swallowed = true;
        else {
          it.have_stitched = true;
          const int64_t ops = record_cigar_ops(w.stitched.data());
          if (ops < 0) throw_bad_record_layout();
          ub_iv += (uint64_t)ops;
        }
      }
    }
    if (swallowed) {
      carry.swap(w.stitched);
      w.offs.clear();
    } else if (it.guess_start == (int64_t)pos) {  // the worker's pre-walk started at the right byte: take it
      ub_iv += it.guess_ub_iv;
      carry.assign(buf + it.guess_tail, buf + usize);
    } else {
      w.offs.clear();
      pos = walk_records(buf, pos, usize, false, [&](size_t rec) {
        const int64_t ops = record_cigar_ops(buf + rec);
        if (ops < 0) throw_bad_record_layout();
        w.offs.push_back((uint32_t)rec);
        ub_iv += (uint64_t)ops;
        return true;
      });
      carry.assign(buf + pos, buf + usize);
    }
    const uint32_t n_rec = (uint32_t)w.offs.size() + (it.have_stitched ? 1u : 0u);
    if (n_rec > cap_r || ub_iv > cap_i) throw ExitError(1, "a decode work item holds more records than a device batch");
    if (used_r + (uint64_t)n_rec > cap_r || used_i + ub_iv > cap_i) {  // close the current batch, open the next
      BatchInfo& b = batches[cur_seq];
      b.final_r = used_r;
      b.final_i = used_i;
      b.final_items = items_in_batch;
      b.closed.store(1, std::memory_order_release);
      ++cur_seq;
      used_r = used_i = items_in_batch = 0;
      needed_seq.store((int64_t)cur_seq, std::memory_order_release);
    }
    it.seq = cur_seq;
    it.r0 = used_r;
    it.i0 = used_i;
    it.ub_iv = (uint32_t)ub_iv;
    it.n_rec = n_rec;
    used_r += n_rec;
    used_i += (uint32_t)ub_iv;
    if (n_rec) ++items_in_batch;
  };

  // Run the chain over every consecutive inflated item (no-op if another thread is already doing so).
  auto run_chain = [&](double& t_scan) {
    for (;;) {
      if (!chain_mu.try_lock()) return;
      const double t0 = pipeline_now();
      size_t h = chain_head.load(std::memory_order_relaxed);
      try {
        while (h < n_items && items[h].inflated.load(std::memory_order_acquire)) {
          chain_step(h);
          if (items[h].n_rec) {
            std::lock_guard<std::mutex> g(q_mu);
            extract_q.push_back(h);
          } else {
            put_ctx(items[h].ctx);
            items_finished.fetch_add(1);
          }
          ++h;
          // bytes left over after the last item are a record cut short: htslib's bam_read1 fails there and the reference
          // panics on the Err (contig.rs:113-115)
          if (h == n_items && !carry.empty()) throw Panic("Error reading BAM record: truncated");
          chain_head.store(h, std::memory_order_release);
        }
      } catch (...) {
        chain_mu.unlock();
        throw;
      }
      chain_mu.unlock();
      t_scan += pipeline_now() - t0;
      // an item may have become inflated between our last check and the unlock: look again
      if (h < n_items && items[h].inflated.load(std::memory_order_acquire)) continue;
      return;
    }
  };

  auto plausible = [&](const uint8_t* buf, size_t s, size_t usize) { return record_plausible(buf, s, usize, n_ref); };
  // Guess the first record boundary of an item and pre-walk its block_size chain while the data is cache-hot.
  auto prewalk = [&](Item& it, WorkCtx& w, size_t index) {
    const uint8_t* buf = w.buf.get();
    const size_t usize = it.usize;
    it.guess_start = -1;
    w.offs.clear();
    size_t start = (size_t)-1;
    if (index == 0) {
      start = (size_t)skip0;  // known exactly
    } else {
      const size_t limit = std::min<size_t>(usize, 1u << 18);
      for (size_t s = 0; s < limit && start == (size_t)-1; ++s) {
        if (!plausible(buf, s, usize)) continue;
        size_t q = s;
        int ok = 0;
        while (ok < 6) {  // a run of six consistent headers (or reaching the end of the item) confirms the guess
          if (q + 36 > usize) { ok = 6; break; }
          if (!plausible(buf, q, usize)) break;
          q += 4 + (size_t)rd_u32(buf + q);
          ++ok;
        }
        if (ok >= 6) start = s;
      }
      if (start == (size_t)-1) return;  // nothing recognisable (e.g. the inside of one huge record): chain step walks it
    }
    size_t pos = start;
    uint64_t ub = 0;
    while (pos + 4 <= usize) {
      const uint32_t bs = rd_u32(buf + pos);
      if (bs < 32 || pos + 4 + (size_t)bs > usize) break;
      const int64_t ops = record_cigar_ops(buf + pos);
      if (ops < 0) {  // fields overrun the record: let the chain step raise the error
        w.offs.clear();
        return;
      }
      w.offs.push_back((uint32_t)pos);
      ub += (uint64_t)ops;
      pos += 4 + (size_t)bs;
    }
    if (pos + 4 <= usize && rd_u32(buf + pos) < 32) {  // corrupt chain: let the chain step raise the error
      w.offs.clear();
      return;
    }
    it.guess_start = (int64_t)start;
    it.guess_tail = pos;
    it.guess_ub_iv = ub;
  };

  auto extract = [&](size_t i, uint64_t& my_primaries) {
    Item& it = items[i];
    WorkCtx& w = ctxs[it.ctx];
    const cmb_read_batch& b = slots[it.seq % n_staging].ptrs;
    uint32_t r = it.r0, iv = it.i0;
    Tuple t;
    auto put = [&](const uint8_t* rec) {
      const uint32_t n_iv = decode_bam_record(rec, t, b.iv_start + iv, b.iv_len + iv);
      put_tuple(b, r, iv, t, nullptr, nullptr);
      iv += n_iv;
      ++r;
      if (!(t.flag & 0x900)) ++my_primaries;
    };
    if (it.have_stitched) put(w.stitched.data());
    const uint8_t* buf = w.buf.get();
    for (uint32_t o : w.offs) put(buf + o);
    for (const uint32_t end_iv = it.i0 + it.ub_iv; iv < end_iv; ++iv) {  // unused part of the interval reservation
      b.iv_start[iv] = CMB_IV_PAD;
      b.iv_len[iv] = 0;
    }
  };

  auto worker = [&]() {
    double t_inf = 0, t_scan = 0, t_ext = 0, t_idle = 0;
    uint64_t my_records = 0, my_primaries = 0;
    try {
      BgzfInflater inflater;
      bool inflate_done = false;
      while (!abort) {
        // 1. extraction first: it frees buffers and completes batches
        size_t ei = (size_t)-1;
        {
          std::lock_guard<std::mutex> g(q_mu);
          if (!extract_q.empty()) {
            ei = extract_q.front();
            if (slots[items[ei].seq % n_staging].have_seq.load(std::memory_order_acquire) == (int64_t)items[ei].seq) extract_q.pop_front();
            else ei = (size_t)-1;  // its staging batch has not been handed out yet (the coordinator is about to)
          }
        }
        if (ei != (size_t)-1) {
          const double t0 = pipeline_now();
          extract(ei, my_primaries);
          my_records += items[ei].n_rec;
          put_ctx(items[ei].ctx);
          batches[items[ei].seq].done.fetch_add(1, std::memory_order_acq_rel);
          items_finished.fetch_add(1);
          t_ext += pipeline_now() - t0;
          continue;
        }
        // 2. inflate the next item
        if (!inflate_done) {
          const int c = get_ctx();
          if (c >= 0) {
            const size_t j = next_inflate.fetch_add(1);
            if (j >= n_items) {
              put_ctx(c);
              inflate_done = true;
              continue;
            }
            const double t0 = pipeline_now();
            WorkCtx& w = ctxs[c];
            if (w.cap < max_item + 8) {
              w.buf.reset(new uint8_t[max_item + 8]);
              w.cap = max_item + 8;
            }
            bx.inflate(items[j].b0, items[j].b1, w.buf.get(), inflater);
            prewalk(items[j], w, j);
            items[j].ctx = c;
            items[j].inflated.store(1, std::memory_order_release);
            t_inf += pipeline_now() - t0;
            run_chain(t_scan);
            continue;
          }
        }
        // 3. nothing to do right now
        if (items_finished.load() >= n_items) break;
        const double t0 = pipeline_now();
        run_chain(t_scan);  // in case the head became ready while nobody was looking
        std::this_thread::sleep_for(std::chrono::microseconds(20));
        t_idle += pipeline_now() - t0;
      }
    } catch (...) {
      fail(std::current_exception());
    }
    tot_records += my_records;
    tot_primaries += my_primaries;
    {
      std::lock_guard<std::mutex> g(stat_mu);
      stats.inflate_s += t_inf;
      stats.scan_s += t_scan;
      stats.extract_s += t_ext;
      stats.idle_s += t_idle;
    }
    workers_left.fetch_sub(1);
  };

  workers_left = nt;
  std::vector<std::thread> pool;
  for (int k = 0; k < nt; ++k) pool.emplace_back(worker);

  // ---- coordinator: the only thread that touches the device ABI
  int64_t acquired = 0, submitted = 0;
  try {
    for (;;) {
      bool progressed = false;
      // keep one batch acquired ahead of the chain so that extraction never waits for staging memory
      while (acquired <= needed_seq.load(std::memory_order_acquire) + 1 && acquired - submitted < (int64_t)n_staging) {
        Slot& s = slots[acquired % n_staging];
        acquire(&s.ptrs);
        s.have_seq.store(acquired, std::memory_order_release);
        ++acquired;
        progressed = true;
      }
      if (submitted < acquired) {
        BatchInfo& b = batches[submitted];
        if (b.closed.load(std::memory_order_acquire) && b.done.load(std::memory_order_acquire) == b.final_items) {
          Slot& s = slots[submitted % n_staging];
          s.ptrs.iv_begin[b.final_r] = b.final_i;
          submit(b.final_r, b.final_i);
          ++submitted;
          progressed = true;
        }
      }
      if (abort) break;
      if (workers_left.load() == 0 && !progressed) {
        bool more = submitted < acquired && batches[submitted].closed.load();
        if (!more) break;
      }
      if (!progressed) std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
  } catch (...) {
    fail(std::current_exception());
  }
  for (auto& th : pool) th.join();
  if (first_error) {
    try {  // hand back every acquired batch so that the context can be reused
      for (; submitted < acquired; ++submitted) submit(0, 0);
    } catch (...) {
    }
    std::rethrow_exception(first_error);
  }
  // ---- the last, still open batch (and a batch acquired ahead but never used)
  for (; submitted < acquired; ++submitted) {
    Slot& s = slots[submitted % n_staging];
    BatchInfo& b = batches[submitted];
    if (b.closed.load()) {
      s.ptrs.iv_begin[b.final_r] = b.final_i;
      submit(b.final_r, b.final_i);
    } else if ((uint64_t)submitted == cur_seq) {
      s.ptrs.iv_begin[used_r] = used_i;
      submit(used_r, used_i);
    } else {
      submit(0, 0);
    }
  }
  PipelineCounts c = stats;
  c.n_records = tot_records;
  c.primaries = tot_primaries;
  c.n_items = (uint32_t)n_items;
  c.n_workers = (uint32_t)nt;
  return c;
}

}  // namespace cmbh
