// libcoverm_b200 -- multi-GPU: the NCCL communicator of a context (cmb_comm_*), and the gather of every rank's rows and
// histogram pairs after a sample (cmb_allgather_stats).
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include <strings.h>
#include <unistd.h>

#include "cmb_context.cuh"

namespace {

// rows[i].hist_offset += base for the rows that carry histogram pairs (cmb_allgather_stats: local -> global pair offsets)
__global__ void __launch_bounds__(256) k_rebase_hist_offsets(cmb_contig_stats* rows, uint32_t n, uint64_t base) {
  const uint32_t i = blockIdx.x * 256 + threadIdx.x;
  if (i < n && rows[i].hist_count) rows[i].hist_offset += base;
}

// NCCL writes its banner / debug lines to stdout by default; stdout carries the coverage table.
void nccl_output_to_stderr() {
  static const bool once = [] {
    // NCCL honours NCCL_DEBUG_FILE only above the VERSION level: at NCCL_DEBUG=VERSION the banner goes to stdout regardless
    const char* lvl = getenv("NCCL_DEBUG");
    if (lvl && !strcasecmp(lvl, "VERSION")) setenv("NCCL_DEBUG", "WARN", 1);  // WARN prints the same banner, to the debug file
    if (!getenv("NCCL_DEBUG_FILE")) setenv("NCCL_DEBUG_FILE", "/dev/stderr", 0);
    return true;
  }();
  (void)once;
}
// While a communicator is created, file descriptor 1 points at stderr: whatever NCCL (or a plugin it loads) prints during
// initialisation cannot end up in the coverage table.  Nothing else writes to stdout at that point (tables are printed at the end).
struct StdoutGuard {
  static std::mutex& mu() { static std::mutex m; return m; }
  std::lock_guard<std::mutex> lock{mu()};
  int saved = -1;
  StdoutGuard() {
    fflush(stdout);
    saved = dup(1);
    if (saved >= 0) dup2(2, 1);
  }
  ~StdoutGuard() {
    fflush(stdout);
    if (saved >= 0) {
      dup2(saved, 1);
      close(saved);
    }
  }
};
}  // namespace

extern "C" {

int cmb_comm_unique_id(uint8_t id[CMB_COMM_ID_BYTES]) {
  nccl_output_to_stderr();
  static_assert(sizeof(ncclUniqueId) == CMB_COMM_ID_BYTES, "ncclUniqueId is 128 bytes");
  if (!id) return fail(nullptr, CMB_E_ARG, "cmb_comm_unique_id: null argument");
  ncclUniqueId u;
  StdoutGuard guard;
  NCCL_TRY(nullptr, ncclGetUniqueId(&u));
  memcpy(id, &u, sizeof u);
  return CMB_OK;
}

int cmb_comm_init(cmb_ctx* c, const uint8_t id[CMB_COMM_ID_BYTES], int rank, int n_ranks) {
  if (!c || !id || n_ranks < 1 || rank < 0 || rank >= n_ranks) return fail(c, CMB_E_ARG, "cmb_comm_init: bad arguments");
  if (c->comm) return fail(c, CMB_E_ARG, "cmb_comm_init: the context already has a communicator");
  nccl_output_to_stderr();
  CU_TRY(c, cudaSetDevice(c->device));
  ncclUniqueId u;
  memcpy(&u, id, sizeof u);
  {
    StdoutGuard guard;
    NCCL_TRY(c, ncclCommInitRank(&c->comm, n_ranks, u, rank));
  }
  c->comm_rank = rank;
  c->comm_size = n_ranks;
  return CMB_OK;
}

int cmb_comm_init_local(cmb_ctx* const* ctxs, int n_ranks) {
  if (!ctxs || n_ranks < 1) return fail(nullptr, CMB_E_ARG, "cmb_comm_init_local: bad arguments");
  std::vector<int> devs(n_ranks);
  for (int r = 0; r < n_ranks; ++r) {
    if (!ctxs[r] || ctxs[r]->comm) return fail(ctxs[r], CMB_E_ARG, "cmb_comm_init_local: null context or communicator already set");
    devs[r] = ctxs[r]->device;
  }
  std::vector<ncclComm_t> comms(n_ranks);
  nccl_output_to_stderr();
  {
    StdoutGuard guard;
    NCCL_TRY(ctxs[0], ncclCommInitAll(comms.data(), n_ranks, devs.data()));
  }
  auto barrier = std::make_shared<LocalBarrier>();
  barrier->n = n_ranks;
  for (int r = 0; r < n_ranks; ++r) {
    ctxs[r]->local_barrier = barrier;
    ctxs[r]->comm = comms[r];
    ctxs[r]->comm_rank = r;
    ctxs[r]->comm_size = n_ranks;
  }
  return CMB_OK;
}

void cmb_comm_destroy(cmb_ctx* c) {
  if (!c || !c->comm) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  ncclCommDestroy(c->comm);
  c->comm = nullptr;
  c->local_barrier.reset();
  c->comm_rank = 0;
  c->comm_size = 1;
}

int cmb_comm_allgather(cmb_ctx* c, const void* send, void* recv, size_t bytes) {
  if (!c || !send || !recv || !bytes) return fail(c, CMB_E_ARG, "cmb_comm_allgather: bad arguments");
  if (!c->comm) return fail(c, CMB_E_ARG, "cmb_comm_allgather: no communicator (cmb_comm_init first)");
  CU_TRY(c, cudaSetDevice(c->device));
  const size_t need = bytes * (size_t)(c->comm_size + 1);
  if (int rc = c->d_xchg.ensure(c, need, need + 4096)) return rc;
  uint8_t* d_send = c->d_xchg;
  uint8_t* d_recv = c->d_xchg + bytes;
  if (c->local_barrier) c->local_barrier->arrive_and_wait();
  CU_TRY(c, cudaMemcpyAsync(d_send, send, bytes, cudaMemcpyHostToDevice, c->stream));
  NCCL_TRY(c, ncclAllGather(d_send, d_recv, bytes, ncclChar, c->comm, c->stream));
  CU_TRY(c, cudaMemcpyAsync(recv, d_recv, bytes * (size_t)c->comm_size, cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return CMB_OK;
}

int cmb_allgather_stats(cmb_ctx* c, const uint32_t* tid_cuts, const uint64_t* pair_base, cmb_contig_stats* stats, cmb_hist_pair* pairs) {
  NvtxRange nvtx_fn("cmb_allgather_stats: NCCL gather");
  if (!c || !tid_cuts) return fail(c, CMB_E_ARG, "cmb_allgather_stats: null argument");
  if (!c->comm) return fail(c, CMB_E_ARG, "cmb_allgather_stats: no communicator (cmb_comm_init first)");
  if (!c->ended || !c->ref.d_rows) return fail(c, CMB_E_ARG, "cmb_allgather_stats: no ended sample");
  const int N = c->comm_size, me = c->comm_rank;
  if (tid_cuts[0] != 0 || tid_cuts[N] != c->n_contigs || tid_cuts[me] != c->tid_begin || tid_cuts[me + 1] != c->tid_end)
    return fail(c, CMB_E_ARG, "cmb_allgather_stats: tid_cuts do not match this context's shard");
  for (int r = 0; r < N; ++r)
    if (tid_cuts[r] > tid_cuts[r + 1]) return fail(c, CMB_E_ARG, "cmb_allgather_stats: tid_cuts must be non-decreasing");
  CU_TRY(c, cudaSetDevice(c->device));
  const bool csr = pair_base && (c->params.want & CMB_WANT_HIST_CSR);
  if (csr) {
    const uint64_t total = pair_base[N];
    if (pair_base[me + 1] - pair_base[me] > c->ref.d_pairs.cap) return fail(c, CMB_E_ARG, "cmb_allgather_stats: pair_base exceeds this rank's pairs");
    if (int rc = c->d_pairs_all.ensure(c, total, total + total / 8 + 1024)) return rc;
    const uint32_t n_own = c->tid_end - c->tid_begin;
    if (n_own && pair_base[me]) {
      k_rebase_hist_offsets<<<(n_own + 255) / 256, 256, 0, c->stream>>>(c->ref.d_rows + c->tid_begin, n_own, pair_base[me]);
      CU_TRY(c, cudaGetLastError());
    }
  }
  if (c->local_barrier) c->local_barrier->arrive_and_wait();
  // every rank broadcasts its own row range in place: afterwards each rank's table is complete (an all-gather with ragged counts)
  NCCL_TRY(c, ncclGroupStart());
  for (int r = 0; r < N; ++r) {
    const size_t n = (size_t)(tid_cuts[r + 1] - tid_cuts[r]) * sizeof(cmb_contig_stats);
    if (!n) continue;
    cmb_contig_stats* p = c->ref.d_rows + tid_cuts[r];
    NCCL_TRY(c, ncclBroadcast(p, p, n, ncclChar, r, c->comm, c->stream));
  }
  if (csr) {
    for (int r = 0; r < N; ++r) {
      const size_t n = (size_t)(pair_base[r + 1] - pair_base[r]) * sizeof(cmb_hist_pair);
      if (!n) continue;
      NCCL_TRY(c, ncclBroadcast(c->ref.d_pairs, c->d_pairs_all + pair_base[r], n, ncclChar, r, c->comm, c->stream));
    }
  }
  NCCL_TRY(c, ncclGroupEnd());
  if (stats) CU_TRY(c, cudaMemcpyAsync(stats, c->ref.d_rows, sizeof(cmb_contig_stats) * (size_t)c->n_contigs, cudaMemcpyDeviceToHost, c->stream));
  if (csr && pairs && pair_base[N])
    CU_TRY(c, cudaMemcpyAsync(pairs, c->d_pairs_all, sizeof(cmb_hist_pair) * pair_base[N], cudaMemcpyDeviceToHost, c->stream));
  CU_TRY(c, cudaStreamSynchronize(c->stream));
  return CMB_OK;
}

}  // extern "C"
