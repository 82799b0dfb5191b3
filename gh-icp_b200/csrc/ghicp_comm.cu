// ghicp_comm.cu — multi-GPU exchange of the GH-ICP inner loop (one process per GPU).
// Source rows are sharded in contiguous blocks of ceil(N/world); the target set, the loop state and
// everything O(N+M) is replicated.  Per iteration ONE grouped NCCL exchange carries the per-rank
// partial CD sums, the row minima / partners / feature distances of the rank's rows and (NNR) the
// per-rank column minima; KM additionally all-gathers the per-row candidate counts and the candidate
// edges.  NCCL is dlopen'ed here: a single-GPU process never touches an NCCL symbol.
#include <dlfcn.h>
#include <nccl.h>

#include <cstring>

#include "ghicp_internal.h"

namespace ghicp_b200 {

namespace {
struct NcclApi {
  void *h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void *, void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi g_nccl;

bool load_nccl(std::string &err) {
  if (g_nccl.h) return true;
  const char *names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char *n : names) {
    g_nccl.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (g_nccl.h) break;
  }
  if (!g_nccl.h) { err = std::string("dlopen(libnccl.so.2): ") + dlerror(); return false; }
#define SYM(field, name)                                                              \
  g_nccl.field = reinterpret_cast<decltype(g_nccl.field)>(dlsym(g_nccl.h, name));      \
  if (!g_nccl.field) { err = std::string("dlsym ") + name + " failed"; return false; }
  SYM(GetUniqueId, "ncclGetUniqueId");
  SYM(CommInitRank, "ncclCommInitRank");
  SYM(CommDestroy, "ncclCommDestroy");
  SYM(AllGather, "ncclAllGather");
  SYM(Broadcast, "ncclBroadcast");
  SYM(GroupStart, "ncclGroupStart");
  SYM(GroupEnd, "ncclGroupEnd");
  SYM(GetErrorString, "ncclGetErrorString");
#undef SYM
  return true;
}
}  // namespace

#define NCK(c, call)                                                                                \
  do {                                                                                              \
    ncclResult_t r__ = (call);                                                                      \
    if (r__ != ncclSuccess) {                                                                       \
      set_error((c), std::string(#call) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "nccl error")); \
      return GHICP_E_NCCL;                                                                          \
    }                                                                                               \
  } while (0)

int comm_unique_id(void *id128) {
  std::string err;
  if (!load_nccl(err)) { set_error(nullptr, err); return GHICP_E_NCCL; }
  ncclUniqueId id;
  NCK(nullptr, g_nccl.GetUniqueId(&id));
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  std::memcpy(id128, &id, 128);
  return GHICP_OK;
}

int comm_init(Ctx *c, const void *id128, int rank, int world) {
  if (world < 1 || rank < 0 || rank >= world) { set_error(c, "comm_init: bad rank/world"); return GHICP_E_ARG; }
  if (c->N > 0) { set_error(c, "comm_init must be called before ghicp_set_keypoints"); return GHICP_E_ARG; }
  c->rank = rank; c->world = world;
  if (world == 1) return GHICP_OK;
  std::string err;
  if (!load_nccl(err)) { set_error(c, err); return GHICP_E_NCCL; }
  ncclUniqueId id;
  std::memcpy(&id, id128, 128);
  ncclComm_t comm;
  NCK(c, g_nccl.CommInitRank(&comm, world, id, rank));
  c->nccl_comm = comm;
  return GHICP_OK;
}

void comm_destroy(Ctx *c) {
  if (c->nccl_comm && g_nccl.CommDestroy) g_nccl.CommDestroy((ncclComm_t)c->nccl_comm);
  c->nccl_comm = nullptr;
}

// The per-iteration exchange of the NN / NNR paths (and the statistics of every path).
// what: EX_STATS = partial CD sums, EX_ROWS = row minima/partners/FD, EX_COLS = column minima
int comm_exchange(Ctx *c, int what) {
  if (c->world == 1) return GHICP_OK;
  ncclComm_t comm = (ncclComm_t)c->nccl_comm;
  cudaStream_t st = c->stream;
  const size_t sh = (size_t)c->shard;
  NCK(c, g_nccl.GroupStart());
  if (what & EX_STATS) NCK(c, g_nccl.AllGather(c->d_xstats + 4 * c->rank, c->d_xstats, 4, ncclDouble, comm, st));
  if (what & EX_ROWS) {
    NCK(c, g_nccl.AllGather(c->d_row_cd + sh * c->rank, c->d_row_cd, sh, ncclDouble, comm, st));
    NCK(c, g_nccl.AllGather(c->d_row_idx + sh * c->rank, c->d_row_idx, sh, ncclInt32, comm, st));
    NCK(c, g_nccl.AllGather(c->d_row_fd + sh * c->rank, c->d_row_fd, sh, ncclFloat32, comm, st));
  }
  if (what & EX_COLS) {
    // this rank's partial column minima sit in d_col_cd / d_col_idx
    NCK(c, g_nccl.AllGather(c->d_col_cd, c->d_colg_cd, (size_t)c->M, ncclUint64, comm, st));
    NCK(c, g_nccl.AllGather(c->d_col_idx, c->d_colg_idx, (size_t)c->M, ncclInt32, comm, st));
  }
  NCK(c, g_nccl.GroupEnd());
  return GHICP_OK;
}

// First use of a communicator sets up its channels (hundreds of ms): do it once when the workspaces are
// allocated instead of inside the first iteration.
int comm_warmup(Ctx *c) {
  if (c->world == 1 || !c->d_xstats) return GHICP_OK;
  NCK(c, g_nccl.AllGather(c->d_xstats + 4 * c->rank, c->d_xstats, 4, ncclDouble, (ncclComm_t)c->nccl_comm, c->stream));
  if (cudaStreamSynchronize(c->stream) != cudaSuccess) { set_error(c, "comm warm-up failed"); return GHICP_E_NCCL; }
  return GHICP_OK;
}

// KM: per-row candidate counts of the rank's rows → all ranks
int comm_gather_counts(Ctx *c) {
  if (c->world == 1) return GHICP_OK;
  ncclComm_t comm = (ncclComm_t)c->nccl_comm;
  const size_t sh = (size_t)c->shard;
  NCK(c, g_nccl.AllGather(c->d_cnt + sh * c->rank, c->d_cnt, sh, ncclInt32, comm, c->stream));
  return GHICP_OK;
}

// KM: candidate edges (column, gain, FD) of every rank's rows → all ranks.  cut[r] = CSR offset of the
// first row of rank r (cut[world] = nnz); variable sizes → one broadcast per owner inside a group.
int comm_gather_edges(Ctx *c, const long long *cut) {
  if (c->world == 1) return GHICP_OK;
  ncclComm_t comm = (ncclComm_t)c->nccl_comm;
  cudaStream_t st = c->stream;
  NCK(c, g_nccl.GroupStart());
  for (int r = 0; r < c->world; ++r) {
    const size_t off = (size_t)cut[r], cnt = (size_t)(cut[r + 1] - cut[r]);
    if (cnt == 0) continue;
    NCK(c, g_nccl.Broadcast(c->d_csr_col + off, c->d_csr_col + off, cnt, ncclInt32, r, comm, st));
    NCK(c, g_nccl.Broadcast(c->d_csr_gain + off, c->d_csr_gain + off, cnt, ncclDouble, r, comm, st));
    NCK(c, g_nccl.Broadcast(c->d_csr_fd + off, c->d_csr_fd + off, cnt, ncclFloat32, r, comm, st));
  }
  NCK(c, g_nccl.GroupEnd());
  return GHICP_OK;
}

// The one exchange of a settled KM iteration: every rank's candidate block (header with its partial CD sums + gate-checked
// edges) to every rank, in stream, nothing read by the host.
int comm_allgather_bytes(Ctx *c, const void *send, void *recv, size_t bytes) {
  if (c->world == 1) return GHICP_OK;
  NCK(c, g_nccl.AllGather(send, recv, bytes, ncclInt8, (ncclComm_t)c->nccl_comm, c->stream));
  return GHICP_OK;
}

}  // namespace ghicp_b200
