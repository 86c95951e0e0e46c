// comm.cu -- multi-GPU entry points of the C-ABI: pairs shard across GPUs, the only communication is ONE ncclAllGather of the
// fixed-size result records per batch (SURVEY.md 8e: registration pairs are independent end to end; NVLink carries ~47 KB per rank
// at 2048 pairs).  Two ways to run, both host code in C++ as the north star asks:
//   (A) one process, several devices   qb200_comm_init_all + qb200_register_batch_sharded  (ncclCommInitAll, one host thread per device)
//   (B) one process per device         qb200_comm_unique_id + qb200_comm_init_rank + qb200_register_batch_rank (torchrun / mpirun)
// The gather runs on its own stream from pinned / device staging buffers; in (B) it can be deferred so that it overlaps the next
// batch's kernels and no rank ever waits for the slowest rank inside a step.
//
// libnccl is opened with dlopen at the first comm call (the library stays loadable on hosts without NCCL, and a process that already
// carries NCCL -- e.g. through torch.distributed -- shares that instance).
#include <dlfcn.h>
#include <nccl.h>
#include <sched.h>
#include <stdlib.h>
#include <string.h>
#include <thread>
#include <vector>

#include "handle.cuh"

namespace {

struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommInitAll)(ncclComm_t*, int, const int*) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};

NcclApi& nccl() {
  static NcclApi api;
  static bool tried = false;
  if (tried) return api;
  tried = true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* n : names) {
    api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (api.lib) break;
  }
  if (!api.lib) return api;
#define QB_SYM(field, name) *(void**)(&api.field) = dlsym(api.lib, name)
  QB_SYM(GetUniqueId, "ncclGetUniqueId");
  QB_SYM(CommInitRank, "ncclCommInitRank");
  QB_SYM(CommInitAll, "ncclCommInitAll");
  QB_SYM(CommDestroy, "ncclCommDestroy");
  QB_SYM(AllGather, "ncclAllGather");
  QB_SYM(GroupStart, "ncclGroupStart");
  QB_SYM(GroupEnd, "ncclGroupEnd");
  QB_SYM(GetErrorString, "ncclGetErrorString");
#undef QB_SYM
  api.ok = api.GetUniqueId && api.CommInitRank && api.CommInitAll && api.CommDestroy && api.AllGather && api.GroupStart && api.GroupEnd;
  return api;
}

#define QB_NCCL_TRY(h, expr)                                                              \
  do {                                                                                    \
    ncclResult_t _r = (expr);                                                             \
    if (_r != ncclSuccess) {                                                              \
      (h)->fail(__FILE__, __LINE__, nccl().GetErrorString ? nccl().GetErrorString(_r) : "NCCL error"); \
      return QB200_ERR_CUDA;                                                              \
    }                                                                                     \
  } while (0)

// staging for n_local records per rank
int ensure_staging(qb200_handle* h, int n_local) {
  if (n_local <= h->comm_cap) return QB200_OK;
  cudaSetDevice(h->cfg.device);
  // the old buffers go first, so the device never holds two sets
  h->comm_cap = 0;
  h->d_send.reset(); h->d_recv.reset(); h->h_send.reset(); h->h_recv.reset();
  const size_t one = (size_t)n_local, all = one * (size_t)h->comm_world;
  QB_CUDA_TRY(h, h->d_send.alloc(one));
  QB_CUDA_TRY(h, h->d_recv.alloc(all));
  QB_CUDA_TRY(h, h->h_send.alloc(2 * one));  // two halves: the pipelined mode fills one while the other is gathered
  QB_CUDA_TRY(h, h->h_recv.alloc(all));
  h->comm_cap = n_local;
  return QB200_OK;
}

int comm_common_init(qb200_handle* h, int world, int rank) {
  h->comm_world = world;
  h->comm_rank = rank;
  cudaSetDevice(h->cfg.device);
  if (!h->comm_stream) QB_CUDA_TRY(h, h->comm_stream.create(cudaStreamNonBlocking));
  if (!h->comm_done) QB_CUDA_TRY(h, h->comm_done.create(cudaEventDisableTiming));
  return QB200_OK;
}

// enqueue H2D of this rank's records + the all-gather + D2H of everything on the comm stream (no host wait)
int enqueue_gather(qb200_handle* h, int n_local, bool group_managed, const qb200_result* src = nullptr) {
  const size_t one = (size_t)n_local * sizeof(qb200_result);
  QB_CUDA_TRY(h, cudaMemcpyAsync(h->d_send, src ? src : h->h_send, one, cudaMemcpyHostToDevice, h->comm_stream));
  (void)group_managed;
  QB_NCCL_TRY(h, nccl().AllGather(h->d_send, h->d_recv, one, ncclChar, (ncclComm_t)h->comm, h->comm_stream));
  return QB200_OK;
}

int enqueue_readback(qb200_handle* h, int n_local) {
  const size_t all = (size_t)n_local * sizeof(qb200_result) * (size_t)h->comm_world;
  QB_CUDA_TRY(h, cudaMemcpyAsync(h->h_recv, h->d_recv, all, cudaMemcpyDeviceToHost, h->comm_stream));
  QB_CUDA_TRY(h, cudaEventRecord(h->comm_done, h->comm_stream));
  return QB200_OK;
}

// rank-major staging -> round-robin global order: pair g = i * world + r
void scatter_round_robin(const qb200_result* rank_major, int world, int n_local, qb200_result* out, int n_total) {
  for (int r = 0; r < world; ++r)
    for (int i = 0; i < n_local; ++i) {
      const int g = i * world + r;
      if (g < n_total) out[g] = rank_major[(size_t)r * n_local + i];
    }
}

}  // namespace

namespace qb {
void comm_release(qb200_handle* h) {
  if (!h) return;
  if (h->comm && nccl().ok) nccl().CommDestroy((ncclComm_t)h->comm);
  h->comm = nullptr;
  h->comm_cap = 0;
  h->comm_world = 0;
}
}  // namespace qb

extern "C" {

int qb200_comm_unique_id(void* id128) {
  if (!id128) return QB200_ERR_BAD_ARG;
  if (!nccl().ok) return QB200_ERR_UNSUPPORTED;
  static_assert(sizeof(ncclUniqueId) == QB200_UNIQUE_ID_BYTES, "ncclUniqueId size");
  ncclUniqueId id;
  if (nccl().GetUniqueId(&id) != ncclSuccess) return QB200_ERR_CUDA;
  memcpy(id128, &id, sizeof(id));
  return QB200_OK;
}

int qb200_comm_init_rank(qb200_handle* h, int32_t world, int32_t rank, const void* id128) {
  if (!h || !id128 || world < 1 || rank < 0 || rank >= world) return QB200_ERR_BAD_ARG;
  if (!nccl().ok) { h->fail(__FILE__, __LINE__, "libnccl.so.2 not found"); return QB200_ERR_UNSUPPORTED; }
  if (h->comm) qb::comm_release(h);
  int rc = comm_common_init(h, world, rank);
  if (rc) return rc;
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  ncclComm_t c = nullptr;
  QB_NCCL_TRY(h, nccl().CommInitRank(&c, world, id, rank));
  h->comm = c;
  return QB200_OK;
}

int qb200_comm_init_all(qb200_handle** hs, int32_t n_dev) {
  if (!hs || n_dev < 1 || n_dev > 64) return QB200_ERR_BAD_ARG;
  for (int i = 0; i < n_dev; ++i)
    if (!hs[i]) return QB200_ERR_BAD_ARG;
  if (!nccl().ok) { hs[0]->fail(__FILE__, __LINE__, "libnccl.so.2 not found"); return QB200_ERR_UNSUPPORTED; }
  std::vector<int> devs(n_dev);
  std::vector<ncclComm_t> comms(n_dev, nullptr);
  for (int i = 0; i < n_dev; ++i) {
    if (hs[i]->comm) qb::comm_release(hs[i]);
    devs[i] = hs[i]->cfg.device;
    const int rc = comm_common_init(hs[i], n_dev, i);
    if (rc) return rc;
  }
  QB_NCCL_TRY(hs[0], nccl().CommInitAll(comms.data(), n_dev, devs.data()));
  for (int i = 0; i < n_dev; ++i) hs[i]->comm = comms[i];
  return QB200_OK;
}

// Bind the calling host thread to the CPU cores of the NUMA node the handle's GPU hangs off (2-socket boxes: launches and pinned
// copies issued from the far socket cost ~2x).  Returns the number of cores bound, 0 when the topology is unknown / not NUMA.
int qb200_bind_numa(qb200_handle* h) {
  if (!h) return QB200_ERR_BAD_ARG;
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof(bus), h->cfg.device) != cudaSuccess) return 0;
  for (char* c = bus; *c; ++c)
    if (*c >= 'A' && *c <= 'Z') *c = (char)(*c - 'A' + 'a');
  char path[128];
  snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
  FILE* f = fopen(path, "r");
  if (!f) return 0;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  if (node < 0) return 0;
  snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
  f = fopen(path, "r");
  if (!f) return 0;
  char list[1024] = {0};
  if (!fgets(list, sizeof(list), f)) list[0] = 0;
  fclose(f);
  cpu_set_t want, have, both;
  CPU_ZERO(&want);
  for (char* tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
    int a = 0, b = 0;
    const int k = sscanf(tok, "%d-%d", &a, &b);
    if (k == 1) b = a;
    if (k >= 1)
      for (int c = a; c <= b && c < CPU_SETSIZE; ++c) CPU_SET(c, &want);
  }
  if (sched_getaffinity(0, sizeof(have), &have) != 0) return 0;
  CPU_AND(&both, &want, &have);   // stay inside the cgroup / taskset the process was given
  const int n = CPU_COUNT(&both);
  if (n == 0) return 0;
  if (sched_setaffinity(0, sizeof(both), &both) != 0) return 0;
  return n;
}

// wait for the gather in flight and hand out its records
static int gather_wait(qb200_handle* h) {
  if (h->pend_gather_n <= 0) return QB200_OK;
  cudaSetDevice(h->cfg.device);
  QB_CUDA_TRY(h, cudaEventSynchronize(h->comm_done));
  // whatever the caller records on the handle's stream next is ordered after the gather
  QB_CUDA_TRY(h, cudaStreamWaitEvent(h->lane[0]->stream, h->comm_done, 0));
  scatter_round_robin(h->h_recv, h->comm_world, h->pend_gather_n, h->pend_gather_dst, h->comm_world * h->pend_gather_n);
  h->pend_gather_n = 0;
  h->pend_gather_dst = nullptr;
  return QB200_OK;
}

// pipelined mode: the local batch that has been queued but not gathered yet -> complete its records, start its gather
static int pipe_finish(qb200_handle* h) {
  if (h->pipe_n <= 0) return QB200_OK;
  const qb200_result* src = h->h_send + (size_t)h->pipe_buf * h->comm_cap;
  int rc = qb::collect_batch(h, src);          // every wave that writes into this half
  if (rc == QB200_OK) rc = gather_wait(h);     // the gather before it owns d_send / h_recv
  if (rc == QB200_OK) rc = enqueue_gather(h, h->pipe_n, false, src);
  if (rc == QB200_OK) rc = enqueue_readback(h, h->pipe_n);
  if (rc == QB200_OK) { h->pend_gather_n = h->pipe_n; h->pend_gather_dst = h->pipe_dst; }
  h->pipe_n = 0;
  h->pipe_dst = nullptr;
  return rc;
}

int qb200_comm_wait(qb200_handle* h) {
  if (!h) return QB200_ERR_BAD_ARG;
  const int rc = pipe_finish(h);
  const int rc2 = gather_wait(h);
  return rc ? rc : rc2;
}

int qb200_register_batch_rank(qb200_handle* h, const qb200_pair* local_pairs, int32_t n_local, const qb200_params* p, qb200_mem_kind kind,
                              qb200_result* all_results, int32_t defer) {
  if (!h || n_local < 0 || (n_local > 0 && (!local_pairs || !all_results))) return QB200_ERR_BAD_ARG;
  if (!h->comm) { h->fail(__FILE__, __LINE__, "qb200_comm_init_rank / _init_all has not been called on this handle"); return QB200_ERR_BAD_ARG; }
  int rc;
  if (defer == 2 && n_local > 0 && n_local <= h->comm_cap) {
    // Pipelined (a stream of batches): queue this rank's batch k+1 first, then complete batch k's records (its waves are the
    // oldest in flight) and start ITS gather; the gather of batch k-1 is collected on the way.  qb200_comm_wait ends the stream.
    if ((rc = gather_wait(h))) return rc;
    const int buf = h->pipe_n > 0 ? 1 - h->pipe_buf : 0;
    if ((rc = qb200_register_batch_enqueue(h, local_pairs, n_local, p, kind, h->h_send + (size_t)buf * h->comm_cap))) return rc;
    if ((rc = pipe_finish(h))) return rc;
    h->pipe_n = n_local;
    h->pipe_dst = all_results;
    h->pipe_buf = buf;
    return QB200_OK;
  }
  rc = qb200_comm_wait(h);  // a deferred gather of the previous batch still owns the staging buffers
  if (rc) return rc;
  if (n_local == 0) return QB200_OK;
  if ((rc = ensure_staging(h, n_local))) return rc;
  if (defer == 2) {  // first batch of a pipelined stream (the staging buffers have just been sized)
    if ((rc = qb200_register_batch_enqueue(h, local_pairs, n_local, p, kind, h->h_send))) return rc;
    h->pipe_n = n_local;
    h->pipe_dst = all_results;
    h->pipe_buf = 0;
    return QB200_OK;
  }
  if ((rc = qb200_register_batch(h, local_pairs, n_local, p, kind, h->h_send))) return rc;
  if ((rc = enqueue_gather(h, n_local, false))) return rc;
  if ((rc = enqueue_readback(h, n_local))) return rc;
  h->pend_gather_n = n_local;
  h->pend_gather_dst = all_results;
  return defer ? QB200_OK : qb200_comm_wait(h);
}

int qb200_register_batch_sharded(qb200_handle** hs, int32_t n_dev, const qb200_pair* pairs, int32_t n_pairs, const qb200_params* p,
                                 qb200_mem_kind kind, qb200_result* results) {
  if (!hs || n_dev < 1 || n_pairs < 0 || (n_pairs > 0 && (!pairs || !results)) || !p) return QB200_ERR_BAD_ARG;
  for (int i = 0; i < n_dev; ++i)
    if (!hs[i] || !hs[i]->comm || hs[i]->comm_world != n_dev || hs[i]->comm_rank != i) return QB200_ERR_BAD_ARG;
  if (n_pairs == 0) return QB200_OK;
  const int n_local = (n_pairs + n_dev - 1) / n_dev;  // equal counts for the all-gather; missing pairs stay zero records
  std::vector<std::vector<qb200_pair>> shard(n_dev);
  for (int g = 0; g < n_pairs; ++g) shard[g % n_dev].push_back(pairs[g]);   // SURVEY.md 8e: pair p -> device p mod G
  std::vector<int> rcs(n_dev, QB200_OK);
  std::vector<std::thread> th;
  for (int d = 0; d < n_dev; ++d) {
    rcs[d] = ensure_staging(hs[d], n_local);
    if (rcs[d]) return rcs[d];
    memset(hs[d]->h_send, 0, (size_t)n_local * sizeof(qb200_result));
  }
  for (int d = 0; d < n_dev; ++d)
    th.emplace_back([&, d]() {
      if (!shard[d].empty()) rcs[d] = qb200_register_batch(hs[d], shard[d].data(), (int)shard[d].size(), p, kind, hs[d]->h_send);
    });
  for (auto& t : th) t.join();
  for (int d = 0; d < n_dev; ++d)
    if (rcs[d]) { if (d) hs[0]->fail(__FILE__, __LINE__, hs[d]->err); return rcs[d]; }
  // one grouped all-gather over every device of this process
  for (int d = 0; d < n_dev; ++d) {
    cudaSetDevice(hs[d]->cfg.device);
    QB_CUDA_TRY(hs[d], cudaMemcpyAsync(hs[d]->d_send, hs[d]->h_send, (size_t)n_local * sizeof(qb200_result), cudaMemcpyHostToDevice, hs[d]->comm_stream));
  }
  QB_NCCL_TRY(hs[0], nccl().GroupStart());
  for (int d = 0; d < n_dev; ++d)
    QB_NCCL_TRY(hs[d], nccl().AllGather(hs[d]->d_send, hs[d]->d_recv, (size_t)n_local * sizeof(qb200_result), ncclChar, (ncclComm_t)hs[d]->comm,
                                        hs[d]->comm_stream));
  QB_NCCL_TRY(hs[0], nccl().GroupEnd());
  int rc = enqueue_readback(hs[0], n_local);
  if (rc) return rc;
  for (int d = 0; d < n_dev; ++d) {
    cudaSetDevice(hs[d]->cfg.device);
    QB_CUDA_TRY(hs[d], cudaStreamSynchronize(hs[d]->comm_stream));
  }
  scatter_round_robin(hs[0]->h_recv, n_dev, n_local, results, n_pairs);
  return QB200_OK;
}

}  // extern "C"
