// comm.cu -- the one exchange step of the scene-sharded path, inside the library: NCCL send/recv over NVLink to scatter a
// request from an ingest rank to the ranks that own its scenes and to gather the assigned track records back.
//
// Scenes are independent (`compatible()` needs equal scene ids, src/trackers/sort.rs:250-251) and track state is sticky per
// GPU, so a multi-GPU tracker is N independent single-GPU trackers plus this exchange -- the GPU counterpart of the
// reference's voting-shard fan-out (src/trackers/sort/batch_api.rs:197-207: one channel per voting thread, results collected
// on PredictionBatchResult's channel).  One process per GPU; the caller (bench.py under torchrun, or a Rust host) ships the
// 128-byte NCCL unique id from rank 0 to the other ranks over whatever control channel it has.
//
// NCCL is resolved at run time (dlopen "libnccl.so.2"): the library has no link-time dependency on it, a process that never
// creates a communicator never loads it, and inside a PyTorch process the already loaded libnccl is the one that is used.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstdio>
#include <cstring>
#include <string>

#include "../../include/similari_b200.h"
#include "sb_host.cuh"

namespace {

using sb::fail;

typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
enum { kNcclUint8 = 1 };

struct Nccl {
  void* h = nullptr;
  int (*GetUniqueId)(ncclUniqueId*) = nullptr;
  int (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  int (*CommDestroy)(ncclComm_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  int (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  int (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  std::string err;
};

Nccl* nccl() {
  static Nccl n;
  static bool tried = false;
  if (tried) return &n;
  tried = true;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) {
    n.h = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
    if (n.h) break;
  }
  if (!n.h) { n.err = "libnccl.so.2 not found (dlopen)"; return &n; }
#define SYM(field, name)                                                   \
  *(void**)(&n.field) = dlsym(n.h, name);                                  \
  if (!n.field) { n.err = std::string("symbol missing in libnccl: ") + name; n.h = nullptr; return &n; }
  SYM(GetUniqueId, "ncclGetUniqueId")
  SYM(CommInitRank, "ncclCommInitRank")
  SYM(CommDestroy, "ncclCommDestroy")
  SYM(GroupStart, "ncclGroupStart")
  SYM(GroupEnd, "ncclGroupEnd")
  SYM(Send, "ncclSend")
  SYM(Recv, "ncclRecv")
  SYM(GetErrorString, "ncclGetErrorString")
#undef SYM
  return &n;
}

}  // namespace

struct sb200_comm {
  ncclComm_t comm = nullptr;
  int rank = 0, world = 1, device = 0;
};

#define NC(x)                                                                                            \
  do {                                                                                                   \
    int r_ = (x);                                                                                        \
    if (r_ != 0) return fail(SB200_ERR_CUDA, "%s failed: %s", #x, nccl()->GetErrorString(r_));            \
  } while (0)

extern "C" {

int sb200_comm_unique_id(void* out128) {
  if (!out128) return fail(SB200_ERR_INVALID, "out128 is NULL");
  Nccl* n = nccl();
  if (!n->h) return fail(SB200_ERR_CUDA, "%s", n->err.c_str());
  ncclUniqueId id;
  NC(n->GetUniqueId(&id));
  memcpy(out128, &id, 128);
  return 0;
}

int sb200_comm_create(int32_t rank, int32_t world, const void* id128, int32_t device, sb200_comm** out) {
  if (!id128 || !out || world < 1 || rank < 0 || rank >= world) return fail(SB200_ERR_INVALID, "bad arguments");
  *out = nullptr;
  Nccl* n = nccl();
  if (!n->h) return fail(SB200_ERR_CUDA, "%s", n->err.c_str());
  if (cudaSetDevice(device) != cudaSuccess) return fail(SB200_ERR_CUDA, "cudaSetDevice failed");
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  sb200_comm* c = new sb200_comm();
  c->rank = rank; c->world = world; c->device = device;
  int r = n->CommInitRank(&c->comm, world, id, rank);
  if (r != 0) { delete c; return fail(SB200_ERR_CUDA, "ncclCommInitRank failed: %s", n->GetErrorString(r)); }
  *out = c;
  return 0;
}

void sb200_comm_destroy(sb200_comm* c) {
  if (!c) return;
  if (c->comm) nccl()->CommDestroy(c->comm);
  delete c;
}

// One grouped exchange of `ncols` row-major columns: column k has row_bytes[k] bytes per detection; the root's copy of
// column k holds all shards back to back (rank r owns rows [det_range[r], det_range[r + 1])).
static int exchange(sb200_comm* c, int root, const int32_t* det_range, int ncols, const size_t* row_bytes,
                    void* const* root_cols, void* const* my_cols, bool scatter, cudaStream_t st) {
  Nccl* n = nccl();
  if (cudaSetDevice(c->device) != cudaSuccess) return fail(SB200_ERR_CUDA, "cudaSetDevice failed");
  const int me = c->rank;
  const size_t my_rows = (size_t)(det_range[me + 1] - det_range[me]);
  NC(n->GroupStart());
  for (int k = 0; k < ncols; ++k) {
    if (!my_cols[k]) continue;
    const size_t rb = row_bytes[k];
    if (me == root) {
      if (!root_cols[k]) { n->GroupEnd(); return fail(SB200_ERR_INVALID, "root column is NULL"); }
      char* all = reinterpret_cast<char*>(root_cols[k]);
      for (int r = 0; r < c->world; ++r) {
        const size_t rows = (size_t)(det_range[r + 1] - det_range[r]);
        if (rows == 0) continue;
        char* slab = all + (size_t)det_range[r] * rb;
        if (r == root) {   // the root's own shard: a device copy, no self-send
          if (scatter) cudaMemcpyAsync(my_cols[k], slab, rows * rb, cudaMemcpyDeviceToDevice, st);
          else cudaMemcpyAsync(slab, my_cols[k], rows * rb, cudaMemcpyDeviceToDevice, st);
        } else if (scatter) {
          NC(n->Send(slab, rows * rb, kNcclUint8, r, c->comm, st));
        } else {
          NC(n->Recv(slab, rows * rb, kNcclUint8, r, c->comm, st));
        }
      }
    } else if (my_rows > 0) {
      if (scatter) NC(n->Recv(my_cols[k], my_rows * rb, kNcclUint8, root, c->comm, st));
      else NC(n->Send(my_cols[k], my_rows * rb, kNcclUint8, root, c->comm, st));
    }
  }
  NC(n->GroupEnd());
  return 0;
}

int sb200_shard_scatter(sb200_comm* c, int32_t root, const int32_t* det_range, int32_t feature_dim, const float* all_boxes,
                        const float* all_features, const uint8_t* all_has_feature, const float* all_quality,
                        const int64_t* all_custom_ids, float* my_boxes, float* my_features, uint8_t* my_has_feature,
                        float* my_quality, int64_t* my_custom_ids, void* cuda_stream) {
  if (!c || !det_range || root < 0 || root >= c->world || !my_boxes) return fail(SB200_ERR_INVALID, "bad arguments");
  const size_t rb[5] = {24, (size_t)feature_dim * 4, 1, 4, 8};
  void* rootc[5] = {(void*)all_boxes, (void*)all_features, (void*)all_has_feature, (void*)all_quality, (void*)all_custom_ids};
  void* myc[5] = {my_boxes, my_features, my_has_feature, my_quality, my_custom_ids};
  return exchange(c, root, det_range, 5, rb, rootc, myc, /*scatter=*/true, reinterpret_cast<cudaStream_t>(cuda_stream));
}

int sb200_shard_gather(sb200_comm* c, int32_t root, const int32_t* det_range, const sb200_predict_out* mine,
                       const sb200_predict_out* all, void* cuda_stream) {
  if (!c || !det_range || root < 0 || root >= c->world || !mine) return fail(SB200_ERR_INVALID, "bad arguments");
  if (c->rank == root && !all) return fail(SB200_ERR_INVALID, "the root needs the `all` columns");
  const size_t rb[6] = {8, 4, 4, 1, 24, 24};
  sb200_predict_out none{};
  const sb200_predict_out& a = all ? *all : none;
  void* rootc[6] = {a.ids, a.epochs, a.lengths, a.voting_types, a.predicted_boxes, a.observed_boxes};
  void* myc[6] = {mine->ids, mine->epochs, mine->lengths, mine->voting_types, mine->predicted_boxes, mine->observed_boxes};
  return exchange(c, root, det_range, 6, rb, rootc, myc, /*scatter=*/false, reinterpret_cast<cudaStream_t>(cuda_stream));
}

}  // extern "C"
