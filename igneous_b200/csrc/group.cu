// group.cu -- the one collective of the hot path: an NCCL all-gather of every
// rank's CCL boundary planes over NVLink / NVSwitch (replaces the face files of
// igneous/tasks/image/ccl.py:177-194 and their re-download in :245-268).
// NCCL is resolved with dlopen at first use; nothing links against it.
#include <dlfcn.h>

#include "group.h"

namespace {

typedef struct { char internal[128]; } nccl_uid_t;
typedef void* nccl_comm_t;
typedef int (*fn_get_uid)(nccl_uid_t*);
typedef int (*fn_init_rank)(nccl_comm_t*, int, nccl_uid_t, int);
typedef int (*fn_allgather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t);
typedef int (*fn_destroy)(nccl_comm_t);
typedef const char* (*fn_errstr)(int);

struct NcclApi {
  void* handle = nullptr;
  fn_get_uid get_uid = nullptr;
  fn_init_rank init_rank = nullptr;
  fn_allgather allgather = nullptr;
  fn_destroy destroy = nullptr;
  fn_errstr errstr = nullptr;
};

NcclApi g_nccl;

int load_nccl() {
  if (g_nccl.handle) return IGN_OK;
  const char* names[] = {"libnccl.so.2", "libnccl.so"};
  void* h = nullptr;
  for (const char* n : names) {
    h = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
    if (h) break;
  }
  if (!h) {
    ign::set_error("cannot dlopen libnccl.so.2: %s", dlerror());
    return IGN_ERR_NCCL;
  }
  g_nccl.get_uid = (fn_get_uid)dlsym(h, "ncclGetUniqueId");
  g_nccl.init_rank = (fn_init_rank)dlsym(h, "ncclCommInitRank");
  g_nccl.allgather = (fn_allgather)dlsym(h, "ncclAllGather");
  g_nccl.destroy = (fn_destroy)dlsym(h, "ncclCommDestroy");
  g_nccl.errstr = (fn_errstr)dlsym(h, "ncclGetErrorString");
  if (!g_nccl.get_uid || !g_nccl.init_rank || !g_nccl.allgather || !g_nccl.destroy) {
    ign::set_error("libnccl is missing required symbols");
    return IGN_ERR_NCCL;
  }
  g_nccl.handle = h;
  return IGN_OK;
}

int nccl_fail(const char* what, int rc) {
  ign::set_error("%s failed: %s", what, g_nccl.errstr ? g_nccl.errstr(rc) : "nccl error");
  return IGN_ERR_NCCL;
}

}  // namespace

using namespace ign;

extern "C" {

int ign_group_unique_id(void* id128) {
  IGN_REQUIRE(id128, IGN_ERR_INVALID, "null argument");
  IGN_TRY(load_nccl());
  nccl_uid_t uid;
  const int rc = g_nccl.get_uid(&uid);
  if (rc != 0) return nccl_fail("ncclGetUniqueId", rc);
  memcpy(id128, &uid, sizeof(uid));
  return IGN_OK;
}

int ign_group_init(ign_ctx* ctx, int rank, int nranks, const void* id128, ign_group** out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(id128 && out && nranks >= 1 && rank >= 0 && rank < nranks, IGN_ERR_INVALID, "bad group argument");
  IGN_TRY(load_nccl());
  nccl_uid_t uid;
  memcpy(&uid, id128, sizeof(uid));
  ign_group* g = new ign_group();
  g->ctx = ctx;
  g->rank = rank;
  g->nranks = nranks;
  g->d_send = g->d_recv = nullptr;
  g->send_bytes = g->recv_bytes = 0;
  const int rc = g_nccl.init_rank((nccl_comm_t*)&g->comm, nranks, uid, rank);
  if (rc != 0) {
    delete g;
    return nccl_fail("ncclCommInitRank", rc);
  }
  *out = g;
  return IGN_OK;
}

int ign_group_destroy(ign_group* g) {
  if (!g) return IGN_OK;
  if (g_nccl.destroy) g_nccl.destroy((nccl_comm_t)g->comm);
  cudaSetDevice(g->ctx->device);
  if (g->d_send) cudaFree(g->d_send);
  if (g->d_recv) cudaFree(g->d_recv);
  delete g;
  return IGN_OK;
}

int ign_group_allgather(ign_group* g, const void* send_dev, uint64_t bytes, void* recv_dev) {
  IGN_REQUIRE(g && send_dev && recv_dev, IGN_ERR_INVALID, "null argument");
  IGN_TRY(activate(g->ctx));
  const int rc = g_nccl.allgather(send_dev, recv_dev, (size_t)bytes, /*ncclUint8*/ 1, (nccl_comm_t)g->comm, g->ctx->stream);
  if (rc != 0) return nccl_fail("ncclAllGather", rc);
  g->ctx->launches++;  // NCCL's kernel
  return IGN_OK;
}

}  // extern "C"
