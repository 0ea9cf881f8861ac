// group.h -- the NCCL communicator of one rank (group.cu) as seen by ccl.cu
#pragma once
#include "common.cuh"

struct ign_group {
  ign_ctx* ctx;
  void* comm;  // ncclComm_t
  int rank, nranks;
  // grow-only device buffers of ign_ccl6_sharded_dev: this rank's plane record, every rank's records
  char *d_send, *d_recv;
  size_t send_bytes, recv_bytes;
};
