// mesher.h -- state shared by mesh.cu (marching cubes + weld) and simplify.cu
#pragma once
#include <vector>

#include "common.cuh"

// persistent result of ign_mesh_begin*
struct ign_mesher {
  ign_ctx* ctx;
  uint64_t K;            // dense labels 1..K
  uint64_t T, U;         // triangles, unique vertices
  uint64_t* d_uniq_vkeys;  // [U]
  uint32_t* d_faces;       // [3T] label-local vertex indices
  bool pooled;             // buffers live in ctx->mesh_pool
  // after ign_mesh_simplify: positions are float3 (physical units, no
  // voxel-centre shift) in d_pos_f; d_faces / offsets describe the simplified meshes
  bool simplified;
  float* d_pos_f;
  float res[3];
  int simp_factor;
  float simp_max_error;
  uint32_t simp_counters[17];  // ign_mesh_simplify_counters
  std::vector<uint64_t> ids;       // original label of dense id i+1
  std::vector<uint32_t> tri_off;   // [K+2]
  std::vector<uint32_t> vert_off;  // [K+2]
  std::vector<uint64_t> present;   // original ids with at least one triangle
};

