// bvh_build_device.h — the device builders of the BVH2 and of its 4-wide collapse: node for node the trees of build_bvh / build_wide_bvh.
#pragma once
#include <cuda_runtime.h>

#include "bvh.h"

namespace etxb {

// Device arrays allocated by build_bvh_device with cudaMalloc; the caller owns (and frees) them.
struct DeviceBvhOut {
  BvhNode* nodes = nullptr;
  uint32_t node_count = 0;
  F4* tri_pos = nullptr;         // 3 entries per leaf slot
  uint32_t* tri_index = nullptr; // leaf slot -> triangle (only when requested)
  uint32_t slot_count = 0;
  uint32_t max_depth = 0;
};

// The same tree as build_bvh over the same vertex / triangle records (positions: first 3 floats of each vertex record; indices: first 3 uint32
// of each triangle record; strides in bytes), all on `stream`.  Scratch is freed before it returns; it synchronises `stream`.
cudaError_t build_bvh_device(const float* positions, uint32_t position_stride_bytes, const uint32_t* indices, uint32_t index_stride_bytes, uint32_t tri_count,
  bool want_tri_index, cudaStream_t stream, DeviceBvhOut& out);

// The same tree as build_wide_bvh from the device BVH2 `nodes`; *out is cudaMalloc'd (the caller frees it).  Synchronises `stream`.
cudaError_t build_wide_bvh_device(const BvhNode* nodes, uint32_t node_count, cudaStream_t stream, WideNode** out, uint32_t* out_count, uint32_t* max_stack);

}  // namespace etxb
