// bvh_build_device.cu — the BVH2 and its 4-wide collapse built on the device, byte for byte the trees of build_bvh / build_wide_bvh
// (bvh_build.cpp, the specification: the oracle, the parity build and every golden traverse that builder's trees).
//
// Float semantics.  The host builder is compiled with -ffp-contract=off under the default x86-64 floating-point environment (SSE, round to
// nearest, denormals kept).  This translation unit is compiled with -fmad=false -ftz=false -prec-div=true in every flavour (build.py): the
// product flavour's -ftz=true would flush denormal operands even of a comparison, and its approximate division would move bin boundaries.
// Every expression below is the host's, in the host's order: 0.5f * (lo + hi), float(kBins) / (cmax - cmin), the truncating bin index,
// half_area as dx*dy + dy*dz + dz*dx, the cost A_l * n_l + A_r * n_r with its strict <, the leaf test, the wide tree's quantisation.
// Float-to-int conversions follow x86-64's cvttss2si (NaN and out-of-range values give INT_MIN, which the clamps then map to 0), not the
// device's saturating conversion.
//
// Reductions.  A box grows by std::min / std::max, which replace only on a strict <: between +0 and -0 the element that comes first in the
// range's current order wins, a NaN is never selected, +inf never replaces a lo's initial FLT_MAX and -inf never replaces a hi's initial
// -FLT_MAX.  The parallel reductions (node bounds, centroid boxes, the 48 bin boxes of a range) therefore reduce 64-bit keys
// (canonical value, position in the order, sign of a zero): the value clamped to the initial FLT_MAX / -FLT_MAX, -0 ordered as +0, ties
// going to the first position.  The keys are totally ordered, so any reduction order (atomics included) picks the element the sequential
// loop keeps.  Per-triangle boxes, the SAH sweep, the leaf decisions and the wide tree's node boxes are serial per thread, as on the host.
//
// Structure.  Level by level over the active ranges of the triangle order array, one block per range: bounds and centroid box, the 16-bin
// SAH over the three axes, and a stable partition (a block scan over the split flags, left side in place, right side through a scratch copy)
// that reproduces std::stable_partition.  Ranges of up to two triangles become leaves in their parent's block.  Inner nodes are numbered as
// the host's recursion numbers them: its pre-order sorts inner nodes by (first triangle, depth), so a node's index is the number of inner
// nodes starting before its first triangle plus its depth below the topmost node starting there.  The breadth-first top-512 permutation
// follows.  The wide collapse runs level by level over the wide nodes (greedy opening, quantisation), then numbers them in the host's
// pre-order from subtree sizes and applies its own top-512 permutation.
#include "bvh_build_device.h"

#include <algorithm>
#include <cstdint>
#include <vector>

namespace etxb {
namespace {

constexpr int kBins = 16;
constexpr float kFltMax = 3.402823466e+38f;
constexpr uint32_t kTopNodes = 512;
constexpr uint32_t kNone = 0xffffffffu;
constexpr uint32_t kSmallRange = 512;  // ranges up to this many triangles take a one-warp block
constexpr int kScanTile = 1024;        // elements per block of the exclusive scan (256 threads x 4)

struct TriRec {
  float lo[3], hi[3], c[3];
};
struct Range {
  uint32_t begin, end, parent, info;  // info: depth | slot << 8 | force_inner << 9; parent: raw node id (kNone at the root)
};
struct Counters {
  uint32_t big, small, nodes, max_depth;
};

// x86-64 cvttss2si: NaN and values outside the int range convert to INT_MIN
__device__ __forceinline__ int host_int(float x) { return ((x >= -2147483648.0f) && (x < 2147483648.0f)) ? __float2int_rz(x) : int(0x80000000u); }

__device__ __forceinline__ int bin_of(float c, float cmin, float scale) {
  const int b = host_int((c - cmin) * scale);
  return min(kBins - 1, max(0, b));
}

// std::min / std::max as the host's Box::grow applies them
__device__ __forceinline__ float smin(float acc, float v) { return (v < acc) ? v : acc; }
__device__ __forceinline__ float smax(float acc, float v) { return (acc < v) ? v : acc; }

__device__ __forceinline__ uint32_t ordered(float v) {
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unordered(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o); }

// key of `v` at order position `pos` (< 2^31) for a lo (smallest key wins) and for a hi (largest key wins)
__device__ __forceinline__ unsigned long long lo_key(float v, uint32_t pos) {
  uint32_t u = __float_as_uint((v < kFltMax) ? v : kFltMax);
  uint32_t sign = 0;
  if ((u << 1) == 0u) {
    sign = u >> 31;
    u = 0u;
  }
  return (static_cast<unsigned long long>(ordered(__uint_as_float(u))) << 32) | (static_cast<unsigned long long>(pos) << 1) | sign;
}
__device__ __forceinline__ unsigned long long hi_key(float v, uint32_t pos) {
  uint32_t u = __float_as_uint((v > -kFltMax) ? v : -kFltMax);
  uint32_t sign = 0;
  if ((u << 1) == 0u) {
    sign = u >> 31;
    u = 0u;
  }
  return (static_cast<unsigned long long>(ordered(__uint_as_float(u))) << 32) | (static_cast<unsigned long long>(0x7fffffffu - pos) << 1) | sign;
}
__device__ __forceinline__ unsigned long long kmin(unsigned long long a, unsigned long long b) { return (b < a) ? b : a; }
__device__ __forceinline__ unsigned long long kmax(unsigned long long a, unsigned long long b) { return (a < b) ? b : a; }
__device__ __forceinline__ float key_value(unsigned long long k) {
  const float v = unordered(uint32_t(k >> 32));
  return (k & 1ull) ? -0.0f : v;  // the sign bit is set only for a zero
}
// the initial FLT_MAX / -FLT_MAX: after every element's key (positions are below 2^31), with a clear sign bit
__device__ __forceinline__ unsigned long long lo_identity() { return (static_cast<unsigned long long>(ordered(kFltMax)) << 32) | 0xfffffffeull; }
__device__ __forceinline__ unsigned long long hi_identity() { return static_cast<unsigned long long>(ordered(-kFltMax)) << 32; }

struct Box {
  float lo[3], hi[3];
  __device__ void clear() {
    for (int k = 0; k < 3; ++k) {
      lo[k] = kFltMax;
      hi[k] = -kFltMax;
    }
  }
  __device__ void grow(const float* l, const float* h) {
    for (int k = 0; k < 3; ++k) {
      lo[k] = smin(lo[k], l[k]);
      hi[k] = smax(hi[k], h[k]);
    }
  }
  __device__ float half_area() const {
    const float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
    if (dx < 0.0f) return 0.0f;
    return dx * dy + dy * dz + dz * dx;
  }
};

__device__ __forceinline__ int32_t leaf_ref(uint32_t begin, uint32_t count) { return int32_t(~((begin << 2) | (count - 1u))); }

__device__ void link(BvhNode* raw, uint32_t parent, uint32_t slot, const float* lo, const float* hi, int32_t ref) {
  BvhNode& p = raw[parent];
  for (int k = 0; k < 3; ++k) {
    if (slot == 0u) {
      p.lo0[k] = lo[k];
      p.hi0[k] = hi[k];
    } else {
      p.lo1[k] = lo[k];
      p.hi1[k] = hi[k];
    }
  }
  if (slot == 0u)
    p.child0 = ref;
  else
    p.child1 = ref;
}

// ---- per-triangle boxes and centroids ------------------------------------------------------------------------------------------------------
__global__ void k_bvh_triangles(const float* positions, uint32_t pstride, const uint32_t* indices, uint32_t istride, uint32_t n, TriRec* tri, uint32_t* order) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  Box b;
  b.clear();
  for (int k = 0; k < 3; ++k) {
    const float* p = positions + size_t(indices[size_t(t) * istride + k]) * pstride;
    b.grow(p, p);
  }
  TriRec r;
  for (int k = 0; k < 3; ++k) {
    r.lo[k] = b.lo[k];
    r.hi[k] = b.hi[k];
    r.c[k] = 0.5f * (b.lo[k] + b.hi[k]);
  }
  tri[t] = r;
  order[t] = t;
}

struct LevelArgs {
  const TriRec* tri;
  uint32_t* order;
  uint32_t* tmp;
  BvhNode* raw;
  uint2* raw_key;  // (first triangle, depth) of each inner node
  Range* next;
  uint32_t cap;
  Counters* ctr;
};

__device__ void push_child(const LevelArgs& a, uint32_t begin, uint32_t end, uint32_t parent, uint32_t slot, uint32_t depth) {
  const uint32_t count = end - begin;
  if (count <= 2u) {
    // a leaf whatever the rest of build() would compute: its box, in the range's order, and its max_depth
    atomicMax(&a.ctr->max_depth, depth);
    Box b;
    b.clear();
    for (uint32_t i = begin; i < end; ++i) {
      const TriRec& r = a.tri[a.order[i]];
      b.grow(r.lo, r.hi);
    }
    link(a.raw, parent, slot, b.lo, b.hi, leaf_ref(begin, count));
    return;
  }
  const Range r = {begin, end, parent, depth | (slot << 8)};
  if (count > kSmallRange)
    a.next[atomicAdd(&a.ctr->big, 1u)] = r;
  else
    a.next[a.cap - 1u - atomicAdd(&a.ctr->small, 1u)] = r;
}

// build() of one range per block (bvh_build.cpp Builder::build without the recursion: the children are the next level's ranges)
template <int NT>
__global__ void __launch_bounds__(NT) k_bvh_level(LevelArgs a, const Range* ranges) {
  constexpr int NW = NT / 32;
  const Range rg = ranges[blockIdx.x];
  const uint32_t begin = rg.begin, end = rg.end, count = end - begin;
  const uint32_t depth = rg.info & 0xffu;
  const bool force_inner = ((rg.info >> 9) & 1u) != 0u;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;

  __shared__ unsigned long long s_box[12];  // bounds lo, hi; centroid box lo, hi
  __shared__ unsigned long long s_bin[3 * kBins * 6];
  __shared__ uint32_t s_cnt[3 * kBins];
  __shared__ uint32_t s_warp[NW];
  __shared__ float s_cmin[3], s_scale[3];
  __shared__ uint32_t s_axes;     // axes to bin
  __shared__ int s_axis, s_best_bin;  // the SAH split to partition by (s_axis < 0: none)
  __shared__ uint32_t s_left, s_right;

  // ---- bounds and centroid box --------------------------------------------------------------------------------------------------------
  if (tid < 12) s_box[tid] = ((tid % 6u) < 3u) ? lo_identity() : hi_identity();
  unsigned long long k[12];
  for (int j = 0; j < 12; ++j) k[j] = ((j % 6) < 3) ? lo_identity() : hi_identity();
  for (uint32_t i = begin + tid; i < end; i += NT) {
    const TriRec r = a.tri[a.order[i]];
    for (int c = 0; c < 3; ++c) {
      k[c] = kmin(k[c], lo_key(r.lo[c], i));
      k[3 + c] = kmax(k[3 + c], hi_key(r.hi[c], i));
      k[6 + c] = kmin(k[6 + c], lo_key(r.c[c], i));
      k[9 + c] = kmax(k[9 + c], hi_key(r.c[c], i));
    }
  }
  for (int off = 16; off > 0; off >>= 1)
    for (int j = 0; j < 12; ++j) {
      const unsigned long long o = __shfl_xor_sync(0xffffffffu, k[j], off);
      k[j] = ((j % 6) < 3) ? kmin(k[j], o) : kmax(k[j], o);
    }
  __syncthreads();
  if (lane == 0)
    for (int j = 0; j < 12; ++j) {
      if ((j % 6) < 3)
        atomicMin(&s_box[j], k[j]);
      else
        atomicMax(&s_box[j], k[j]);
    }
  __syncthreads();

  Box bounds, cbox;
  for (int c = 0; c < 3; ++c) {
    bounds.lo[c] = key_value(s_box[c]);
    bounds.hi[c] = key_value(s_box[3 + c]);
    cbox.lo[c] = key_value(s_box[6 + c]);
    cbox.hi[c] = key_value(s_box[9 + c]);
  }
  const bool must_split = (count > uint32_t(kBvhMaxLeafTris)) || force_inner;
  uint32_t levels_needed = 1;
  while ((1ull << levels_needed) < count) levels_needed++;
  const bool depth_limited = depth + levels_needed + 2u >= uint32_t(kBvhStackSize);
  // outcome without a partition: 0 leaf (or the single-triangle root), 1 median split in the current order
  const bool sah = (count > 1u) && !depth_limited && !((count <= uint32_t(kBvhMaxLeafTris)) && !force_inner && (count <= 2u));
  if (tid == 0) {
    atomicMax(&a.ctr->max_depth, depth);
    uint32_t axes = 0;
    if (sah)
      for (int c = 0; c < 3; ++c) {
        const float cmin = cbox.lo[c], cmax = cbox.hi[c];
        if (!(cmax > cmin)) continue;
        axes |= 1u << c;
        s_cmin[c] = cmin;
        s_scale[c] = float(kBins) / (cmax - cmin);
      }
    s_axes = axes;
    s_axis = -1;
  }
  __syncthreads();

  // ---- 16 bins per axis -----------------------------------------------------------------------------------------------------------------
  const uint32_t axes = s_axes;
  if (axes != 0u) {
    for (uint32_t j = tid; j < 3u * kBins * 6u; j += NT) s_bin[j] = ((j % 6u) < 3u) ? lo_identity() : hi_identity();
    for (uint32_t j = tid; j < 3u * kBins; j += NT) s_cnt[j] = 0u;
    __syncthreads();
    for (uint32_t i = begin + tid; i < end; i += NT) {
      const TriRec r = a.tri[a.order[i]];
      for (int c = 0; c < 3; ++c) {
        if (!(axes & (1u << c))) continue;
        const int b = bin_of(r.c[c], s_cmin[c], s_scale[c]);
        unsigned long long* bb = s_bin + (c * kBins + b) * 6;
        for (int q = 0; q < 3; ++q) {
          atomicMin(bb + q, lo_key(r.lo[q], i));
          atomicMax(bb + 3 + q, hi_key(r.hi[q], i));
        }
        atomicAdd(&s_cnt[c * kBins + b], 1u);
      }
    }
    __syncthreads();
    if (tid == 0) {
      float best_cost = kFltMax;
      int best_axis = -1, best_bin = -1;
      for (int c = 0; c < 3; ++c) {
        if (!(axes & (1u << c))) continue;
        float right_area[kBins];
        uint32_t right_count[kBins];
        Box acc;
        acc.clear();
        uint32_t cnt = 0;
        for (int b = kBins - 1; b > 0; --b) {
          float l[3], h[3];
          for (int q = 0; q < 3; ++q) {
            l[q] = key_value(s_bin[(c * kBins + b) * 6 + q]);
            h[q] = key_value(s_bin[(c * kBins + b) * 6 + 3 + q]);
          }
          acc.grow(l, h);
          cnt += s_cnt[c * kBins + b];
          right_area[b] = acc.half_area();
          right_count[b] = cnt;
        }
        acc.clear();
        cnt = 0;
        for (int b = 0; b < kBins - 1; ++b) {
          float l[3], h[3];
          for (int q = 0; q < 3; ++q) {
            l[q] = key_value(s_bin[(c * kBins + b) * 6 + q]);
            h[q] = key_value(s_bin[(c * kBins + b) * 6 + 3 + q]);
          }
          acc.grow(l, h);
          cnt += s_cnt[c * kBins + b];
          if (cnt == 0 || right_count[b + 1] == 0) continue;
          const float cost = acc.half_area() * float(cnt) + right_area[b + 1] * float(right_count[b + 1]);
          if (cost < best_cost) {
            best_cost = cost;
            best_axis = c;
            best_bin = b;
          }
        }
      }
      if (best_axis >= 0) {
        const float leaf_cost = bounds.half_area() * float(count);
        if (must_split || (best_cost + bounds.half_area() * 1.0f < leaf_cost)) {
          s_axis = best_axis;
          s_best_bin = best_bin;
        }
      }
      s_left = 0u;
      s_right = 0u;
    }
    __syncthreads();
  }

  // ---- stable partition by the SAH split --------------------------------------------------------------------------------------------------
  uint32_t mid = begin;
  bool split_found = false;
  const int axis = s_axis;
  if (axis >= 0) {
    const int best_bin = s_best_bin;
    const float cmin = s_cmin[axis], scale = s_scale[axis];
    for (uint32_t i0 = begin; i0 < end; i0 += NT) {
      const uint32_t i = i0 + tid;
      const bool valid = i < end;
      const uint32_t t = valid ? a.order[i] : 0u;
      const bool left = valid && (bin_of(a.tri[t].c[axis], cmin, scale) <= best_bin);
      const uint32_t ballot = __ballot_sync(0xffffffffu, left);
      if (lane == 0) s_warp[warp] = __popc(ballot);
      __syncthreads();
      uint32_t before = 0, total = 0;
      for (int w = 0; w < NW; ++w) {
        if (w < int(warp)) before += s_warp[w];
        total += s_warp[w];
      }
      const uint32_t lrank = before + __popc(ballot & ((1u << lane) - 1u));
      if (valid) {
        if (left)
          a.order[begin + s_left + lrank] = t;  // at or before position i, which every thread of the block has read
        else
          a.tmp[begin + s_right + (i - i0) - lrank] = t;
      }
      __syncthreads();
      if (tid == 0) {
        s_left += total;
        s_right += min(uint32_t(NT), end - i0) - total;
      }
      __syncthreads();
    }
    mid = begin + s_left;
    for (uint32_t j = tid; j < s_right; j += NT) a.order[mid + j] = a.tmp[begin + j];
    __syncthreads();
    split_found = (mid > begin) && (mid < end);
  }
  if (tid != 0) return;
  if ((count > 1u) && !split_found && must_split) {
    // depth limit, or degenerate centroids: median split in the current order
    mid = begin + count / 2u;
    split_found = (mid > begin) && (mid < end);
  }

  if (!split_found) {
    if (force_inner) {
      // single triangle at the root: inner node with the leaf in child0 and an empty box in child1
      const uint32_t raw = atomicAdd(&a.ctr->nodes, 1u);
      a.raw_key[raw] = make_uint2(begin, depth);
      BvhNode n = {};
      for (int c = 0; c < 3; ++c) {
        n.lo0[c] = bounds.lo[c];
        n.hi0[c] = bounds.hi[c];
        n.lo1[c] = kFltMax;
        n.hi1[c] = -kFltMax;
      }
      n.child0 = leaf_ref(begin, count);
      n.child1 = n.child0;
      a.raw[raw] = n;
      return;
    }
    link(a.raw, rg.parent, (rg.info >> 8) & 1u, bounds.lo, bounds.hi, leaf_ref(begin, count));
    return;
  }
  const uint32_t raw = atomicAdd(&a.ctr->nodes, 1u);
  a.raw_key[raw] = make_uint2(begin, depth);
  if (rg.parent != kNone) link(a.raw, rg.parent, (rg.info >> 8) & 1u, bounds.lo, bounds.hi, int32_t(raw));
  push_child(a, begin, mid, raw, 0u, depth + 1u);
  push_child(a, mid, end, raw, 1u, depth + 1u);
}

// ---- exclusive scan (in place) ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_bvh_scan_tiles(uint32_t* data, uint32_t n, uint32_t* sums) {
  __shared__ uint32_t s[256];
  const uint32_t base = blockIdx.x * kScanTile + threadIdx.x * 4u;
  uint32_t v[4], sum = 0;
  for (int j = 0; j < 4; ++j) {
    v[j] = (base + j < n) ? data[base + j] : 0u;
    sum += v[j];
  }
  s[threadIdx.x] = sum;
  __syncthreads();
  for (uint32_t off = 1; off < 256u; off <<= 1) {
    const uint32_t add = (threadIdx.x >= off) ? s[threadIdx.x - off] : 0u;
    __syncthreads();
    s[threadIdx.x] += add;
    __syncthreads();
  }
  uint32_t run = s[threadIdx.x] - sum;
  for (int j = 0; j < 4; ++j) {
    if (base + j < n) data[base + j] = run;
    run += v[j];
  }
  if (threadIdx.x == 255u) sums[blockIdx.x] = s[255];
}
__global__ void k_bvh_scan_add(uint32_t* data, uint32_t n, const uint32_t* offsets) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) data[i] += offsets[i / kScanTile];
}

uint32_t blocks(uint32_t n, uint32_t per) { return (n + per - 1u) / per; }

// scratch for the tile sums of every recursion level of a scan over n elements
size_t scan_scratch(uint32_t n) {
  size_t s = 0;
  while (n > 1u) {
    n = blocks(n, kScanTile);
    s += n;
  }
  return s + 1;
}
void scan_exclusive(uint32_t* data, uint32_t n, uint32_t* scratch, cudaStream_t stream) {
  if (n == 0u) return;
  const uint32_t nb = blocks(n, kScanTile);
  k_bvh_scan_tiles<<<nb, 256, 0, stream>>>(data, n, scratch);
  if (nb == 1u) return;
  scan_exclusive(scratch, nb, scratch + nb, stream);
  k_bvh_scan_add<<<blocks(n, 256), 256, 0, stream>>>(data, n, scratch);
}

// ---- numbering ----------------------------------------------------------------------------------------------------------------------------
__global__ void k_bvh_count_starts(const uint2* raw_key, uint32_t nodes, uint32_t* starts, uint32_t* top_depth) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nodes) return;
  atomicAdd(&starts[raw_key[r].x], 1u);
  atomicMin(&top_depth[raw_key[r].x], raw_key[r].y);
}
// host pre-order index of every inner node: inner nodes starting before its first triangle, then its place in the left chain starting there
__global__ void k_bvh_preorder(const uint2* raw_key, uint32_t nodes, const uint32_t* starts_scanned, const uint32_t* top_depth, uint32_t* pre) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nodes) return;
  const uint2 k = raw_key[r];
  pre[r] = starts_scanned[k.x] + (k.y - top_depth[k.x]);
}
__global__ void k_bvh_place(const BvhNode* raw, uint32_t nodes, const uint32_t* pre, BvhNode* out) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= nodes) return;
  BvhNode n = raw[r];
  if (n.child0 >= 0) n.child0 = int32_t(pre[n.child0]);
  if (n.child1 >= 0) n.child1 = int32_t(pre[n.child1]);
  n.pad0 = n.pad1 = 0u;
  out[pre[r]] = n;
}

__device__ __forceinline__ int children(const BvhNode& n, int32_t* kids) {
  kids[0] = n.child0;
  kids[1] = n.child1;
  return 2;
}
__device__ __forceinline__ int children(const WideNode& n, int32_t* kids) {
  for (int k = 0; k < n.count; ++k) kids[k] = n.child[k];
  return n.count;
}
__device__ __forceinline__ void set_children(BvhNode& n, const int32_t* kids) {
  n.child0 = kids[0];
  n.child1 = kids[1];
}
__device__ __forceinline__ void set_children(WideNode& n, const int32_t* kids) {
  for (int k = 0; k < n.count; ++k) n.child[k] = kids[k];
}

// the breadth-first top of the tree (bvh_build.cpp: the kTopNodes loop); new_index holds kNone for every node (one thread)
template <class Node>
__global__ void k_bvh_top(const Node* nodes, uint32_t n, uint32_t* new_index, uint32_t* queue, uint32_t* top_count) {
  uint32_t size = 1;
  queue[0] = 0u;
  new_index[0] = 0u;
  for (uint32_t head = 0; (head < size) && (size < kTopNodes); ++head) {
    int32_t kids[4];
    const int m = children(nodes[queue[head]], kids);
    for (int j = 0; j < m; ++j) {
      const int32_t c = kids[j];
      if ((c >= 0) && (new_index[uint32_t(c)] == kNone) && (size < kTopNodes)) {
        new_index[uint32_t(c)] = size;
        queue[size++] = uint32_t(c);
      }
    }
  }
  *top_count = size;
}
__global__ void k_bvh_top_flags(const uint32_t* new_index, uint32_t n, uint32_t* flags) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) flags[k] = (new_index[k] != kNone) ? 1u : 0u;
}
__device__ __forceinline__ uint32_t final_index(const uint32_t* new_index, const uint32_t* top_before, uint32_t top_count, uint32_t k) {
  const uint32_t t = new_index[k];
  return (t != kNone) ? t : top_count + (k - top_before[k]);
}
template <class Node>
__global__ void k_bvh_reorder(const Node* pre_nodes, uint32_t n, const uint32_t* new_index, const uint32_t* top_before, const uint32_t* top_count, Node* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t tc = *top_count;
  Node nd = pre_nodes[k];
  int32_t kids[4];
  const int m = children(nd, kids);
  for (int j = 0; j < m; ++j)
    if (kids[j] >= 0) kids[j] = int32_t(final_index(new_index, top_before, tc, uint32_t(kids[j])));
  set_children(nd, kids);
  out[final_index(new_index, top_before, tc, k)] = nd;
}

__global__ void k_bvh_leaves(const float* positions, uint32_t pstride, const uint32_t* indices, uint32_t istride, const uint32_t* order, uint32_t n, F4* tri_pos, uint32_t* tri_index) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const uint32_t t = order[s];
  if (tri_index) tri_index[s] = t;
  for (int k = 0; k < 3; ++k) {
    const float* p = positions + size_t(indices[size_t(t) * istride + k]) * pstride;
    tri_pos[size_t(s) * 3 + k] = F4{p[0], p[1], p[2], (k == 0) ? __uint_as_float(t) : 0.0f};
  }
}

// ---- wide collapse ------------------------------------------------------------------------------------------------------------------------
struct WideChild {
  float lo[3], hi[3];
  int32_t ref;
};
__device__ float box_area(const WideChild& c) {
  const float dx = c.hi[0] - c.lo[0], dy = c.hi[1] - c.lo[1], dz = c.hi[2] - c.lo[2];
  return dx * dy + dy * dz + dz * dx;
}
__device__ void children_of(const BvhNode& n, WideChild& a, WideChild& b) {
  for (int k = 0; k < 3; ++k) {
    a.lo[k] = n.lo0[k];
    a.hi[k] = n.hi0[k];
    b.lo[k] = n.lo1[k];
    b.hi[k] = n.hi1[k];
  }
  a.ref = n.child0;
  b.ref = n.child1;
}
// glibc frexpf's exponent: 0 for zero, infinities and NaN
__device__ int frexp_exponent(float x) {
  const uint32_t u = __float_as_uint(x);
  const uint32_t e = (u >> 23) & 0xffu;
  if (e == 0xffu) return 0;
  if (e == 0u) {
    const uint32_t m = u & 0x7fffffu;
    return (m == 0u) ? 0 : (32 - __clz(m)) - 149;
  }
  return int(e) - 126;
}

struct WideItem {
  int32_t bvh2;          // the BVH2 inner node this wide node opens
  uint32_t stack_above;  // stack entries waiting above it
};

// WideBuilder::build of one wide node per thread, its inner children appended to the next level (raw ids are allocation order)
__global__ void k_wide_level(const BvhNode* bvh, WideItem* items, uint32_t first, uint32_t last, WideNode* raw, uint32_t* counter, uint32_t* max_stack) {
  const uint32_t w = first + blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= last) return;
  const WideItem item = items[w];
  WideChild kids[4];
  int count = 2;
  children_of(bvh[item.bvh2], kids[0], kids[1]);
  if (kids[1].ref == kids[0].ref) count = 1;
  while (count < 4) {
    int best = -1;
    float best_area = -1.0f;
    for (int k = 0; k < count; ++k) {
      if ((kids[k].ref >= 0) && (box_area(kids[k]) > best_area)) {
        best_area = box_area(kids[k]);
        best = k;
      }
    }
    if (best < 0) break;
    WideChild a, b;
    children_of(bvh[kids[best].ref], a, b);
    kids[best] = a;
    kids[count++] = b;
  }
  WideNode n = {};
  for (int a = 0; a < 3; ++a) {
    float lo = kids[0].lo[a], hi = kids[0].hi[a];
    for (int k = 1; k < count; ++k) {
      lo = smin(lo, kids[k].lo[a]);
      hi = smax(hi, kids[k].hi[a]);
    }
    n.origin[a] = lo;
    const float d = hi - lo;
    const float extent = (d < 1.0e-30f) ? 1.0e-30f : d;  // std::max(d, 1e-30f)
    int e = frexp_exponent(extent / 255.0f);
    e = max(-126, min(127, e));
    n.exp[a] = uint8_t(e + 127);
    const float step = __uint_as_float(uint32_t(e + 127) << 23);  // ldexp(1.0f, e)
    for (int k = 0; k < count; ++k) {
      int ql = host_int(floorf((kids[k].lo[a] - lo) / step));
      int qh = host_int(ceilf((kids[k].hi[a] - lo) / step));
      ql = max(0, min(255, ql));
      qh = max(0, min(255, qh));
      while ((ql > 0) && (lo + float(ql) * step > kids[k].lo[a])) ql--;
      while ((qh < 255) && (lo + float(qh) * step < kids[k].hi[a])) qh++;
      n.qlo[k][a] = uint8_t(ql);
      n.qhi[k][a] = uint8_t(qh);
    }
  }
  n.count = uint8_t(count);
  const uint32_t below = item.stack_above + uint32_t(count - 1);
  atomicMax(max_stack, below);
  for (int k = 0; k < count; ++k) {
    if (kids[k].ref >= 0) {
      const uint32_t id = atomicAdd(counter, 1u);
      items[id] = WideItem{kids[k].ref, below};
      n.child[k] = int32_t(id);
    } else {
      n.child[k] = kids[k].ref;
    }
  }
  for (int k = count; k < 4; ++k) n.child[k] = int32_t(0x80000000u);
  raw[w] = n;
}
__global__ void k_wide_sizes(const WideNode* raw, uint32_t first, uint32_t last, uint32_t* size) {
  const uint32_t w = first + blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= last) return;
  uint32_t s = 1;
  for (int k = 0; k < raw[w].count; ++k)
    if (raw[w].child[k] >= 0) s += size[raw[w].child[k]];
  size[w] = s;
}
__global__ void k_wide_preorder(const WideNode* raw, uint32_t first, uint32_t last, const uint32_t* size, uint32_t* pre) {
  const uint32_t w = first + blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= last) return;
  uint32_t run = pre[w] + 1u;
  for (int k = 0; k < raw[w].count; ++k) {
    const int32_t c = raw[w].child[k];
    if (c >= 0) {
      pre[c] = run;
      run += size[c];
    }
  }
}
__global__ void k_wide_place(const WideNode* raw, uint32_t n, const uint32_t* pre, WideNode* out) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n) return;
  WideNode nd = raw[w];
  for (int k = 0; k < nd.count; ++k)
    if (nd.child[k] >= 0) nd.child[k] = int32_t(pre[nd.child[k]]);
  out[pre[w]] = nd;
}

// device allocations released when the build returns
struct Scratch {
  std::vector<void*> ptrs;
  ~Scratch() {
    for (void* p : ptrs) cudaFree(p);
  }
  template <class T>
  cudaError_t get(T** p, size_t n) {
    *p = nullptr;
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), std::max<size_t>(n, 1) * sizeof(T));
    if (e == cudaSuccess) ptrs.push_back(*p);
    return e;
  }
};

#define BVH_TRY(call)                       \
  do {                                      \
    cudaError_t e__ = (call);               \
    if (e__ != cudaSuccess) return e__;     \
  } while (0)

// the breadth-first top-512 permutation of a tree whose n nodes are in the host builder's pre-order
template <class Node>
cudaError_t top_reorder(const Node* pre_nodes, uint32_t n, Node* out, Scratch& s, cudaStream_t stream) {
  uint32_t *new_index, *flags, *queue, *top_count, *sums;
  BVH_TRY(s.get(&new_index, n));
  BVH_TRY(s.get(&flags, n));
  BVH_TRY(s.get(&queue, kTopNodes));
  BVH_TRY(s.get(&top_count, 1));
  BVH_TRY(s.get(&sums, scan_scratch(n)));
  BVH_TRY(cudaMemsetAsync(new_index, 0xff, size_t(n) * 4, stream));
  k_bvh_top<Node><<<1, 1, 0, stream>>>(pre_nodes, n, new_index, queue, top_count);
  k_bvh_top_flags<<<blocks(n, 256), 256, 0, stream>>>(new_index, n, flags);
  scan_exclusive(flags, n, sums, stream);
  k_bvh_reorder<Node><<<blocks(n, 256), 256, 0, stream>>>(pre_nodes, n, new_index, flags, top_count, out);
  return cudaGetLastError();
}

cudaError_t build_bvh_impl(const float* positions, uint32_t pstride, const uint32_t* indices, uint32_t istride, uint32_t n, bool want_tri_index, cudaStream_t stream,
  DeviceBvhOut& out, Scratch& s) {
  if (n == 0u) {
    // the zero-triangle tree of build_bvh: one inner node whose children are an empty leaf that is never reached
    BvhNode root = {};
    for (int k = 0; k < 3; ++k) {
      root.lo0[k] = root.lo1[k] = kFltMax;
      root.hi0[k] = root.hi1[k] = -kFltMax;
    }
    root.child0 = root.child1 = int32_t(~0u);
    const F4 zero[3] = {};
    const uint32_t none = kNone;
    BVH_TRY(cudaMemcpyAsync(out.nodes, &root, sizeof(root), cudaMemcpyHostToDevice, stream));
    BVH_TRY(cudaMemcpyAsync(out.tri_pos, zero, sizeof(zero), cudaMemcpyHostToDevice, stream));
    if (out.tri_index) BVH_TRY(cudaMemcpyAsync(out.tri_index, &none, 4, cudaMemcpyHostToDevice, stream));
    BVH_TRY(cudaStreamSynchronize(stream));
    out.node_count = 1;
    out.slot_count = 1;
    out.max_depth = 1;
    return cudaSuccess;
  }
  TriRec* tri;
  uint32_t *order, *tmp, *pre, *starts, *top_depth, *sums;
  BvhNode *raw, *pre_nodes;
  uint2* raw_key;
  Range *cur, *next;
  Counters* ctr;
  BVH_TRY(s.get(&tri, n));
  BVH_TRY(s.get(&order, n));
  BVH_TRY(s.get(&tmp, n));
  BVH_TRY(s.get(&raw, n));
  BVH_TRY(s.get(&raw_key, n));
  BVH_TRY(s.get(&cur, n));
  BVH_TRY(s.get(&next, n));
  BVH_TRY(s.get(&ctr, 1));
  k_bvh_triangles<<<blocks(n, 256), 256, 0, stream>>>(positions, pstride, indices, istride, n, tri, order);
  BVH_TRY(cudaMemsetAsync(ctr, 0, sizeof(Counters), stream));
  const Range root = {0u, n, kNone, 1u | (1u << 9)};
  BVH_TRY(cudaMemcpyAsync(cur, &root, sizeof(root), cudaMemcpyHostToDevice, stream));
  uint32_t big = (n > kSmallRange) ? 1u : 0u, small = 1u - big;
  if (small) BVH_TRY(cudaMemcpyAsync(cur + (n - 1u), &root, sizeof(root), cudaMemcpyHostToDevice, stream));
  Counters c = {};
  while (big + small > 0u) {
    BVH_TRY(cudaMemsetAsync(ctr, 0, 2 * sizeof(uint32_t), stream));  // the next level's range counts (node count and max_depth accumulate)
    const LevelArgs a = {tri, order, tmp, raw, raw_key, next, n, ctr};
    if (big) k_bvh_level<256><<<big, 256, 0, stream>>>(a, cur);
    if (small) k_bvh_level<32><<<small, 32, 0, stream>>>(a, cur + (n - small));
    BVH_TRY(cudaGetLastError());
    BVH_TRY(cudaMemcpyAsync(&c, ctr, sizeof(c), cudaMemcpyDeviceToHost, stream));
    BVH_TRY(cudaStreamSynchronize(stream));
    big = c.big;
    small = c.small;
    std::swap(cur, next);
  }
  const uint32_t nodes = c.nodes;
  BVH_TRY(s.get(&pre, nodes));
  BVH_TRY(s.get(&pre_nodes, nodes));
  BVH_TRY(s.get(&starts, n));
  BVH_TRY(s.get(&top_depth, n));
  BVH_TRY(s.get(&sums, scan_scratch(n)));
  BVH_TRY(cudaMemsetAsync(starts, 0, size_t(n) * 4, stream));
  BVH_TRY(cudaMemsetAsync(top_depth, 0xff, size_t(n) * 4, stream));
  k_bvh_count_starts<<<blocks(nodes, 256), 256, 0, stream>>>(raw_key, nodes, starts, top_depth);
  scan_exclusive(starts, n, sums, stream);
  k_bvh_preorder<<<blocks(nodes, 256), 256, 0, stream>>>(raw_key, nodes, starts, top_depth, pre);
  k_bvh_place<<<blocks(nodes, 256), 256, 0, stream>>>(raw, nodes, pre, pre_nodes);
  BVH_TRY(top_reorder(pre_nodes, nodes, out.nodes, s, stream));
  k_bvh_leaves<<<blocks(n, 256), 256, 0, stream>>>(positions, pstride, indices, istride, order, n, out.tri_pos, out.tri_index);
  BVH_TRY(cudaGetLastError());
  BVH_TRY(cudaStreamSynchronize(stream));
  out.node_count = nodes;
  out.slot_count = n;
  out.max_depth = c.max_depth;
  return cudaSuccess;
}

cudaError_t build_wide_impl(const BvhNode* bvh, uint32_t bvh_nodes, cudaStream_t stream, WideNode* out, uint32_t* out_count, uint32_t* max_stack, Scratch& s) {
  WideItem* items;
  WideNode *raw, *pre_nodes;
  uint32_t *counter, *size, *pre;
  BVH_TRY(s.get(&items, bvh_nodes));
  BVH_TRY(s.get(&raw, bvh_nodes));
  BVH_TRY(s.get(&counter, 2));  // next raw id, max_stack
  const WideItem root = {0, 0u};
  const uint32_t init[2] = {1u, 0u};
  BVH_TRY(cudaMemcpyAsync(items, &root, sizeof(root), cudaMemcpyHostToDevice, stream));
  BVH_TRY(cudaMemcpyAsync(counter, init, sizeof(init), cudaMemcpyHostToDevice, stream));
  std::vector<uint32_t> level = {0u, 1u};  // raw ids of level L: [level[L], level[L + 1])
  uint32_t got[2] = {1u, 0u};
  for (;;) {
    const uint32_t first = level[level.size() - 2], last = level.back();
    k_wide_level<<<blocks(last - first, 128), 128, 0, stream>>>(bvh, items, first, last, raw, counter, counter + 1);
    BVH_TRY(cudaGetLastError());
    BVH_TRY(cudaMemcpyAsync(got, counter, sizeof(got), cudaMemcpyDeviceToHost, stream));
    BVH_TRY(cudaStreamSynchronize(stream));
    if (got[0] == last) break;
    level.push_back(got[0]);
  }
  const uint32_t n = got[0];
  BVH_TRY(s.get(&size, n));
  BVH_TRY(s.get(&pre, n));
  BVH_TRY(s.get(&pre_nodes, n));
  for (size_t L = level.size() - 1; L-- > 0;)
    k_wide_sizes<<<blocks(level[L + 1] - level[L], 256), 256, 0, stream>>>(raw, level[L], level[L + 1], size);
  BVH_TRY(cudaMemsetAsync(pre, 0, 4, stream));
  for (size_t L = 0; L + 1 < level.size(); ++L)
    k_wide_preorder<<<blocks(level[L + 1] - level[L], 256), 256, 0, stream>>>(raw, level[L], level[L + 1], size, pre);
  k_wide_place<<<blocks(n, 256), 256, 0, stream>>>(raw, n, pre, pre_nodes);
  BVH_TRY(top_reorder(pre_nodes, n, out, s, stream));
  BVH_TRY(cudaStreamSynchronize(stream));
  *out_count = n;
  *max_stack = got[1];
  return cudaSuccess;
}

}  // namespace

cudaError_t build_bvh_device(const float* positions, uint32_t position_stride_bytes, const uint32_t* indices, uint32_t index_stride_bytes, uint32_t tri_count,
  bool want_tri_index, cudaStream_t stream, DeviceBvhOut& out) {
  out = DeviceBvhOut{};
  // inner nodes: at most tri_count - 1, or the one root of an empty or single-triangle mesh
  const size_t cap = std::max<uint32_t>(tri_count, 1u);
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&out.nodes), cap * sizeof(BvhNode));
  if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void**>(&out.tri_pos), cap * 3 * sizeof(F4));
  if ((e == cudaSuccess) && want_tri_index) e = cudaMalloc(reinterpret_cast<void**>(&out.tri_index), cap * sizeof(uint32_t));
  if (e == cudaSuccess) {
    Scratch s;
    e = build_bvh_impl(positions, position_stride_bytes / 4u, indices, index_stride_bytes / 4u, tri_count, want_tri_index, stream, out, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);  // the scratch is freed after the last kernel that reads it
  }
  if (e != cudaSuccess) {
    cudaFree(out.nodes);
    cudaFree(out.tri_pos);
    cudaFree(out.tri_index);
    out = DeviceBvhOut{};
  }
  return e;
}

cudaError_t build_wide_bvh_device(const BvhNode* nodes, uint32_t node_count, cudaStream_t stream, WideNode** out, uint32_t* out_count, uint32_t* max_stack) {
  *out = nullptr;
  *out_count = 0;
  *max_stack = 0;
  // a wide node per BVH2 inner node at most
  cudaError_t e = cudaMalloc(reinterpret_cast<void**>(out), std::max<size_t>(node_count, 1) * sizeof(WideNode));
  if (e == cudaSuccess) {
    Scratch s;
    e = build_wide_impl(nodes, node_count, stream, *out, out_count, max_stack, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
  }
  if (e != cudaSuccess) {
    cudaFree(*out);
    *out = nullptr;
    *out_count = 0;
  }
  return e;
}

}  // namespace etxb
