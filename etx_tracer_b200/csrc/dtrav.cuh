// dtrav.cuh — the traversal kernels: persistent warps, the top of the BVH staged in shared memory by TMA, lane refill.
//
// Replaces the reference's ray caster for the wavefront stages (Embree rtcIntersect1 behind Raytracing::trace / trace_transmittance,
// sources/etx/rt/rt.cxx:250-279, 428-466, 468-579).  On the thread-per-ray kernel a warp lives as long as its longest ray, so most of its
// lanes idle, and every node fetch is a dependent trip to L1 / L2.  Here:
//   * the first kNodeletNodes BVH nodes are the top ~9 levels in breadth-first order (bvh_build.cpp; the rest stays depth-first), the ones every ray walks through;
//     each CTA copies them once into shared memory with one cp.async.bulk (TMA bulk copy, completion on an mbarrier) — 32 KB per CTA, the
//     kernel is persistent, so the copy is amortised over thousands of rays;
//   * rays come from a compacted list (queue of path ids / SoA shadow segments) through a shared cursor: a warp refills its idle lanes with
//     fresh rays (ballot + one atomic per refill) as soon as fewer than kRefillLanes of its 32 lanes are still traversing, instead of waiting
//     for its longest ray (Aila & Laine's persistent while-while with dynamic fetch, adapted to a queue that stays on the device);
//   * the per-ray traversal is the SAME near-first stack walk as bvh.h's traverse() — same nodes, same candidate order, same float operations.
// The product build's k_shadow_resolve runs these walks.
#pragma once
#include "dtrace.cuh"

namespace etxb {

constexpr uint32_t kNodeletNodes = 512u;  // 32 KB: the top of the tree in breadth-first order
constexpr uint32_t kRefillLanes = 20u;    // refill when fewer lanes than this are still traversing

// ---- TMA bulk copy + mbarrier (PTX ISA 8.x, sm_90+) ------------------------------------------------------------------------------------------
DEV uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
DEV void mbar_init(uint64_t* bar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(arrivals) : "memory");
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
DEV void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
DEV void bulk_copy_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes),
               "r"(smem_u32(bar))
               : "memory");
}
DEV void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
    "{\n"
    ".reg .pred P1;\n"
    "LAB_WAIT:\n"
    "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
    "@P1 bra DONE;\n"
    "bra LAB_WAIT;\n"
    "DONE:\n"
    "}\n" ::"r"(smem_u32(bar)),
    "r"(phase)
    : "memory");
}

// one CTA-wide staging of the first `staged` nodes; returns how many are in shared memory
DEV uint32_t nodelet_stage(BvhNode* s_nodes, uint64_t* s_bar, const BvhNode* g_nodes, uint32_t node_count) {
  const uint32_t staged = umin(node_count, kNodeletNodes);
  if (threadIdx.x == 0) mbar_init(s_bar, 1u);
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(s_bar, staged * uint32_t(sizeof(BvhNode)));
    bulk_copy_g2s(s_nodes, g_nodes, staged * uint32_t(sizeof(BvhNode)), s_bar);
  }
  mbar_wait(s_bar, 0u);
  return staged;
}

struct StagedNodes {
  const BvhNode* s_nodes;
  const BvhNode* g_nodes;
  uint32_t staged;
  DEV BvhNode load(int32_t i) const {
    float4 a, b, c, d;
    if (uint32_t(i) < staged) {
      const float4* p = reinterpret_cast<const float4*>(s_nodes + i);
      a = p[0];
      b = p[1];
      c = p[2];
      d = p[3];
    } else {
      const float4* p = reinterpret_cast<const float4*>(g_nodes + i);
      a = __ldg(p + 0);
      b = __ldg(p + 1);
      c = __ldg(p + 2);
      d = __ldg(p + 3);
    }
    BvhNode n;
    n.lo0[0] = a.x; n.lo0[1] = a.y; n.lo0[2] = a.z;
    n.hi0[0] = a.w; n.hi0[1] = b.x; n.hi0[2] = b.y;
    n.lo1[0] = b.z; n.lo1[1] = b.w; n.lo1[2] = c.x;
    n.hi1[0] = c.y; n.hi1[1] = c.z; n.hi1[2] = c.w;
    n.child0 = __float_as_int(d.x);
    n.child1 = __float_as_int(d.y);
    n.pad0 = 0;
    n.pad1 = 0;
    return n;
  }
};

// the state of one ray between steps of the walk (bvh.h traverse(), unrolled into a resumable form)
struct RayWalk {
  float ox, oy, oz, dx, dy, dz, ix, iy, iz, tmin, tmax;
  int32_t cur, sp;
  DEV void begin(V3 o, V3 d, float t0, float t1) {
    ox = o.x; oy = o.y; oz = o.z;
    dx = d.x; dy = d.y; dz = d.z;
    ix = 1.0f / d.x; iy = 1.0f / d.y; iz = 1.0f / d.z;
    tmin = t0;
    tmax = t1;
    cur = 0;  // the root is always an inner node
    sp = 0;
  }
};

// One step: an inner node (descend / push) or a whole leaf (<= 4 triangles through `visit`), then the pop.  Returns true when the ray is done.
// Same decisions, in the same order, as traverse() in bvh.h.
template <class Visitor>
DEV bool walk_step(RayWalk& r, int32_t* stack, const StagedNodes& nodes, const float4* tri_pos, Visitor& visit, uint32_t& n_nodes, uint32_t& n_tris) {
  if (r.cur >= 0) {
    BvhNode n = nodes.load(r.cur);
    n_nodes += 1u;
    float t0, t1;
    bool h0 = slab(n.lo0, n.hi0, r.ox, r.oy, r.oz, r.ix, r.iy, r.iz, r.tmin, r.tmax, t0);
    bool h1 = slab(n.lo1, n.hi1, r.ox, r.oy, r.oz, r.ix, r.iy, r.iz, r.tmin, r.tmax, t1);
    if (h0 && h1) {
      bool first0 = t0 <= t1;
      int32_t nearc = first0 ? n.child0 : n.child1;
      int32_t farc = first0 ? n.child1 : n.child0;
      if (r.sp < kBvhStackSize) stack[r.sp++] = farc;
      r.cur = nearc;
      return false;
    } else if (h0) {
      r.cur = n.child0;
      return false;
    } else if (h1) {
      r.cur = n.child1;
      return false;
    }
  } else {
    uint32_t ref = uint32_t(~r.cur);
    uint32_t first = ref >> 2;
    uint32_t count = (ref & 3u) + 1u;
    for (uint32_t k = 0; k < count; ++k) {
      uint32_t slot = first + k;
      float4 va = __ldg(tri_pos + slot * 3u + 0u), vb = __ldg(tri_pos + slot * 3u + 1u), vc = __ldg(tri_pos + slot * 3u + 2u);
      F4 a = {va.x, va.y, va.z, va.w}, b = {vb.x, vb.y, vb.z, vb.w}, c = {vc.x, vc.y, vc.z, vc.w};
      n_tris += 1u;
      float t, u, v;
      if (tri_test(a, b, c, r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, r.tmin, r.tmax, t, u, v)) {
        int action = visit(f2u(a.w), u, v, t);
        if (action == kCandAccept) {
          r.tmax = t;
        } else if (action == kCandTerminate) {
          return true;
        }
      }
    }
  }
  if (r.sp == 0) return true;
  r.cur = stack[--r.sp];
  return false;
}

// idle lanes of the warp take the next entries of a device-side work list; returns false for a lane that got none.  `exhausted` becomes true
// (warp-uniform) once the cursor has run past the end.
DEV bool warp_refill(bool idle, uint32_t* cursor, uint32_t total, uint32_t& index, bool& exhausted) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t idle_mask = __ballot_sync(0xffffffffu, idle);
  if ((idle_mask == 0u) || exhausted) return false;
  uint32_t base = 0;
  if (lane == 0u) base = atomicAdd(cursor, __popc(idle_mask));
  base = __shfl_sync(0xffffffffu, base, 0);
  exhausted = (base + __popc(idle_mask)) >= total;
  if (!idle) return false;
  index = base + __popc(idle_mask & ((1u << lane) - 1u));
  return index < total;
}

}  // namespace etxb
