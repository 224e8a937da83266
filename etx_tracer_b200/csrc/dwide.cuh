// dwide.cuh — traversal of the 4-wide quantised BVH (bvh.h WideNode, bvh_build.cpp build_wide_bvh): product build only.
//
// The reference casts rays through Embree's wide, compressed BVH (rt.cxx:66-88, 250-279); round 1 replaced it by a BVH2 walk shared with the
// oracle (bvh.h) because the candidate order feeds the sampler.  The product build's stochastic stages already run on their own streams, so for
// scenes with stochastic BSDFs its two dedicated traversal kernels (closest hit, shadow-segment resolve) walk THIS tree instead: one 64-byte
// node holds four children (8-bit boxes on a power-of-two grid anchored at the node's corner, decoded with one multiply-add per plane, always
// containing the exact box), so a ray makes about half the dependent fetches and moves half the bytes per box; children are visited near to
// far, and a stacked child carries its entry distance, so it is dropped at the pop once a closer hit has been found.  Triangles, leaves and the
// intersection test are the BVH2's; the closest hit found is the same, the ORDER candidates are met in (hence the sampler draws of the alpha test)
// is this tree's — covered by the statistical parity tests, not by the bit-exact ones (the parity build keeps the BVH2 everywhere).
#pragma once
#include "dtrav.cuh"

namespace etxb {

struct WideHit {
  float t;
  int32_t ref;
};

struct WideNodes {
  const WideNode* s_nodes;  // may be null: nothing staged
  const WideNode* g_nodes;
  uint32_t staged;
};

// decodes node `i`, tests its children against the ray and returns the hit ones sorted near to far in out[0 .. n)
DEV int wide_node_hits(const WideNodes& nodes, int32_t i, const RayWalk& r, WideHit out[4]) {
  uint4 a, b, c, d;
  if (uint32_t(i) < nodes.staged) {
    const uint4* p = reinterpret_cast<const uint4*>(nodes.s_nodes + i);
    a = p[0];
    b = p[1];
    c = p[2];
    d = p[3];
  } else {
    const uint4* p = reinterpret_cast<const uint4*>(nodes.g_nodes + i);
    a = __ldg(p + 0);
    b = __ldg(p + 1);
    c = __ldg(p + 2);
    d = __ldg(p + 3);
  }
  // bytes 0..11 origin, 12..14 exponents, 15 count, 16..27 qlo[4][3], 28..39 qhi[4][3], 40..55 child[4]
  const float ox = __uint_as_float(a.x), oy = __uint_as_float(a.y), oz = __uint_as_float(a.z);
  const float sx = __uint_as_float((a.w & 0xffu) << 23), sy = __uint_as_float(((a.w >> 8) & 0xffu) << 23), sz = __uint_as_float(((a.w >> 16) & 0xffu) << 23);
  const uint32_t count = a.w >> 24;
  const uint32_t qw[6] = {b.x, b.y, b.z, b.w, c.x, c.y};  // 24 bytes: qlo then qhi
  const int32_t child[4] = {int32_t(c.z), int32_t(c.w), int32_t(d.x), int32_t(d.y)};
  auto q = [&](uint32_t byte) { return float((qw[byte >> 2] >> ((byte & 3u) * 8u)) & 0xffu); };
  // plane distances straight from the quantised coordinates: t = (origin + q * step - ray_o) * inv_d = q * (step * inv_d) + (origin - ray_o) * inv_d —
  // one multiply-add per plane, the two per-axis constants once per node (the compressed wide BVH's standard form)
  const float ax = sx * r.ix, ay = sy * r.iy, az = sz * r.iz;
  const float bx = (ox - r.ox) * r.ix, by = (oy - r.oy) * r.iy, bz = (oz - r.oz) * r.iz;
  // the four entry distances (kMaxFloat = missed / unused slot), then a 5-comparator sorting network: everything stays in registers
  float t[4];
  int32_t ref[4];
#pragma unroll
  for (uint32_t k = 0; k < 4u; ++k) {
    const float tx0 = fmaf(q(k * 3u + 0u), ax, bx), tx1 = fmaf(q(12u + k * 3u + 0u), ax, bx);
    const float ty0 = fmaf(q(k * 3u + 1u), ay, by), ty1 = fmaf(q(12u + k * 3u + 1u), ay, by);
    const float tz0 = fmaf(q(k * 3u + 2u), az, bz), tz1 = fmaf(q(12u + k * 3u + 2u), az, bz);
    const float tn = fmaxf(fmaxf(fminf(tx0, tx1), fminf(ty0, ty1)), fmaxf(fminf(tz0, tz1), r.tmin));
    float tf = fminf(fminf(fmaxf(tx0, tx1), fmaxf(ty0, ty1)), fminf(fmaxf(tz0, tz1), r.tmax));
    tf = tf * 1.0000004f;  // conservative far plane (2 ulp), like bvh.h slab()
    const bool hit = (k < count) && (tn <= tf);
    t[k] = hit ? tn : kMaxFloat;
    ref[k] = child[k];
  }
  auto cswap = [&](int i, int j) {
    if (t[j] < t[i]) {
      float tt = t[i];
      t[i] = t[j];
      t[j] = tt;
      int32_t rr = ref[i];
      ref[i] = ref[j];
      ref[j] = rr;
    }
  };
  cswap(0, 1);
  cswap(2, 3);
  cswap(0, 2);
  cswap(1, 3);
  cswap(1, 2);
  int n = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    out[k] = {t[k], ref[k]};
    n += (t[k] < kMaxFloat) ? 1 : 0;
  }
  return n;
}

// the state of one ray in the wide tree
struct WideWalk {
  RayWalk ray;
  int32_t cur;  // current reference (wide node or leaf); kWideDone when the stack ran empty
  int32_t sp;
};
constexpr int32_t kWideDone = int32_t(0x80000000u);

// One step: a wide node (descend into the nearest hit child, stack the others far to near) or a leaf (its triangles through `visit`), then the
// pop, skipping stacked children that start beyond the current tmax.  Returns true when the ray is done.
template <class Visitor>
DEV bool wide_step(WideWalk& w, WideHit* stack, const WideNodes& nodes, const float4* tri_pos, Visitor& visit, uint32_t& n_nodes, uint32_t& n_tris) {
  if (w.cur >= 0) {
    WideHit hits[4];
    const int n = wide_node_hits(nodes, w.cur, w.ray, hits);
    n_nodes += 1u;
    if (n > 0) {
#pragma unroll
      for (int k = 3; k >= 1; --k) {  // far to near, so that the nearest of the stacked ones pops first
        if ((k < n) && (w.sp < kWideStackSize)) stack[w.sp++] = hits[k];
      }
      w.cur = hits[0].ref;
      return false;
    }
  } else {
    uint32_t ref = uint32_t(~w.cur);
    uint32_t first = ref >> 2;
    uint32_t count = (ref & 3u) + 1u;
    for (uint32_t k = 0; k < count; ++k) {
      uint32_t slot = first + k;
      float4 va = __ldg(tri_pos + slot * 3u + 0u), vb = __ldg(tri_pos + slot * 3u + 1u), vc = __ldg(tri_pos + slot * 3u + 2u);
      F4 a = {va.x, va.y, va.z, va.w}, b = {vb.x, vb.y, vb.z, vb.w}, c = {vc.x, vc.y, vc.z, vc.w};
      n_tris += 1u;
      float t, u, v;
      if (tri_test(a, b, c, w.ray.ox, w.ray.oy, w.ray.oz, w.ray.dx, w.ray.dy, w.ray.dz, w.ray.tmin, w.ray.tmax, t, u, v)) {
        int action = visit(f2u(a.w), u, v, t);
        if (action == kCandAccept) {
          w.ray.tmax = t;
        } else if (action == kCandTerminate) {
          return true;
        }
      }
    }
  }
  for (;;) {
    if (w.sp == 0) return true;
    WideHit h = stack[--w.sp];
    if (h.t <= w.ray.tmax) {  // a closer hit found meanwhile makes the whole subtree irrelevant
      w.cur = h.ref;
      return false;
    }
  }
}

DEV void wide_begin(WideWalk& w, V3 o, V3 d, float t0, float t1) {
  w.ray.begin(o, d, t0, t1);
  // the plane distances are formed as q * (step / d) + (origin - o) / d: a direction component of exactly zero would turn them into inf - inf;
  // a huge finite reciprocal keeps the slab logic (the ray is inside the slab's extent or misses it) without NaNs.  The triangle test uses d itself.
  auto safe_inv = [](float x) { return (fabsf(x) > 1.0e-20f) ? 1.0f / x : copysignf(1.0e20f, x); };
  w.ray.ix = safe_inv(d.x);
  w.ray.iy = safe_inv(d.y);
  w.ray.iz = safe_inv(d.z);
  w.cur = 0;
  w.sp = 0;
}

// One ray through the whole tree (global memory, nothing staged); n_nodes / n_tris count the nodes and triangles it tested.
template <class Visitor>
DEV void wide_trace(const DeviceScene& sc, V3 o, V3 d, float tmin, float tmax, Visitor& visit, uint32_t& n_nodes, uint32_t& n_tris) {
  const WideNodes nodes{nullptr, sc.wide_nodes, 0u};
  WideWalk walk;
  WideHit stack[kWideStackSize];
  wide_begin(walk, o, d, tmin, tmax);
  while (!wide_step(walk, stack, nodes, sc.bvh_tris, visit, n_nodes, n_tris)) {
  }
}

// The candidate test of a closest-hit query (Raytracing::trace, rt.cxx:428-466): Void surfaces and alpha-rejected hits are skipped, any
// other candidate becomes the closest hit so far.
struct ClosestHitVisitor {
  const DeviceScene& sc;
  Smp* smp;
  HitRec* best;
  DEV int operator()(uint32_t triangle_index, float u, float v, float t) {
    const etxb_material& mat = sc.materials[load_triangle_material(sc, triangle_index)];
    if (mat.cls == ETXB_MAT_VOID) return kCandIgnore;
    if (alpha_test_rejects(sc, mat, triangle_index, u, v, *smp)) return kCandIgnore;
    *best = {u, v, t, triangle_index};
    return kCandAccept;
  }
};

// The closest hit of one ray (tri = kInvalidIndex: none), drawing from `smp` once per alpha-tested candidate.
DEV HitRec trace_closest_wide(const DeviceScene& sc, V3 o, V3 d, float tmin, float tmax, Smp& smp, uint32_t& n_nodes, uint32_t& n_tris) {
  HitRec best = {0.0f, 0.0f, 0.0f, kInvalidIndex};
  ClosestHitVisitor visit{sc, &smp, &best};
  wide_trace(sc, o, d, tmin, tmax, visit, n_nodes, n_tris);
  return best;
}

}  // namespace etxb
