// dtrace.cuh — device ray queries over the shared BVH (bvh.h): closest hit and transmittance.
// Restates Raytracing::trace / trace_transmittance (sources/etx/rt/rt.cxx:428-466, 468-579) with the
// reference's filter semantics: Void materials are skipped, and EVERY other candidate hit draws one value
// from the path's sampler for the stochastic alpha test (scene_bsdf.hxx:128-144).
#pragma once
#include "dscene.cuh"

// A kernel's traversal counters (TraverseStats, bvh.h): real ones in the count build, a null `stats` pointer in the others
#ifdef ETXB_COUNT_TRAVERSAL
#define STATS_DECL TraverseStats stats_obj; TraverseStats* stats = &stats_obj
#define STATS_NODES stats_obj.nodes
#define STATS_TRIS stats_obj.tris
#else
#define STATS_DECL TraverseStats* stats = nullptr
#define STATS_NODES 0u
#define STATS_TRIS 0u
#endif

namespace etxb {

struct DevNodeLoad {
  const BvhNode* nodes;
  DEV BvhNode operator()(int32_t i) const {
    const float4* p = reinterpret_cast<const float4*>(nodes + i);
    float4 a = __ldg(p + 0), b = __ldg(p + 1), c = __ldg(p + 2), d = __ldg(p + 3);
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
struct DevTriLoad {
  const float4* pos;
  DEV F4 operator()(uint32_t i) const {
    float4 v = __ldg(pos + i);
    return F4{v.x, v.y, v.z, v.w};
  }
};

// alpha_test_pass (scene_bsdf.hxx:128-144)
DEV bool alpha_test_rejects(const DeviceScene& sc, const etxb_material& mat, uint32_t triangle_index, float u, float v, Smp& smp) {
  float alpha_diffuse = 1.0f;
  if (mat.scattering.image_index != kInvalidIndex) {
    const DImage& img = sc.images[mat.scattering.image_index];
    if (img.options & kImageHasAlpha) {
      V2 uv = lerp_uv(sc, load_triangle(sc, triangle_index), barycentrics_uv(u, v));
      alpha_diffuse = image_evaluate_alpha(img, uv);
    }
  }
  float alpha_test_value = alpha_diffuse * mat.opacity;
  return alpha_test_value <= smp.next();
}

struct HitRec {
  float u, v, t;
  uint32_t tri;  // kInvalidIndex = miss
};

struct ClosestVisitor {
  const DeviceScene& sc;
  Smp& smp;
  HitRec best;
  DEV int operator()(uint32_t triangle_index, float u, float v, float t) {
    const etxb_material& mat = sc.materials[load_triangle_material(sc, triangle_index)];
    if (mat.cls == ETXB_MAT_VOID) return kCandIgnore;
    if (alpha_test_rejects(sc, mat, triangle_index, u, v, smp)) return kCandIgnore;
    best = {u, v, t, triangle_index};
    return kCandAccept;
  }
};

DEV HitRec trace_closest(const DeviceScene& sc, V3 o, V3 d, float tmin, float tmax, Smp& smp, TraverseStats* stats) {
  ClosestVisitor vis{sc, smp, {0.0f, 0.0f, 0.0f, kInvalidIndex}};
  DevNodeLoad nl{sc.bvh_nodes};
  DevTriLoad tl{sc.bvh_tris};
  traverse(nl, tl, o.x, o.y, o.z, d.x, d.y, d.z, tmin, tmax, vis, stats);
  return vis.best;
}

// The segment set-up of every shadow query (rt.cxx:468-490): false for a degenerate segment, whose squared length is at most kRayEpsilon
// (it counts as unoccluded, :474-477); otherwise the unit direction from p0 and the distance to stop at, short of p1 by
// max(kRayEpsilon, length * kRayEpsilon) so that the surface at p1 is not hit.
DEV bool shadow_segment(V3 p0, V3 p1, V3& direction, float& t_max) {
  direction = p1 - p0;
  t_max = dot(direction, direction);
  if (t_max <= kRayEpsilon) return false;
  t_max = sqrtf(t_max);
  direction /= t_max;
  t_max -= fmaxf(kRayEpsilon, t_max * kRayEpsilon);
  return true;
}

struct Crossing {
  uint32_t primitive_id;
  float u, v, t;
};
constexpr uint32_t kCrossingBufferSize = 63;  // rt.cxx:472

struct ShadowVisitor {
  const DeviceScene& sc;
  Smp& smp;
  Crossing* crossings;
  uint32_t crossing_count;
  bool occluded;
  DEV int operator()(uint32_t triangle_index, float u, float v, float t) {
    const etxb_material& mat = sc.materials[load_triangle_material(sc, triangle_index)];
    if (mat.cls == ETXB_MAT_VOID) return kCandIgnore;
    if (alpha_test_rejects(sc, mat, triangle_index, u, v, smp)) return kCandIgnore;
    if ((mat.cls != ETXB_MAT_BOUNDARY) || (crossing_count + 1u >= kCrossingBufferSize)) {
      occluded = true;
      return kCandTerminate;
    }
    crossings[crossing_count++] = {triangle_index, u, v, t};
    return kCandIgnore;
  }
};

}  // namespace etxb
#include "dmedium.cuh"
namespace etxb {

// Raytracing::trace_transmittance (rt.cxx:468-579): occluded unless every hit is a Boundary; the (<= 63) boundary crossings are
// sorted by t and the per-segment medium transmittance is multiplied in.
// The occlusion half of trace_transmittance for scenes without Boundary materials and media: any non-Void hit on the segment
// occludes (same segment set-up as rt.cxx:468-490).  Used by k_shadow_trace.
struct OcclusionVisitor {
  const DeviceScene& sc;
  bool occluded;
  DEV int operator()(uint32_t triangle_index, float, float, float) {
    if (sc.materials[load_triangle_material(sc, triangle_index)].cls == ETXB_MAT_VOID) return kCandIgnore;
    occluded = true;
    return kCandTerminate;
  }
};
DEV bool trace_occluded(const DeviceScene& sc, V3 p0, V3 p1) {
  V3 direction;
  float t_max;
  if (!shadow_segment(p0, p1, direction, t_max)) return false;
  OcclusionVisitor vis{sc, false};
  DevNodeLoad nl{sc.bvh_nodes};
  DevTriLoad tl{sc.bvh_tris};
  traverse(nl, tl, p0.x, p0.y, p0.z, direction.x, direction.y, direction.z, kRayEpsilon, t_max, vis, static_cast<TraverseStats*>(nullptr));
  return vis.occluded;
}

struct PlainShadowVisitor {
  const DeviceScene& sc;
  Smp& smp;
  bool occluded;
  DEV int operator()(uint32_t triangle_index, float u, float v, float) {
    const etxb_material& mat = sc.materials[load_triangle_material(sc, triangle_index)];
    if (mat.cls == ETXB_MAT_VOID) return kCandIgnore;
    if (alpha_test_rejects(sc, mat, triangle_index, u, v, smp)) return kCandIgnore;
    occluded = true;
    return kCandTerminate;
  }
};

// Out of line: every kernel reaches it from several connection routines, and one BVH traversal dwarfs the call.
// PLAIN: compile-time promise that the scene has no Boundary surfaces, media or subsurface materials (DeviceScene flags, checked by the host).
template <bool SP, bool PLAIN = false>
DEVN Spec<SP> trace_transmittance(const DeviceScene& sc, float wavelength, V3 p0, V3 p1, uint32_t medium_index, Smp& smp, TraverseStats* stats) {
  V3 direction;
  float t_max;
  if (!shadow_segment(p0, p1, direction, t_max)) return Spec<SP>::make(1.0f);
  if constexpr (PLAIN) {
    // scenes without Boundary surfaces and media: the first candidate that passes the alpha test occludes — no crossing list, no media walk
    PlainShadowVisitor pvis{sc, smp, false};
    DevNodeLoad pnl{sc.bvh_nodes};
    DevTriLoad ptl{sc.bvh_tris};
    traverse(pnl, ptl, p0.x, p0.y, p0.z, direction.x, direction.y, direction.z, kRayEpsilon, t_max, pvis, stats);
    return Spec<SP>::make(pvis.occluded ? 0.0f : 1.0f);
  }
  Crossing crossings[kCrossingBufferSize + 1u];
  ShadowVisitor vis{sc, smp, crossings, 0u, false};
  DevNodeLoad nl{sc.bvh_nodes};
  DevTriLoad tl{sc.bvh_tris};
  traverse(nl, tl, p0.x, p0.y, p0.z, direction.x, direction.y, direction.z, kRayEpsilon, t_max, vis, stats);
  if (vis.occluded) return Spec<SP>::make(0.0f);
  if ((vis.crossing_count == 0u) && (medium_index == kInvalidIndex)) return Spec<SP>::make(1.0f);
  uint32_t n = vis.crossing_count;
  for (uint32_t i = 0; i < n; ++i) {
    for (uint32_t j = i + 1; j < n; ++j) {
      if (crossings[i].t > crossings[j].t) {
        Crossing tmp = crossings[i];
        crossings[i] = crossings[j];
        crossings[j] = tmp;
      }
    }
  }
  crossings[n++] = {kInvalidIndex, 0.0f, 0.0f, t_max};
  float current_t = 0.0f;
  V3 origin = p0;
  Spec<SP> result = Spec<SP>::make(1.0f);
  uint32_t current_medium = medium_index;
  for (uint32_t i = 0; i < n; ++i) {
    const Crossing c = crossings[i];
    if (current_medium != kInvalidIndex) {
      float dt = fmaxf(0.0f, c.t - current_t);
      result *= medium_transmittance<SP>(sc, sc.mediums[current_medium], wavelength, smp, origin, direction, dt);
    }
    if (c.primitive_id == kInvalidIndex) break;
    TriRec tri = load_triangle(sc, c.primitive_id);
    const etxb_material& mat = sc.materials[tri.material_index];
    const bool entering = dot(tri.geo_n, direction) < 0.0f;
    current_medium = entering ? mat.int_medium : mat.ext_medium;
    current_t = c.t;
    origin = lerp_pos(sc, tri, barycentrics_uv(c.u, c.v));
  }
  return result;
}

}  // namespace etxb
