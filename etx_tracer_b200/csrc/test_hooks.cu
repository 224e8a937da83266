// test_hooks.cu — the test hooks of the C interface (include/etx_b200.h) that run the device routines of d*.cuh on host-given rays, segments,
// triangle soups and queries, with the kernels they launch.  They reach the context through context.cuh only; the hooks that drive the
// product's own passes (etxb_debug_merge, _denoise, _film_view, _film_error, _noise_estimate, _set_thresholds) stay in module.cu beside them.
#include "bvh_build.h"
#include "bvh_build_device.h"
#include "context.cuh"
#include "dsss.cuh"
#include "dwide.cuh"

namespace etxb {

// thread t of a launch over count x reps threads: query i = t / reps, repetition r = t % reps; false past the last
DEV bool query_thread(uint32_t count, uint32_t reps, uint32_t& t, uint32_t& i, uint32_t& r) {
  t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= count * reps) return false;
  i = t / reps;
  r = t % reps;
  return true;
}

DEV void put3(float* dst, V3 a) {
  dst[0] = a.x;
  dst[1] = a.y;
  dst[2] = a.z;
}

// closest hits of rays (origin, tmin, direction, tmax: 8 floats each), as k_trace_closest finds them; through the 4-wide quantised tree, as
// k_trace_closest_wide finds them, when `wide` (product build, scenes that have one)
__global__ void k_debug_trace(const __grid_constant__ DeviceScene sc, const float* rays, uint32_t* seeds, uint32_t count, uint32_t wide, float* hits_uv_t,
                              uint32_t* hits_tri) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float* r = rays + size_t(i) * 8;
  const V3 o = {r[0], r[1], r[2]}, d = {r[4], r[5], r[6]};
  Smp smp = Smp::resume(seeds[i]);
  uint32_t n_nodes = 0, n_tris = 0;
  const HitRec h = wide ? trace_closest_wide(sc, o, d, r[3], r[7], smp, n_nodes, n_tris) : trace_closest(sc, o, d, r[3], r[7], smp, nullptr);
  seeds[i] = smp.seed;
  hits_tri[i] = h.tri;
  bool hit = h.tri != kInvalidIndex;
  hits_uv_t[size_t(i) * 3 + 0] = hit ? h.u : 0.0f;
  hits_uv_t[size_t(i) * 3 + 1] = hit ? h.v : 0.0f;
  hits_uv_t[size_t(i) * 3 + 2] = hit ? h.t : 0.0f;
}

// occlusion of segments (p0, p1: 6 floats each), as k_shadow_resolve tests them: any non-Void surface in between; through the 4-wide
// quantised tree when `wide` (product build, scenes that have one), the BVH2 otherwise
__global__ void k_debug_occluded(const __grid_constant__ DeviceScene sc, const float* segments, uint32_t count, uint32_t wide, uint32_t* occluded) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float* s = segments + size_t(i) * 6;
  const V3 p0 = {s[0], s[1], s[2]}, p1 = {s[3], s[4], s[5]};
  if (!wide) {
    occluded[i] = trace_occluded(sc, p0, p1) ? 1u : 0u;
    return;
  }
  V3 direction;
  float t_max;
  if (!shadow_segment(p0, p1, direction, t_max)) {
    occluded[i] = 0u;  // a degenerate segment is unoccluded
    return;
  }
  OcclusionVisitor visit{sc, false};
  uint32_t n_nodes = 0, n_tris = 0;
  wide_trace(sc, p0, direction, kRayEpsilon, t_max, visit, n_nodes, n_tris);
  occluded[i] = visit.occluded ? 1u : 0u;
}

__global__ void k_debug_sampler(const uint32_t* a, const uint32_t* b, uint32_t count, uint32_t draws, uint32_t* out_seed, float* out_values) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  Smp s;
  s.init(a[i], b[i]);
  out_seed[size_t(i) * (draws + 1u)] = s.seed;
  for (uint32_t d = 0; d < draws; ++d) {
    out_values[size_t(i) * draws + d] = s.next();
    out_seed[size_t(i) * (draws + 1u) + d + 1u] = s.seed;
  }
}

__global__ void k_debug_math(const __grid_constant__ DeviceScene sc, uint32_t fn, const float* x, const float* y, uint32_t count, float* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float a = x[i], b = y ? y[i] : 0.0f, r = 0.0f;
  switch (fn) {
    case 0: r = m_sin(a); break;
    case 1: r = m_cos(a); break;
    case 2: r = m_exp(a); break;
    case 3: r = m_log(a); break;
    case 4: r = m_pow(a, b); break;
    case 5: r = m_acos(a); break;
    case 6: r = m_atan2(a, b); break;
    case 7: r = spectral_sample_wavelength(a); break;
    case 8: r = spectral_sampling_pdf(a); break;
    case 9: r = spec_to_rgb<true>(sc, Spec<true>{1.0f}, a).x; break;
    case 10: r = spec_to_rgb<true>(sc, Spec<true>{1.0f}, a).y; break;
    case 11: r = spec_to_rgb<true>(sc, Spec<true>{1.0f}, a).z; break;
    case 12: r = m_atan(a); break;
    case 13: r = m_asin(a); break;
    case 14: r = sample_blue_noise(sc, uint32_t(a) & 127u, uint32_t(a) >> 7, uint32_t(b), 0).x; break;
    case 15: r = sample_blue_noise(sc, uint32_t(a) & 127u, uint32_t(a) >> 7, uint32_t(b), 4).y; break;
    default: break;
  }
  out[i] = r;
}

// one thread per etxb_closure_query: `reps` times make_closure + closure_evaluate on a fresh sampler Smp::init(seed, r), as the photon gather
// and the vertex connections call them; float64 running moments (Welford: a constant output keeps a variance of exactly 0) of
// {func.rgb, bsdf.rgb, pdf, rev_pdf}, repetition 0's raw values and the counters of include/etx_b200.h (ETXB_CLOSURE_STATS per query)
template <bool SP>
__global__ void k_debug_closure(const __grid_constant__ DeviceScene sc, const etxb_closure_query* queries, uint32_t count, uint32_t reps, double* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const etxb_closure_query& q = queries[i];
  const V3 nrm = {q.nrm[0], q.nrm[1], q.nrm[2]}, tan = {q.tan[0], q.tan[1], q.tan[2]}, btn = {q.btn[0], q.btn[1], q.btn[2]};
  const V3 w_i = {q.w_i[0], q.w_i[1], q.w_i[2]}, w_o = {q.w_o[0], q.w_o[1], q.w_o[2]};
  const BData d = {{0.0f, 0.0f, 0.0f}, nrm, tan, btn, {q.uv[0], q.uv[1]}, w_i, SP ? q.wavelength : -1.0f, q.path_source, kInvalidIndex};
  double mean[8], m2[8];
  double* o = out + size_t(i) * ETXB_CLOSURE_STATS;
  for (uint32_t k = 0; k < 8; ++k) mean[k] = m2[k] = 0.0;
  uint32_t finite = 0, nonfinite = 0, negative = 0, unsupported = 0;
  for (uint32_t r = 0; r < reps; ++r) {
    Smp smp;
    smp.init(q.seed, r);
    const Closure<SP> c = make_closure<SP>(sc, d, q.material, smp);
    const CEval<SP> e = closure_evaluate<SP>(sc, c, w_o, smp);
    const V3 f = e.func.as_v3(), b = e.bsdf.as_v3();
    const float v[8] = {f.x, f.y, f.z, b.x, b.y, b.z, e.pdf, e.rev_pdf};
    if (r == 0) {
      for (uint32_t k = 0; k < 8; ++k) o[16 + k] = v[k];
    }
    bool ok = true;
    for (uint32_t k = 0; k < 8; ++k) ok = ok && isfinite(v[k]);
    negative += ((e.pdf < 0.0f) || (e.rev_pdf < 0.0f)) ? 1u : 0u;
    unsupported += ((e.pdf == 0.0f) && ((f.x != 0.0f) || (f.y != 0.0f) || (f.z != 0.0f) || (b.x != 0.0f) || (b.y != 0.0f) || (b.z != 0.0f))) ? 1u : 0u;
    if (!ok) {
      nonfinite += 1u;
      continue;
    }
    finite += 1u;
    for (uint32_t k = 0; k < 8; ++k) {
      const double delta = double(v[k]) - mean[k];
      mean[k] += delta / double(finite);
      m2[k] += delta * (double(v[k]) - mean[k]);
    }
  }
  for (uint32_t k = 0; k < 8; ++k) {
    o[k] = mean[k];
    o[8 + k] = (finite > 0) ? m2[k] / double(finite) : 0.0;
  }
  o[24] = double(nonfinite);
  o[25] = double(negative);
  o[26] = double(unsupported);
  for (uint32_t k = 27; k < ETXB_CLOSURE_STATS; ++k) o[k] = 0.0;
}

// one thread per (etxb_sample_query, repetition): bsdf_sample on the sampler Smp::init(seed, r) with the fixed values a bounce pushes
// (mode 0, kernels.cuh / dpt.cuh at every bsdf_sample call) or the query's own (mode 1); record layout in include/etx_b200.h
template <bool SP>
__global__ void k_debug_bsdf_sample(const __grid_constant__ DeviceScene sc, const etxb_sample_query* queries, uint32_t count, uint32_t reps, etxb_sample_result* out) {
  uint32_t t, i, r;
  if (!query_thread(count, reps, t, i, r)) return;
  const etxb_sample_query& q = queries[i];
  const V3 nrm = {q.nrm[0], q.nrm[1], q.nrm[2]}, tan = {q.tan[0], q.tan[1], q.tan[2]}, btn = {q.btn[0], q.btn[1], q.btn[2]};
  const V3 w_i = {q.w_i[0], q.w_i[1], q.w_i[2]};
  const BData d = {{0.0f, 0.0f, 0.0f}, nrm, tan, btn, {q.uv[0], q.uv[1]}, w_i, SP ? q.wavelength : -1.0f, q.path_source, q.medium};
  Smp smp;
  smp.init(q.seed, r);
  etxb_sample_result& o = out[t];
  o.seed_start = smp.seed;
  if (q.mode == 0u) {
    const V2 rnd_bsdf = smp.next_2d();
    smp.next_2d();  // rnd_connection
    const V2 rnd_support = smp.next_2d();
    smp.push_fixed(rnd_bsdf.x, rnd_bsdf.y, rnd_support.x);
  } else {
    smp.push_fixed(q.fixed[0], q.fixed[1], q.fixed[2]);
  }
  const BSample<SP> s = bsdf_sample<SP>(sc, d, sc.materials[q.material], smp);
  smp.pop_fixed();
  const V3 w = s.weight.as_v3();
  o.w_o[0] = s.w_o.x;
  o.w_o[1] = s.w_o.y;
  o.w_o[2] = s.w_o.z;
  o.pdf = s.pdf;
  o.weight[0] = w.x;
  o.weight[1] = w.y;
  o.weight[2] = w.z;
  o.eta = s.eta;
  o.properties = s.properties;
  o.medium_index = s.medium_index;
  o.seed_end = smp.seed;
}

// one thread per (etxb_emitter_query, repetition): the emitter routines of dvcm.cuh as the passes call them; ops and record layout in
// include/etx_b200.h
static_assert(sizeof(etxb_emitter_query) == 80u && sizeof(etxb_emitter_result) == 104u, "etxb_emitter_query / etxb_emitter_result layout");
template <bool SP>
__global__ void k_debug_emitter(const __grid_constant__ DeviceScene sc, const etxb_emitter_query* queries, uint32_t count, uint32_t reps, etxb_emitter_result* out) {
  uint32_t t, i, r;
  if (!query_thread(count, reps, t, i, r)) return;
  const etxb_emitter_query& q = queries[i];
  const float wavelength = SP ? q.wavelength : -1.0f;
  const V3 source = {q.source[0], q.source[1], q.source[2]};
  etxb_emitter_result o = {};
  EmitterSample<SP> s = {};
  s.value = Spec<SP>::make(0.0f);
  s.emitter_index = s.triangle_index = s.medium_index = kInvalidIndex;
  if (q.op == ETXB_EMITTER_SELECT) {
    s.emitter_index = distribution_sample(sc.emitter_dist, sc.emitter_count + 1u, q.rnd[0]);
    s.pdf_sample = emitter_discrete_pdf(sc, sc.emitters[s.emitter_index]);
  } else if (q.op == ETXB_EMITTER_SAMPLE_IN) {
    s = sample_emitter<SP>(sc, wavelength, q.emitter, {q.rnd[0], q.rnd[1]}, source);
  } else if (q.op == ETXB_EMITTER_EMISSION) {
    Smp smp;
    smp.init(q.seed, r);
    o.seed_start = smp.seed;
    s = sample_emission<SP>(sc, wavelength, smp);
    o.seed_end = smp.seed;
  } else {
    const V3 target = {q.target[0], q.target[1], q.target[2]}, direction = {q.direction[0], q.direction[1], q.direction[2]};
    s.emitter_index = q.emitter;
    s.value = emitter_get_radiance<SP>(sc, sc.emitters[q.emitter], wavelength, source, target, direction, {q.uv[0], q.uv[1]}, q.directly_visible != 0u, s.pdf_area,
      s.pdf_dir, s.pdf_dir_out);
  }
  put3(o.value, s.value.as_v3());
  put3(o.origin, s.origin);
  put3(o.normal, s.normal);
  put3(o.direction, s.direction);
  put3(o.barycentric, s.barycentric);
  o.pdf_sample = s.pdf_sample;
  o.pdf_area = s.pdf_area;
  o.pdf_dir = s.pdf_dir;
  o.pdf_dir_out = s.pdf_dir_out;
  o.emitter_index = s.emitter_index;
  o.triangle_index = s.triangle_index;
  o.medium_index = s.medium_index;
  o.flags = (s.is_delta ? 1u : 0u) | (s.is_distant ? 2u : 0u);
  out[t] = o;
}

// one thread per (etxb_medium_query, repetition): the media routines of dmedium.cuh and the shadow-ray walk of dtrace.cuh as the passes
// call them; ops and record layout in include/etx_b200.h
static_assert(sizeof(etxb_medium_query) == 96u && sizeof(etxb_medium_result) == 64u, "etxb_medium_query / etxb_medium_result layout");
template <bool SP>
__global__ void k_debug_medium(const __grid_constant__ DeviceScene sc, const etxb_medium_query* queries, uint32_t count, uint32_t reps, etxb_medium_result* out) {
  uint32_t t, i, r;
  if (!query_thread(count, reps, t, i, r)) return;
  const etxb_medium_query& q = queries[i];
  const float wavelength = SP ? q.wavelength : -1.0f;
  const V3 origin = {q.origin[0], q.origin[1], q.origin[2]}, direction = {q.direction[0], q.direction[1], q.direction[2]};
  etxb_medium_result o = {};
  Smp smp;
  smp.init(q.seed, r);
  o.seed_start = smp.seed;
  if (q.op == ETXB_MEDIUM_BOUNDS) {
    V3 pos = origin, dir = direction;
    o.flag = medium_intersects_bounds(sc.mediums[q.medium], origin, direction, q.max_t, pos, dir, o.t_min, o.t_max) ? 1u : 0u;
    put3(o.pos, pos);
    put3(o.dir, dir);
  } else if (q.op == ETXB_MEDIUM_DENSITY) {
    o.value[0] = medium_sample_density(sc.mediums[q.medium], origin);
  } else if (q.op == ETXB_MEDIUM_TRANSMITTANCE) {
    put3(o.value, medium_transmittance<SP>(sc, sc.mediums[q.medium], wavelength, smp, origin, direction, q.max_t).as_v3());
  } else if (q.op == ETXB_MEDIUM_SAMPLE) {
    const Spec<SP> throughput = Spec<SP>::make3({q.throughput[0], q.throughput[1], q.throughput[2]});
    const MediumSample<SP> s = sample_medium<SP>(sc, sc.mediums[q.medium], wavelength, throughput, smp, origin, direction, q.max_t);
    put3(o.value, s.weight.as_v3());
    put3(o.pos, s.pos);
    o.t = s.sampled_medium_t;
  } else if (q.op == ETXB_MEDIUM_PHASE) {
    o.value[0] = phase_function(direction, {q.w_o[0], q.w_o[1], q.w_o[2]}, q.g);
    put3(o.dir, sample_phase_function(direction, q.g, {q.rnd[0], q.rnd[1]}));
  } else {
    STATS_DECL;  // as every other caller: the count build's trace_transmittance is compiled for a non-null stats pointer
    put3(o.value, trace_transmittance<SP, false>(sc, wavelength, origin, {q.end[0], q.end[1], q.end[2]}, q.medium, smp, stats).as_v3());
  }
  o.seed_end = smp.seed;
  out[t] = o;
}

// one thread per (etxb_subsurface_query, repetition): the subsurface routines of dsss.cuh as the bounces call them; ops and record layout
// in include/etx_b200.h
static_assert(sizeof(etxb_subsurface_query) == 128u && sizeof(etxb_subsurface_probe) == 96u && sizeof(etxb_subsurface_hit) == 64u &&
                sizeof(etxb_subsurface_result) == 1920u, "etxb_subsurface_query / etxb_subsurface_result layout");
template <bool SP>
__global__ void k_debug_subsurface(const __grid_constant__ DeviceScene sc, const etxb_subsurface_query* queries, uint32_t count, uint32_t reps,
                                   etxb_subsurface_result* out) {
  uint32_t t, i, r;
  if (!query_thread(count, reps, t, i, r)) return;
  const etxb_subsurface_query& q = queries[i];
  const float wavelength = SP ? q.wavelength : -1.0f;
  const V3 origin = {q.origin[0], q.origin[1], q.origin[2]}, direction = {q.dir[0], q.dir[1], q.dir[2]};
  const auto put_probe = [](etxb_subsurface_probe& dst, const SSSample& s) {
    put3(dst.o, s.ray_o);
    put3(dst.d, s.ray_d);
    dst.min_t = s.ray_min_t;
    dst.max_t = s.ray_max_t;
    put3(dst.u, s.u);
    put3(dst.v, s.v);
    put3(dst.w, s.w);
    put3(dst.basis_prob, s.basis_prob);
    dst.sampled_radius = s.sampled_radius;
  };
  STATS_DECL;  // as every other caller: the count build's traversals are compiled for a non-null stats pointer
  etxb_subsurface_result& o = out[t];
  Smp smp;
  smp.init(q.seed, r);
  o.seed_start = smp.seed;
  if ((q.op == ETXB_SUBSURFACE_TRACE_MATERIAL) || (q.op == ETXB_SUBSURFACE_CONTINUOUS_TRACE)) {
    HitRec h[kSSPerDirection];
    if (q.op == ETXB_SUBSURFACE_TRACE_MATERIAL) {
      h[0] = trace_material(sc, origin, direction, q.t_min, q.t_max, q.material, smp, stats);
      o.count = (h[0].tri != kInvalidIndex) ? 1u : 0u;
    } else {
      o.count = continuous_trace(sc, origin, direction, q.t_min, q.t_max, q.material, h, q.max_count, smp, stats);
    }
    for (uint32_t k = 0; k < ((q.op == ETXB_SUBSURFACE_TRACE_MATERIAL) ? 1u : o.count); ++k) {
      o.hits[k].u = h[k].u;
      o.hits[k].v = h[k].v;
      o.hits[k].t = h[k].t;
      o.hits[k].tri = h[k].tri;
    }
  } else if (q.op == ETXB_SUBSURFACE_REMAP) {
    for (uint32_t k = 0; k < 3u; ++k) remap_channel(q.color[k], q.distances[k], o.albedo[k], o.extinction[k], o.scattering[k]);
  } else {
    const Isect in = make_intersection(sc, direction, q.triangle, q.u, q.v, 0.0f);
    const etxb_material& mat = sc.materials[in.material_index];
    if (q.op == ETXB_SUBSURFACE_PROFILE) {
      o.s_r = sample_s_r(q.rnd);
      put3(o.eval, ss_evaluate<SP>(sc, wavelength, in.tex, mat, q.radius).as_v3());
      const SSSample s = ss_sample<SP>(sc, wavelength, in, mat, q.direction, smp);
      put_probe(o.probes[0], s);
      o.geometric_weight = ss_geometric_weight({q.normal[0], q.normal[1], q.normal[2]}, s);
    } else {
      if (mat.subsurface.cls == 2u) {  // the gather's three probes are its first draws
        Smp probe_smp = smp;
        for (uint32_t d = 0; d < kSSDirections; ++d) put_probe(o.probes[d], ss_sample<SP>(sc, wavelength, in, mat, d, probe_smp));
      }
      SSGather<SP> g;
      uint32_t rays = 0;
      o.flag = ss_gather<SP>(sc, wavelength, in, smp, g, stats, rays) ? 1u : 0u;
      o.rays = rays;
      if (o.flag) {
        o.count = g.count;
        o.selected = g.selected;
        o.selected_sample_weight = g.selected_sample_weight;
        o.total_weight = g.total_weight;
        for (uint32_t k = 0; k < g.count; ++k) {
          const Isect e = ss_exit_intersection<SP>(sc, g, k, sc.subsurface_exit_material);
          o.hits[k].u = g.hits[k].u;
          o.hits[k].v = g.hits[k].v;
          o.hits[k].t = g.hits[k].t;
          o.hits[k].tri = g.hits[k].tri;
          put3(o.hits[k].w_i, e.w_i);
          put3(o.hits[k].weight, g.weights[k].as_v3());
          put3(o.hits[k].pos, e.pos);
          put3(o.hits[k].nrm, e.nrm);
        }
      }
    }
  }
  o.seed_end = smp.seed;
}

}  // namespace etxb

namespace {

template <class Q, class R>
using QueryKernel = void (*)(DeviceScene, const Q*, uint32_t, uint32_t, R*);

// The host side of every query hook.  After the common refusals, `check` validates the queries against the scene (on the context's
// device); then the queries go up, the kernel instantiation of the scene's build (RGB or spectral) runs over them and the result records
// come back.  Each (query, repetition) has its own thread and record, at most 2^31 of them, unless `stats` is set: then each query has one
// thread that loops over the repetitions and writes `stats` records.  `zero_fill` clears the records first, for kernels that write only
// some fields.
template <class Q, class R, class Check>
int run_queries(etxb_ctx* ctx, const Q* queries, uint32_t count, uint32_t repetitions, R* out, QueryKernel<Q, R> rgb, QueryKernel<Q, R> spectral,
                Check&& check, uint32_t stats = 0u, bool zero_fill = false) {
  if (!ctx || !queries || !out || (repetitions == 0)) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (count == 0) return ETXB_OK;
  if (!stats && (uint64_t(count) * repetitions > 0x7fffffffull))
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "%u queries x %u repetitions exceed 2^31 samples", count, repetitions);
  cudaSetDevice(ctx->device);
  if (int rc = check()) return rc;
  const uint32_t threads = stats ? count : count * repetitions;
  DevBuf<Q> d_queries;
  DevBuf<R> d_out;
  if (int rc = upload(ctx, d_queries, queries, count)) return rc;
  CUDA_OK(ctx, d_out.alloc(stats ? size_t(count) * stats : threads));
  if (zero_fill) CUDA_OK(ctx, cudaMemsetAsync(d_out.ptr, 0, d_out.bytes(), ctx->stream));
  (ctx->spectral ? spectral : rgb)<<<blocks_for(threads, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaGetLastError());
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(out, d_out.ptr, d_out.bytes(), cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

}  // namespace

int etxb_debug_trace(etxb_ctx* ctx, const float* rays, uint32_t* seeds, uint32_t count, float* hits_uv_t, uint32_t* hits_tri) {
  if (!ctx || !rays || !seeds || !hits_uv_t || !hits_tri) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  cudaSetDevice(ctx->device);
  DevBuf<float> d_rays, d_uvt;
  DevBuf<uint32_t> d_seeds, d_tri;
  if (int rc = upload(ctx, d_rays, rays, size_t(count) * 8)) return rc;
  if (int rc = upload(ctx, d_seeds, seeds, count)) return rc;
  CUDA_OK(ctx, d_uvt.alloc(size_t(count) * 3));
  CUDA_OK(ctx, d_tri.alloc(count));
  const uint32_t wide = (ctx->debug_trace_wide && (ctx->dscene.wide_nodes != nullptr)) ? 1u : 0u;
  k_debug_trace<<<blocks_for(count, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_rays.ptr, d_seeds.ptr, count, wide, d_uvt.ptr, d_tri.ptr);
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(seeds, d_seeds.ptr, size_t(count) * 4, cudaMemcpyDeviceToHost));
  CUDA_OK(ctx, cudaMemcpy(hits_uv_t, d_uvt.ptr, d_uvt.bytes(), cudaMemcpyDeviceToHost));
  CUDA_OK(ctx, cudaMemcpy(hits_tri, d_tri.ptr, d_tri.bytes(), cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

int etxb_debug_occluded(etxb_ctx* ctx, const float* segments, uint32_t count, uint32_t* occluded) {
  if (!ctx || !segments || !occluded) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (count == 0) return ETXB_OK;
  cudaSetDevice(ctx->device);
  DevBuf<float> d_segments;
  DevBuf<uint32_t> d_occluded;
  if (int rc = upload(ctx, d_segments, segments, size_t(count) * 6)) return rc;
  CUDA_OK(ctx, d_occluded.alloc(count));
  const uint32_t wide = (ctx->debug_trace_wide && (ctx->dscene.wide_nodes != nullptr)) ? 1u : 0u;
  k_debug_occluded<<<blocks_for(count, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_segments.ptr, count, wide, d_occluded.ptr);
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(occluded, d_occluded.ptr, d_occluded.bytes(), cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

// Test hook: both trees of a triangle soup from the host builder (the specification) or from the device builder, nothing committed
int etxb_debug_build_trees(etxb_ctx* ctx, const float* positions, uint32_t vertex_count, const uint32_t* indices, uint32_t triangle_count, uint32_t device,
  etxb_debug_trees* out) {
  if (!ctx || !out || !out->bvh_nodes || !out->tri_pos || !out->tri_index || !out->wide_nodes || (device > 1u)) return ETXB_ERR_INVALID_ARGUMENT;
  if ((triangle_count && !indices) || (vertex_count && !positions)) return ETXB_ERR_INVALID_ARGUMENT;
  for (uint64_t i = 0; i < uint64_t(triangle_count) * 3u; ++i)
    if (indices[i] >= vertex_count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "triangle %llu: vertex index out of range", (unsigned long long)(i / 3u));
  const size_t cap = std::max<uint32_t>(triangle_count, 1u);
  auto t0 = std::chrono::steady_clock::now();
  if (device == 0u) {
    Bvh bvh;
    build_bvh(positions, 12u, indices, 12u, triangle_count, bvh);
    WideBvh wide;
    build_wide_bvh(bvh, wide);
    out->seconds = seconds_since(t0);
    memcpy(out->bvh_nodes, bvh.nodes.data(), bvh.nodes.size() * sizeof(BvhNode));
    memcpy(out->tri_pos, bvh.tri_pos.data(), bvh.tri_pos.size() * sizeof(F4));
    memcpy(out->tri_index, bvh.tri_index.data(), bvh.tri_index.size() * 4u);
    memcpy(out->wide_nodes, wide.nodes.data(), wide.nodes.size() * sizeof(WideNode));
    out->bvh_node_count = uint32_t(bvh.nodes.size());
    out->slot_count = uint32_t(bvh.tri_index.size());
    out->wide_node_count = uint32_t(wide.nodes.size());
    out->max_depth = bvh.max_depth;
    out->max_stack = wide.max_stack;
    return ETXB_OK;
  }
  cudaSetDevice(ctx->device);
  DevBuf<float> d_pos;
  DevBuf<uint32_t> d_idx;
  if (int rc = upload(ctx, d_pos, positions, size_t(vertex_count) * 3u)) return rc;
  if (int rc = upload(ctx, d_idx, indices, size_t(triangle_count) * 3u)) return rc;
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  t0 = std::chrono::steady_clock::now();
  DeviceBvhOut bvh;
  CUDA_OK(ctx, build_bvh_device(d_pos.ptr, 12u, d_idx.ptr, 12u, triangle_count, true, ctx->stream, bvh));
  DevBuf<BvhNode> nodes;
  DevBuf<F4> tri_pos;
  DevBuf<uint32_t> tri_index;
  adopt(nodes, bvh.nodes, cap);
  adopt(tri_pos, bvh.tri_pos, cap * 3u);
  adopt(tri_index, bvh.tri_index, cap);
  DevBuf<WideNode> wide;
  WideNode* w = nullptr;
  uint32_t wide_count = 0, max_stack = 0;
  CUDA_OK(ctx, build_wide_bvh_device(bvh.nodes, bvh.node_count, ctx->stream, &w, &wide_count, &max_stack));
  adopt(wide, w, wide_count);
  out->seconds = seconds_since(t0);
  CUDA_OK(ctx, cudaMemcpy(out->bvh_nodes, bvh.nodes, size_t(bvh.node_count) * sizeof(BvhNode), cudaMemcpyDeviceToHost));
  CUDA_OK(ctx, cudaMemcpy(out->tri_pos, bvh.tri_pos, size_t(bvh.slot_count) * 3u * sizeof(F4), cudaMemcpyDeviceToHost));
  CUDA_OK(ctx, cudaMemcpy(out->tri_index, bvh.tri_index, size_t(bvh.slot_count) * 4u, cudaMemcpyDeviceToHost));
  CUDA_OK(ctx, cudaMemcpy(out->wide_nodes, w, size_t(wide_count) * sizeof(WideNode), cudaMemcpyDeviceToHost));
  out->bvh_node_count = bvh.node_count;
  out->slot_count = bvh.slot_count;
  out->wide_node_count = wide_count;
  out->max_depth = bvh.max_depth;
  out->max_stack = max_stack;
  return ETXB_OK;
}

// Test hook: which tree etxb_debug_trace and etxb_debug_occluded walk (0: the BVH2 shared with the oracle; 1: the 4-wide quantised tree of the product build).  Returns 1
// when the requested tree exists for the uploaded scene.
int etxb_debug_select_tree(etxb_ctx* ctx, int wide) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  ctx->debug_trace_wide = wide != 0;
  return (!wide || (ctx->dscene.wide_nodes != nullptr)) ? 1 : 0;
}

int etxb_debug_sampler(etxb_ctx* ctx, const uint32_t* a, const uint32_t* b, uint32_t count, uint32_t draws, uint32_t* out_seed, float* out_values) {
  if (!ctx || !a || !b || !out_seed || !out_values) return ETXB_ERR_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  DevBuf<uint32_t> da, db, ds;
  DevBuf<float> dv;
  if (int rc = upload(ctx, da, a, count)) return rc;
  if (int rc = upload(ctx, db, b, count)) return rc;
  CUDA_OK(ctx, ds.alloc(size_t(count) * (draws + 1)));
  CUDA_OK(ctx, dv.alloc(size_t(count) * std::max(draws, 1u)));
  k_debug_sampler<<<blocks_for(count, 128), 128, 0, ctx->stream>>>(da.ptr, db.ptr, count, draws, ds.ptr, dv.ptr);
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(out_seed, ds.ptr, ds.bytes(), cudaMemcpyDeviceToHost));
  if (draws) CUDA_OK(ctx, cudaMemcpy(out_values, dv.ptr, size_t(count) * draws * 4, cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

int etxb_debug_math(etxb_ctx* ctx, uint32_t fn, const float* x, const float* y, uint32_t count, float* out) {
  if (!ctx || !x || !out) return ETXB_ERR_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  DevBuf<float> dx, dy, dout;
  if (int rc = upload(ctx, dx, x, count)) return rc;
  if (y)
    if (int rc = upload(ctx, dy, y, count)) return rc;
  CUDA_OK(ctx, dout.alloc(count));
  k_debug_math<<<blocks_for(count, 128), 128, 0, ctx->stream>>>(ctx->dscene, fn, dx.ptr, y ? dy.ptr : nullptr, count, dout.ptr);
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(out, dout.ptr, dout.bytes(), cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

// Test hook: the vertex closures of dclosure.cuh, query by query (layout and outputs in include/etx_b200.h)
int etxb_debug_closure_eval(etxb_ctx* ctx, const etxb_closure_query* queries, uint32_t count, uint32_t repetitions, double* out) {
  const auto check = [&]() -> int {
    for (uint32_t i = 0; i < count; ++i) {
      if (queries[i].material >= ctx->materials.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "closure query material index out of range");
    }
    return ETXB_OK;
  };
  return run_queries(ctx, queries, count, repetitions, out, k_debug_closure<false>, k_debug_closure<true>, check, ETXB_CLOSURE_STATS);
}

// Test hook: bsdf_sample of dbsdf.cuh, query by query and repetition by repetition (layout and modes in include/etx_b200.h)
int etxb_debug_bsdf_sample(etxb_ctx* ctx, const etxb_sample_query* queries, uint32_t count, uint32_t repetitions, etxb_sample_result* out) {
  const auto check = [&]() -> int {
    for (uint32_t i = 0; i < count; ++i) {
      if (queries[i].material >= ctx->materials.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "sample query %u: material index out of range", i);
      if (queries[i].mode > 1u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "sample query %u: mode must be 0 or 1", i);
    }
    return ETXB_OK;
  };
  return run_queries(ctx, queries, count, repetitions, out, k_debug_bsdf_sample<false>, k_debug_bsdf_sample<true>, check);
}

// Test hook: the emitter routines of dvcm.cuh, query by query and repetition by repetition (layout and ops in include/etx_b200.h)
int etxb_debug_emitter(etxb_ctx* ctx, const etxb_emitter_query* queries, uint32_t count, uint32_t repetitions, etxb_emitter_result* out) {
  const auto check = [&]() -> int {
    if (ctx->emitters.count == 0) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "the scene has no emitter");
    for (uint32_t i = 0; i < count; ++i) {
      if (queries[i].op > ETXB_EMITTER_RADIANCE) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter query %u: op must be 0 to 3", i);
      const bool indexed = (queries[i].op == ETXB_EMITTER_SAMPLE_IN) || (queries[i].op == ETXB_EMITTER_RADIANCE);
      if (indexed && (queries[i].emitter >= ctx->emitters.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter query %u: emitter index out of range", i);
    }
    return ETXB_OK;
  };
  return run_queries(ctx, queries, count, repetitions, out, k_debug_emitter<false>, k_debug_emitter<true>, check);
}

// Test hook: the media routines of dmedium.cuh and the shadow-ray walk of dtrace.cuh, query by query and repetition by repetition (layout
// and ops in include/etx_b200.h).  Every query is checked before the launch against what makes those loops end: a finite local segment,
// tracking steps that still advance t in float32, and a free-flight redraw loop that ends in a few thousand draws on average.
namespace {
constexpr double kMediumCoordMax = 1e15;       // |world coordinate| of an origin or an end point
constexpr double kMediumLocalSegmentMax = 1e18;  // local segment length: its float32 square stays finite
constexpr double kMediumTrackingMax = 65536.0;   // max_sigma x (|local origin| + 2): a mean tracking step of ~1000 float32 ulps of t or more
constexpr double kMediumRedrawMax = 8.0;         // extinction x kRayEpsilon: the homogeneous redraw loop runs exp(8) ~ 3000 times on average

// A heterogeneous medium's tracking from a to b (world points; b = nullptr: a only) ends: finite local points, a local segment whose
// float32 length is finite, and steps of 1 / max_sigma well above an ulp of the local t.
bool tracking_bounded(const DMedium& m, const double* a, const double* b) {
  if ((m.cls != 1u) || !(m.max_sigma > 0.0f)) return true;
  const double lo[3] = {m.bounds_min.x, m.bounds_min.y, m.bounds_min.z}, hi[3] = {m.bounds_max.x, m.bounds_max.y, m.bounds_max.z};
  double magnitude = 0.0, length2 = 0.0;
  for (int k = 0; k < 3; ++k) {
    const double ext = hi[k] - lo[k];
    if (!(ext > 0.0)) return false;
    const double pa = (a[k] - lo[k]) / ext, pb = b ? (b[k] - lo[k]) / ext : pa;
    if (!std::isfinite(pa) || !std::isfinite(pb)) return false;
    magnitude = std::max(magnitude, std::fabs(pa));
    length2 += (pb - pa) * (pb - pa);
  }
  return (std::sqrt(length2) <= kMediumLocalSegmentMax) && (double(m.max_sigma) * (magnitude + 2.0) <= kMediumTrackingMax);
}

double spectrum_max(const std::vector<DSpectrum>& spectra, uint32_t index) {
  if (index >= spectra.size()) return 0.0;
  const DSpectrum& s = spectra[index];
  double v = std::max({double(s.rgb[0]), double(s.rgb[1]), double(s.rgb[2])});
  for (float p : s.power) v = std::max(v, double(p));
  return v;
}
}  // namespace

int etxb_debug_medium(etxb_ctx* ctx, const etxb_medium_query* queries, uint32_t count, uint32_t repetitions, etxb_medium_result* out) {
  const auto check = [&]() -> int {
    std::vector<DMedium> meds(ctx->mediums.count);
    std::vector<DSpectrum> spectra(ctx->spectra.count);
    if (!meds.empty()) CUDA_OK(ctx, cudaMemcpy(meds.data(), ctx->mediums.ptr, meds.size() * sizeof(DMedium), cudaMemcpyDeviceToHost));
    if (!spectra.empty()) CUDA_OK(ctx, cudaMemcpy(spectra.data(), ctx->spectra.ptr, spectra.size() * sizeof(DSpectrum), cudaMemcpyDeviceToHost));
    const auto bounded3 = [](const float* v) {
      return (std::fabs(double(v[0])) <= kMediumCoordMax) && (std::fabs(double(v[1])) <= kMediumCoordMax) && (std::fabs(double(v[2])) <= kMediumCoordMax);
    };
    for (uint32_t i = 0; i < count; ++i) {
      const etxb_medium_query& q = queries[i];
      if (q.op > ETXB_MEDIUM_SEGMENT) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: op must be 0 to 5", i);
      if (ctx->spectral && !std::isfinite(q.wavelength)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: non-finite wavelength", i);
      const bool unset = (q.op == ETXB_MEDIUM_SEGMENT) && (q.medium == ETXB_INVALID_INDEX);
      if ((q.op != ETXB_MEDIUM_PHASE) && !unset && (q.medium >= meds.size())) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: medium index out of range", i);
      if ((q.op == ETXB_MEDIUM_DENSITY) && (ctx->medium_density[q.medium].count == 0)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: density of a homogeneous medium", i);
      if ((q.op != ETXB_MEDIUM_PHASE) && !bounded3(q.origin)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: origin not finite or past 1e15", i);
      const double o[3] = {q.origin[0], q.origin[1], q.origin[2]};
      if (q.op == ETXB_MEDIUM_SEGMENT) {
        if (!bounded3(q.end)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: segment end not finite or past 1e15", i);
        // every medium the walk can track through starts from a point of the segment: bound both ends in each heterogeneous medium
        const double e[3] = {q.end[0], q.end[1], q.end[2]};
        for (const DMedium& m : meds) {
          if (!tracking_bounded(m, o, e) || !tracking_bounded(m, e, o)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: segment too far from a heterogeneous medium to track", i);
        }
        continue;
      }
      if (q.op == ETXB_MEDIUM_DENSITY) continue;
      const float* d = q.direction;
      if (!std::isfinite(d[0]) || !std::isfinite(d[1]) || !std::isfinite(d[2]) || ((d[0] == 0.0f) && (d[1] == 0.0f) && (d[2] == 0.0f)))
        return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: zero or non-finite direction", i);
      if (q.op == ETXB_MEDIUM_PHASE) continue;
      if (!std::isfinite(q.max_t) && (q.max_t != kMaxFloat)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: non-finite max_t", i);
      if ((q.op == ETXB_MEDIUM_SAMPLE) && !(q.max_t >= kRayEpsilon)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: sample needs max_t >= kRayEpsilon", i);
      if (!std::isfinite(q.throughput[0]) || !std::isfinite(q.throughput[1]) || !std::isfinite(q.throughput[2]))
        return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: non-finite throughput", i);
      const DMedium& m = meds[q.medium];
      if (q.max_t < kMaxFloat) {  // medium_intersects_bounds refuses max_t = kMaxFloat before any arithmetic
        double e[3];
        for (int k = 0; k < 3; ++k) e[k] = o[k] + double(d[k]) * double(q.max_t);
        if (!(std::fabs(e[0]) <= 1e30) || !(std::fabs(e[1]) <= 1e30) || !(std::fabs(e[2]) <= 1e30))
          return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: the segment's end overflows", i);
        if (!tracking_bounded(m, o, e)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: segment too long or too far from the medium to track", i);
      }
      if ((q.op == ETXB_MEDIUM_SAMPLE) && (m.cls == 0u) &&
          ((spectrum_max(spectra, m.absorption_index) + spectrum_max(spectra, m.scattering_index)) * kRayEpsilon > kMediumRedrawMax))
        return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium query %u: extinction too high for the free-flight redraw loop", i);
    }
    return ETXB_OK;
  };
  return run_queries(ctx, queries, count, repetitions, out, k_debug_medium<false>, k_debug_medium<true>, check);
}

// Test hook: the subsurface routines of dsss.cuh, query by query and repetition by repetition (layout and ops in include/etx_b200.h).
// Every loop they run is bounded (a traversal of the tree, at most 1024 random-walk steps), so the checks are on indices and finite inputs.
int etxb_debug_subsurface(etxb_ctx* ctx, const etxb_subsurface_query* queries, uint32_t count, uint32_t repetitions, etxb_subsurface_result* out) {
  const auto check = [&]() -> int {
    std::vector<etxb_material> mats(ctx->materials.count);
    std::vector<DTriangle> tris(ctx->triangles.count);
    if (!mats.empty()) CUDA_OK(ctx, cudaMemcpy(mats.data(), ctx->materials.ptr, mats.size() * sizeof(etxb_material), cudaMemcpyDeviceToHost));
    if (!tris.empty()) CUDA_OK(ctx, cudaMemcpy(tris.data(), ctx->triangles.ptr, tris.size() * sizeof(DTriangle), cudaMemcpyDeviceToHost));
    const auto finite = [](const float* v, int n) {
      for (int k = 0; k < n; ++k)
        if (!std::isfinite(v[k])) return false;
      return true;
    };
    for (uint32_t i = 0; i < count; ++i) {
      const etxb_subsurface_query& q = queries[i];
      if (q.op > ETXB_SUBSURFACE_GATHER) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: op must be 0 to 4", i);
      if (ctx->spectral && !std::isfinite(q.wavelength)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: non-finite wavelength", i);
      if (q.op == ETXB_SUBSURFACE_REMAP) {
        if (!finite(q.color, 3) || !finite(q.distances, 3)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: non-finite color or distance", i);
        continue;
      }
      const float* d = q.dir;
      if (!finite(d, 3) || ((d[0] == 0.0f) && (d[1] == 0.0f) && (d[2] == 0.0f)))
        return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: zero or non-finite direction", i);
      if (q.op <= ETXB_SUBSURFACE_CONTINUOUS_TRACE) {
        if ((q.material != ETXB_INVALID_INDEX) && (q.material >= mats.size())) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: material index out of range", i);
        if (!finite(q.origin, 3) || !std::isfinite(q.t_min) || !std::isfinite(q.t_max))
          return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: non-finite origin or ray interval", i);
        if ((q.op == ETXB_SUBSURFACE_CONTINUOUS_TRACE) && ((q.max_count == 0) || (q.max_count > 8u)))
          return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: max_count must be 1 to 8", i);
        continue;
      }
      if (q.triangle >= tris.size()) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: triangle index out of range", i);
      if (!std::isfinite(q.u) || !std::isfinite(q.v)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: non-finite barycentric coordinates", i);
      if (q.op == ETXB_SUBSURFACE_PROFILE) {
        if (q.direction > 2u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: probe direction must be 0 to 2", i);
        if (!std::isfinite(q.rnd) || !std::isfinite(q.radius) || !finite(q.normal, 3))
          return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: non-finite rnd, radius or normal", i);
      } else if (mats[tris[q.triangle].material_index].subsurface.cls == 0u) {
        return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "subsurface query %u: gather on a material without subsurface scattering", i);
      }
    }
    return ETXB_OK;
  };
  return run_queries(ctx, queries, count, repetitions, out, k_debug_subsurface<false>, k_debug_subsurface<true>, check, 0u, /*zero_fill=*/true);
}
