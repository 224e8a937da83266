// kernels_pt.cuh — wavefront kernels of the unidirectional path tracer (SURVEY §8(f) N3; included once, by module.cu, after kernels.cuh).
//
// Reference: CPUPathTracingImpl::execute_range (sources/etx/rt/integrators/path_tracing.cxx:50-83), run_path_iteration
// (rt/shared/path_tracing_shared.hxx:485-510), Film::accumulate_camera_image with the normal / albedo layers and the adaptive-sampling history
// (render/host/film.cxx:173-230), Film::active_pixel (:434-461), Film::estimate_noise_levels (:233-330).
//
// Stage list of one iteration:
//   k_pt_begin -> { k_trace_closest* -> [sort by material] -> k_pt_shade [-> k_shadow_resolve] }* -> k_pt_accumulate
//     -> [k_film_noise_level -> (all-reduce of the active mask over the ranks) -> k_film_noise_dilate]
// The payload lives in the VCM camera path's SoA columns (one PathBuffers allocation serves both integrators): thr.w = sampled_bsdf_pdf,
// mis.x = eta, misc = (seed, path_length, medium, mis_weight), gathered = accumulated, bs_weight_pdf = view_albedo, bs_wo_eta = view_normal.
#pragma once
#include "dpt.cuh"

namespace etxb {

// the film layers only the path tracer writes (film.cxx:14-40) — storage is y-flipped like the camera layer
struct PtFilm {
  float4* normals;
  float4* albedo;
  float4* adaptive;      // StorageCameraAdaptive: the mean over every other sample
  uint32_t* info;        // InternalData: sample_count (bits 0-29), converged (bit 30), tmp (bit 31)
  float* error_level;
};
constexpr uint32_t kPtConverged = 1u << 30u;
constexpr uint32_t kPtTmp = 1u << 31u;
constexpr uint32_t kPtCountMask = kPtConverged - 1u;

template <bool SP>
DEV void pt_store(const PathBuffers& b, uint32_t i, const PtState<SP>& s) {
  V3 t = s.throughput.as_v3(), a = s.accumulated.as_v3();
  b.ray_o[i] = make_float4(s.ray_o.x, s.ray_o.y, s.ray_o.z, s.ray_min_t);
  b.ray_d[i] = make_float4(s.ray_d.x, s.ray_d.y, s.ray_d.z, s.ray_max_t);
  b.thr[i] = make_float4(t.x, t.y, t.z, s.sampled_bsdf_pdf);
  b.mis[i] = make_float4(s.eta, 0.0f, 0.0f, 0.0f);
  b.misc[i] = make_uint4(s.smp.seed, s.path_length, s.medium, s.mis_weight ? 1u : 0u);
  b.gathered[i] = make_float4(a.x, a.y, a.z, 0.0f);
}
template <bool SP>
DEV PtState<SP> pt_load(const PathBuffers& b, uint32_t i) {
  PtState<SP> s;
  float4 o = b.ray_o[i], d = b.ray_d[i], t = b.thr[i], a = b.gathered[i];
  uint4 u = b.misc[i];
  s.ray_o = {o.x, o.y, o.z};
  s.ray_min_t = o.w;
  s.ray_d = {d.x, d.y, d.z};
  s.ray_max_t = d.w;
  s.throughput = Spec<SP>::make3({t.x, t.y, t.z});
  s.sampled_bsdf_pdf = t.w;
  s.accumulated = Spec<SP>::make3({a.x, a.y, a.z});
  s.eta = b.mis[i].x;
  s.smp = Smp::resume(u.x);
  s.path_length = u.y;
  s.medium = u.z;
  s.mis_weight = (u.w & 1u) != 0u;
  s.wavelength = b.wavelength[i];
  s.view_albedo = Spec<SP>::make(0.0f);
  s.view_normal = {0.0f, 0.0f, 0.0f};
  return s;
}

// storage index (y-flipped) of film pixel i = x + y * width
DEV uint32_t pt_film_index(const FilmBuffers& film, uint32_t i) {
  uint32_t px = i % film.width, py = i / film.width;
  return px + (film.height - 1u - py) * film.width;
}

// make_ray_payload for every active pixel (path_tracing.cxx:57-62; Film::active_pixel: a path whose pixel has converged is skipped)
template <bool SP>
__global__ void __launch_bounds__(128) k_pt_begin(const __grid_constant__ LaunchParams p, const __grid_constant__ PtParams pt, const __grid_constant__ PtFilm pf, uint32_t* queue,
                                                  uint32_t* queue_count) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool alive = false;
  if (i < p.path_count) {
    const uint32_t pixel = film_path_pixel(p.film, i, pt.iteration);
    alive = pixel_owned(p, pixel) && ((pf.info[pt_film_index(p.film, pixel)] & kPtConverged) == 0u);
    if (alive) {
      PtState<SP> s = pt_make_payload<SP>(p.scene, pt, pixel % p.film.width, pixel / p.film.width, i);
      p.paths.wavelength[i] = s.wavelength;
      pt_store<SP>(p.paths, i, s);
      p.paths.bs_weight_pdf[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      p.paths.bs_wo_eta[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      // run_path_iteration's first test (:486): a path longer than the limit is not traced at all
      alive = s.path_length <= p.scene.max_path_length;
      if (!alive) p.sampler_end_camera[i] = s.smp.seed;
    } else {
      // a pixel that is skipped (converged, or another rank's tile) has no path in this iteration: its debug taps read zero, like the oracle's
      p.sampler_end_camera[i] = 0u;
      p.camera_value[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
  }
  queue_push(queue, queue_count, alive, i);
}

// run_path_iteration after the trace (:485-510): medium event, surface hit or miss.  A path that goes on is queued for the next bounce; one that
// ends leaves its sums in the path columns for k_pt_accumulate.
template <bool SP, bool PLAIN>
__global__ void __launch_bounds__(128, kBounceMinBlocksPerSm<PLAIN>) k_pt_shade(const __grid_constant__ LaunchParams p, const __grid_constant__ PtParams pt, const uint32_t* queue_in,
                                                                           const uint32_t* count_in, uint32_t* queue_out, uint32_t* count_out) {
  uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t shadow_rays = 0, i = 0;
  bool alive = false;
  STATS_DECL;
  if (q < *count_in) {
    i = queue_in[q];
    const DeviceScene& sc = p.scene;
    PtState<SP> s = pt_load<SP>(p.paths, i);
    float4 hit = p.paths.hit[i];
    const uint32_t tri_index = __float_as_uint(hit.w);
    const bool found = tri_index != kInvalidIndex;
    MediumSample<SP> ms;
    ms.weight = Spec<SP>::make(0.0f);
    ms.pos = {0.0f, 0.0f, 0.0f};
    ms.sampled_medium_t = 0.0f;
    if constexpr (!PLAIN) {
      if (s.medium != kInvalidIndex) {  // try_sampling_medium (:259-268)
        ms = sample_medium<SP>(sc, sc.mediums[s.medium], s.wavelength, s.throughput, s.smp, s.ray_o, s.ray_d, found ? hit.z : kMaxFloat);
        s.throughput *= ms.weight;
      }
    }
    if (ms.sampled_medium()) {
      if constexpr (!PLAIN) {
        pt_handle_sampled_medium<SP, PLAIN>(sc, pt, ms, s, stats, shadow_rays);
        alive = random_continue<SP>(s.path_length, sc.random_path_termination, s.eta, s.smp, s.throughput);
      }
    } else if (found) {
      Isect isect = make_intersection(sc, s.ray_d, tri_index, hit.x, hit.y, hit.z);
      ShadowBatch batch = {p.shadow_p0, p.shadow_p1, p.shadow_value, 0u, 0u};
      ShadowBatch* deferred = nullptr;
      if (PLAIN && p.shadow_atomic) {
        batch.atomic_cursor = p.shadow_count;
        batch.capacity = p.shadow_capacity;
        batch.target = i;
        deferred = &batch;
      }
      const bool first = s.path_length == 1u;
      const uint32_t pixel = film_path_pixel(p.film, i, pt.iteration);
      alive = pt_handle_hit_ray<SP, PLAIN>(sc, pt, isect, pixel % p.film.width, pixel / p.film.width, s, stats, shadow_rays, deferred);
      if (first) {
        V3 a = s.view_albedo.as_v3();
        p.paths.bs_weight_pdf[i] = make_float4(a.x, a.y, a.z, 0.0f);
        p.paths.bs_wo_eta[i] = make_float4(s.view_normal.x, s.view_normal.y, s.view_normal.z, 0.0f);
      }
    } else if (pt.direct) {
      pt_handle_missed_ray<SP>(sc, s);
    }
    // the next run_path_iteration call starts with the length test (:486)
    alive = alive && (s.path_length <= sc.max_path_length);
    pt_store<SP>(p.paths, i, s);
    if (!alive) p.sampler_end_camera[i] = s.smp.seed;
  }
  queue_push(queue_out, count_out, alive, i);
  counter_add(&p.counters->bounces_camera, (q < *count_in) ? 1u : 0u);
  counter_add(&p.counters->rays_shadow, shadow_rays);
  counter_add(&p.counters->nodes, STATS_NODES);
  counter_add(&p.counters->tris, STATS_TRIS);
}

// The end of execute_range's loop body (path_tracing.cxx:68-81) + Film::accumulate_camera_image (film.cxx:173-230) for every pixel that was
// active in this iteration: colour, normal and albedo running means, the every-other-sample mean the noise estimate compares against, the
// per-pixel sample counter.  At pixel size > 1 the path leaves colour (camera_value), albedo (bs_weight_pdf) and normal (bs_wo_eta) for
// k_film_fill_blocks.
template <bool SP>
__global__ void __launch_bounds__(256) k_pt_accumulate(const __grid_constant__ LaunchParams p, const __grid_constant__ PtParams pt, const __grid_constant__ PtFilm pf) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.path_count) return;
  const uint32_t pixel = film_path_pixel(p.film, i, pt.iteration);
  const uint32_t fi = pt_film_index(p.film, pixel);
  const uint32_t info = pf.info[fi];
  if (!pixel_owned(p, pixel) || (info & kPtConverged)) return;
  const float wavelength = p.paths.wavelength[i];
  float4 acc = p.paths.gathered[i], alb = p.paths.bs_weight_pdf[i], nrm = p.paths.bs_wo_eta[i];
  const float pdf = sampling_pdf<SP>(wavelength);
  V3 normal = {nrm.x, nrm.y, nrm.z};
  V3 albedo = spec_to_rgb<SP>(p.scene, Spec<SP>::make3({alb.x, alb.y, alb.z}) / pdf, wavelength);
  V3 color = spec_to_rgb<SP>(p.scene, Spec<SP>::make3({acc.x, acc.y, acc.z}) / pdf, wavelength);
  if ((pt.radiance_clamp > 0.0f) && (p.paths.misc[i].y > 1u)) {
    float lum = luminance(color);
    if (lum > pt.radiance_clamp) color *= pt.radiance_clamp / lum;
  }
  if (p.film.pixel_size != 1u) {
    p.paths.bs_weight_pdf[i] = make_float4(albedo.x, albedo.y, albedo.z, 0.0f);
    p.camera_value[i] = make_float4(color.x, color.y, color.z, 0.0f);
    return;
  }
  const uint32_t sample_index = info & kPtCountMask;
  float4 c_old = p.film.camera[fi], n_old = pf.normals[fi], a_old = pf.albedo[fi], v_old = pf.adaptive[fi];
  V3 c = color, n = normal, a = albedo, v = color;
  if (sample_index != 0u) {
    double ds = double(sample_index);
    float t = float(ds / (ds + 1.0));
    c = {lerpf(color.x, c_old.x, t), lerpf(color.y, c_old.y, t), lerpf(color.z, c_old.z, t)};
    n = {lerpf(normal.x, n_old.x, t), lerpf(normal.y, n_old.y, t), lerpf(normal.z, n_old.z, t)};
    a = {lerpf(albedo.x, a_old.x, t), lerpf(albedo.y, a_old.y, t), lerpf(albedo.z, a_old.z, t)};
    v = {v_old.x, v_old.y, v_old.z};
    if ((sample_index % 2u) == 0u) {
      t = float(ds / (ds + 2.0));
      v = {lerpf(color.x, v_old.x, t), lerpf(color.y, v_old.y, t), lerpf(color.z, v_old.z, t)};
    }
  }
  p.film.camera[fi] = make_float4(c.x, c.y, c.z, 1.0f);
  pf.normals[fi] = make_float4(n.x, n.y, n.z, 1.0f);
  pf.albedo[fi] = make_float4(a.x, a.y, a.z, 1.0f);
  pf.adaptive[fi] = make_float4(v.x, v.y, v.z, 1.0f);
  pf.info[fi] = (info & ~kPtCountMask) | ((sample_index + 1u) & kPtCountMask);
  p.camera_value[i] = make_float4(color.x, color.y, color.z, 0.0f);
}

// Film::accumulate_camera_image at pixel size s > 1 (film.cxx:173-230): the reference loops over the block of the path's pixel, clipped to
// the film; here every film pixel reads its block's path and lerps with its own sample count — coalesced writes, the same cost for any s.
// VCM: the camera layer, every block every iteration.  PT: also normal, albedo, the every-other-sample mean and the count, for the blocks
// whose path ran (its chosen pixel had not converged; the other pixels of the block are not tested, as in the reference).
template <bool PT>
__global__ void __launch_bounds__(256) k_film_fill_blocks(const __grid_constant__ LaunchParams p, const __grid_constant__ PtFilm pf, uint32_t iteration) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const FilmBuffers& film = p.film;
  if (i >= film.width * film.height) return;
  const uint32_t px = i % film.width, py = film.height - 1u - i / film.width;
  const uint32_t path = (px / film.pixel_size) + (py / film.pixel_size) * film.dims_x;
  uint32_t sample_index = p.camera_sample_index, info = 0u;
  if constexpr (PT) {
    if (pf.info[pt_film_index(film, film_path_pixel(film, path, iteration))] & kPtConverged) return;
    info = pf.info[i];
    sample_index = info & kPtCountMask;
  }
  const float4 cv = p.camera_value[path];
  const V3 color = {cv.x, cv.y, cv.z};
  const float4 c_old = film.camera[i];
  V3 c = color;
  double ds = double(sample_index);
  float t = float(ds / (ds + 1.0));
  if (sample_index != 0u) c = {lerpf(color.x, c_old.x, t), lerpf(color.y, c_old.y, t), lerpf(color.z, c_old.z, t)};
  film.camera[i] = make_float4(c.x, c.y, c.z, 1.0f);
  if constexpr (PT) {
    const float4 nrm = p.paths.bs_wo_eta[path], alb = p.paths.bs_weight_pdf[path];
    const V3 normal = {nrm.x, nrm.y, nrm.z}, albedo = {alb.x, alb.y, alb.z};
    const float4 n_old = pf.normals[i], a_old = pf.albedo[i], v_old = pf.adaptive[i];
    V3 n = normal, a = albedo, v = color;
    if (sample_index != 0u) {
      n = {lerpf(normal.x, n_old.x, t), lerpf(normal.y, n_old.y, t), lerpf(normal.z, n_old.z, t)};
      a = {lerpf(albedo.x, a_old.x, t), lerpf(albedo.y, a_old.y, t), lerpf(albedo.z, a_old.z, t)};
      v = {v_old.x, v_old.y, v_old.z};
      if ((sample_index % 2u) == 0u) {
        t = float(ds / (ds + 2.0));
        v = {lerpf(color.x, v_old.x, t), lerpf(color.y, v_old.y, t), lerpf(color.z, v_old.z, t)};
      }
    }
    pf.normals[i] = make_float4(n.x, n.y, n.z, 1.0f);
    pf.albedo[i] = make_float4(a.x, a.y, a.z, 1.0f);
    pf.adaptive[i] = make_float4(v.x, v.y, v.z, 1.0f);
    pf.info[i] = (info & ~kPtCountMask) | ((sample_index + 1u) & kPtCountMask);
  }
}

// Film::estimate_noise_levels (film.cxx:233-330) as three steps that work on any set of 32x32 pixel tiles:
//   k_film_noise_level   the first pass on this rank's pixels, and the packed ACTIVE MASK: bit = 1 where a pixel has not converged after it;
//   exchange             on a context with a communicator, the ranks all-reduce (sum) the mask — every word has one owner, so the sum is the
//                        one-GPU mask — and the small stats behind it;
//   k_film_noise_dilate  the two dilation passes, read from the mask alone, written to this rank's pixels.
// Mask layout: storage row r holds ceil(W / 32) words, word k the pixels x = 32k .. 32k + 31 (bit x % 32).  A tile is 32 pixels wide and
// starts at a multiple of 32, and a storage row is one film row (y-flipped), so a word never spans two ranks.  The words of other ranks stay
// zero on a rank, and zero reads as converged.
// After the mask: kNoiseStats words, all-reduced with it (the float sum in a call of its own).
constexpr uint32_t kNoiseStatConverged = 0u;  // pixels that converged in this pass (the reference's `active_pixels`)
constexpr uint32_t kNoiseStatProcessed = 1u;  // CPUPathTracingImpl::pixels_processed of the iteration (written by the host)
constexpr uint32_t kNoiseStatError = 2u;      // bits of the float sum of the error levels of this pass
constexpr uint32_t kNoiseStats = 3u;
__host__ __device__ inline uint32_t noise_mask_words_per_row(uint32_t width) { return (width + 31u) / 32u; }

// first pass: error level of every owned pixel that has not converged, the convergence decision, the mask word (one warp per word, one ballot),
// and the two sums noise_level() is made of (atomic adds: the summation order is not the reference's, which is itself thread-order dependent).
__global__ void __launch_bounds__(256) k_film_noise_level(const __grid_constant__ FilmBuffers film, const __grid_constant__ PtFilm pf, float threshold, uint32_t rank,
                                                          uint32_t world, uint32_t* mask, uint32_t* stats) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x, lane = t & 31u, word = t >> 5u;
  const uint32_t wpr = noise_mask_words_per_row(film.width);
  const uint32_t r = word / wpr, x = (word % wpr) * 32u + lane;
  float error_level = 0.0f;
  uint32_t converged = 0u;
  bool active = false;
  if ((r < film.height) && (x < film.width) && (tile_rank(film.width, x, film.height - 1u - r, world) == rank)) {
    const uint32_t i = x + r * film.width;
    uint32_t info = pf.info[i];
    if ((info & kPtConverged) == 0u) {
      float4 c = film.camera[i], a = pf.adaptive[i];
      float error_diff = fabsf(c.x - a.x) + fabsf(c.y - a.y) + fabsf(c.z - a.z);
      float error_norm = fabsf(c.x) + fabsf(c.y) + fabsf(c.z);
      error_level = error_diff / (((error_norm < 1.0f) ? sqrtf(error_norm) : error_norm) + kEpsilon);
      converged = (error_level < threshold) ? 1u : 0u;
      active = (converged == 0u);
      pf.error_level[i] = error_level;
      pf.info[i] = (info & kPtCountMask) | (converged ? (kPtConverged | kPtTmp) : 0u);
    }
  }
  const uint32_t bits = __ballot_sync(0xffffffffu, active);
  uint32_t n = __reduce_add_sync(0xffffffffu, converged);
  float sum = error_level;
  for (uint32_t o = 16u; o > 0u; o >>= 1u) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((lane == 0u) && (r < film.height)) {
    mask[word] = bits;
    if (n) atomicAdd(stats + kNoiseStatConverged, n);
    if (sum != 0.0f) atomicAdd(reinterpret_cast<float*>(stats + kNoiseStatError), sum);
  }
}

// Which pixels of word k of a mask row have an active pixel x - 4 .. x + 5 in that row (pixels off the film read as converged)
DEV uint32_t noise_row_window(const uint32_t* row, uint32_t k, uint32_t wpr) {
  const uint32_t prev = (k > 0u) ? row[k - 1u] : 0u, cur = row[k], next = (k + 1u < wpr) ? row[k + 1u] : 0u;
  uint32_t d = cur;
#pragma unroll
  for (uint32_t s = 1u; s <= 5u; ++s) d |= __funnelshift_r(cur, next, s);  // bit x: pixel x + s
#pragma unroll
  for (uint32_t s = 1u; s <= 4u; ++s) d |= __funnelshift_l(prev, cur, s);  // bit x: pixel x - s
  return d;
}

// second and third pass (:283-320) as one gather over the mask.  The reference clears `tmp` of x - 5 .. x + 4 around every active pixel, then
// `converged` of y - 5 .. y + 4 around every pixel without `tmp`.  A pixel has `tmp` after the first pass exactly when it is not active (a pixel
// converged in an earlier estimate kept both bits), so pixel p loses `tmp` when its row window [x - 4, x + 5] holds an active pixel, and
// `converged` when the row window of any row in [y - 4, y + 5] does (test_pt_tiles_model.py checks this against the scatter form).
__global__ void __launch_bounds__(256) k_film_noise_dilate(uint32_t width, uint32_t height, uint32_t rank, uint32_t world, const uint32_t* mask, uint32_t* info) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x, lane = t & 31u, word = t >> 5u;
  const uint32_t wpr = noise_mask_words_per_row(width);
  const uint32_t r = word / wpr, k = word % wpr, x = k * 32u + lane;
  if ((r >= height) || (x >= width) || (tile_rank(width, x, height - 1u - r, world) != rank)) return;
  const uint32_t i = x + r * width;
  uint32_t v = info[i];
  if ((v & (kPtConverged | kPtTmp)) == 0u) return;  // an active pixel has neither bit to lose
  const uint32_t row = noise_row_window(mask + r * wpr, k, wpr);
  uint32_t box = row;
  const uint32_t r0 = (r >= 4u) ? (r - 4u) : 0u, r1 = umin(height - 1u, r + 5u);
  for (uint32_t q = r0; q <= r1; ++q)
    if (q != r) box |= noise_row_window(mask + q * wpr, k, wpr);
  const uint32_t bit = 1u << lane;
  if (row & bit) v &= ~kPtTmp;
  if (box & bit) v &= ~kPtConverged;
  info[i] = v;
}

// Film::layer for the layers the VCM integrator leaves empty (film.cxx:406-414): normals are shown as n * 0.5 + 0.5
__global__ void __launch_bounds__(256) k_film_layer_normals(const float4* normals, float4* out, uint32_t count) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float4 n = normals[i];
  out[i] = make_float4(n.x * 0.5f + 0.5f, n.y * 0.5f + 0.5f, n.z * 0.5f + 0.5f, 1.0f);
}

}  // namespace etxb
