// oracle_preview.cxx — the coarse preview (Film pixel size > 1) restated on top of the oracle.  TEST INFRASTRUCTURE.
//
// oracle_vcm.cxx is compiled here as it is, with four of its exports renamed (the macros below); this file adds what Film::set_pixel_size
// changes (render/host/film.cxx:147-230, 345-461; rt/integrators/vcm_cpu.cxx:95-207; path_tracing.cxx:50-83) and exports the four again:
//   * Film::dimensions() = ceil(W / s) x ceil(H / s) and pixel_count() its product: each integrator traces pixel_count() paths;
//   * Film::active_pixel: the block origin of path i offset inside the block and clamped to the film — by pm::preview_offset (portable_math.h,
//     the definition the device calls) where the reference calls rand(), which no run can repeat;
//   * VCM: the radius from dimensions() * s, eta_vcm from pixel_count(); light path i seeded with i; camera path i with the located pixel;
//   * Film::accumulate_camera_image over the pixel's block clipped to the film, each pixel with its own count;
//   * Film::atomic_add_light_iteration to the s x s pixels of the splat's block, coordinates clamped to the film.
// At pixel size 1 every call goes to oracle_vcm.cxx's own code.  Built into liboracle_preview_parity.so by build_oracle_preview.sh.
#define oracle_create oracle_full_create
#define oracle_begin oracle_full_begin
#define oracle_run_iterations oracle_full_run_iterations
#define oracle_read_buffer oracle_full_read_buffer
#include "oracle_vcm.cxx"
#undef oracle_create
#undef oracle_begin
#undef oracle_run_iterations
#undef oracle_read_buffer

#include <mutex>
#include <unordered_map>

#include "portable_math.h"

namespace etx {
namespace {

struct PreviewFilm {
  uint32_t pixel_size = 1, target_pixel_size = 1;  // Film::pixel_size and the stored target Film::clear applies (film.cxx:365)
};
std::mutex g_preview_m;
std::unordered_map<const void*, PreviewFilm> g_preview;

PreviewFilm& preview_of(const void* h) {
  std::lock_guard<std::mutex> lock(g_preview_m);
  return g_preview[h];
}

uint2 dimensions(const Oracle& o, uint32_t s) {
  return {(o.width + s - 1u) / s, (o.height + s - 1u) / s};
}
uint32_t reduced_count(const Oracle& o, uint32_t s) {
  uint2 d = dimensions(o, s);
  return d.x * d.y;
}

// Film::active_pixel (film.cxx:434-461): the pixel path `index` samples, and whether it has not converged
bool active_pixel(const Oracle& o, uint32_t s, uint32_t index, uint32_t iteration, uint2& location) {
  uint2 dim = dimensions(o, s);
  uint2 a_location = {(index % dim.x) * s, (index / dim.x) * s};
  uint32_t dx = 0, dy = 0;
  pm::preview_offset(index, iteration, s, dx, dy);
  a_location.x += dx;
  a_location.y += dy;
  uint32_t linear_index = min(a_location.x, o.width - 1u) + min(a_location.y, o.height - 1u) * o.width;
  location = {linear_index % o.width, linear_index / o.width};
  return o.film_converged[location.x + (o.height - 1u - location.y) * o.width] == 0;
}

// film.cxx:147-171: the s x s pixels of the splat's block, coordinates clamped (the last column / row of a partial block receives it more than once)
void add_light_block(Oracle& o, uint32_t s, const float3& value, const float2& ndc, bool atomic) {
  if (dot(value, value) == 0.0f)
    return;
  float2 uv = ndc * 0.5f + 0.5f;
  const uint2 dim = dimensions(o, s);
  uint32_t x = static_cast<uint32_t>(uv.x * dim.x) * s;
  uint32_t y = static_cast<uint32_t>(uv.y * dim.y) * s;
  if ((x >= o.width) || (y >= o.height))
    return;
  const uint32_t p_base_x = (x / s) * s, p_base_y = (y / s) * s;
  for (uint32_t v = 0; v < s; ++v) {
    const uint32_t py = min(p_base_y + v, o.height - 1u);
    for (uint32_t u = 0; u < s; ++u) {
      const uint32_t px = min(p_base_x + u, o.width - 1u);
      float3& dst = o.film_light_iteration[px + (o.height - 1u - py) * o.width];
      if (atomic) {
        atomic_add_f(&dst.x, value.x);
        atomic_add_f(&dst.y, value.y);
        atomic_add_f(&dst.z, value.z);
      } else {
        dst.x += value.x;
        dst.y += value.y;
        dst.z += value.z;
      }
    }
  }
}

// film.cxx:173-230: the pixel's block clipped to the film; oracle_vcm.cxx's per-pixel update (each pixel's own count) for every pixel of it
template <class F>
void for_block(const Oracle& o, uint32_t s, const uint2& pixel, F&& fn) {
  const uint32_t p_base_x = (pixel.x / s) * s, p_base_y = (pixel.y / s) * s;
  for (uint32_t py = p_base_y, pye = min(p_base_y + s, o.height); py < pye; ++py)
    for (uint32_t px = p_base_x, pxe = min(p_base_x + s, o.width); px < pxe; ++px)
      fn(uint2{px, py});
}

// start_next_iteration (vcm_cpu.cxx:95-113) with the radius from dimensions() * pixel_size() and eta_vcm from pixel_count()
void start_preview_iteration(Oracle& o, uint32_t s) {
  auto& it = o.iteration;
  float used_radius = o.options.initial_radius;
  if (used_radius == 0.0f) {
    uint2 current_dim = dimensions(o, s) * s;
    uint32_t max_dim = max(current_dim.x, current_dim.y);
    used_radius = 5.0f * o.scene.bounding_sphere_radius / float(max_dim);
  }
  float radius_scale = 1.0f / (1.0f + float(it.iteration) / float(o.options.radius_decay));
  it.current_radius = used_radius * radius_scale;
  float eta_vcm = kPi * sqr(it.current_radius) * float(reduced_count(o, s));
  it.vc_weight = 1.0f / eta_vcm;
  it.vm_weight = o.options.enable_merging() ? eta_vcm : 0.0f;
  it.vm_normalization = 1.0f / eta_vcm;
}

// run_iteration (oracle_vcm.cxx) over pixel_count() paths
void run_preview_iteration(Oracle& o, uint32_t s, uint32_t threads) {
  auto t0 = std::chrono::steady_clock::now();
  const Scene& scene = o.scene;
  const Camera& camera = o.camera;
  auto& it = o.iteration;
  const uint32_t pixel_count = reduced_count(o, s);

  start_preview_iteration(o, s);

  o.light_paths.assign(pixel_count, VCMLightPath{});
  o.light_vertices.clear();
  o.light_sampler_end.assign(pixel_count, 0u);
  o.camera_sampler_end.assign(pixel_count, 0u);
  o.camera_value.assign(pixel_count, float3{});

  const uint32_t grains = grain_count(pixel_count, threads);
  std::vector<std::vector<VCMLightVertex>> local_vertices(grains);
  std::vector<uint64_t> local_bounces(std::max(1u, threads), 0), local_splats(std::max(1u, threads), 0);
  parallel_ranges(pixel_count, threads, [&](uint32_t begin, uint32_t end, uint32_t grain, uint32_t tid) {
    auto& verts = local_vertices[grain];
    verts.reserve(4llu * (end - begin));
    for (uint32_t i = begin; i < end; ++i) {
      VCMPathState state = vcm_generate_emitter_state(i, scene, it);
      LightStepResult step = {};
      step.continue_tracing = (state.flags & VCMPathState::Valid) == VCMPathState::Valid;
      uint32_t path_begin = static_cast<uint32_t>(verts.size());
      while (step.continue_tracing) {
        step = vcm_light_step(scene, camera, it, o.options, i, state, o.rt);
        local_bounces[tid] += 1;
        if (step.add_vertex) {
          verts.emplace_back(step.vertex_to_add);
        }
        for (uint32_t k = 0; k < step.splat_count; ++k) {
          const float3 val = step.values_to_splat[k].to_rgb() / step.values_to_splat[k].sampling_pdf();
          if (dot(val, val) > kEpsilon) {
            add_light_block(o, s, val, step.splat_uvs[k], threads > 1);
            local_splats[tid] += 1;
          }
        }
      }
      auto& lp = o.light_paths[i];
      lp.spect = state.spect;
      lp.index = path_begin;
      lp.count = static_cast<uint32_t>(verts.size() - path_begin);
      lp.pixel_index = i;
      o.light_sampler_end[i] = state.sampler.seed;
    }
    flush_thread_counters(o.counters);
  });
  {
    const uint32_t chunk = (threads <= 1) ? pixel_count : kGrain;
    for (uint32_t g = 0; g < local_vertices.size(); ++g) {
      uint32_t base = static_cast<uint32_t>(o.light_vertices.size());
      uint32_t b = std::min(pixel_count, g * chunk), e = std::min(pixel_count, b + chunk);
      for (uint32_t i = b; i < e; ++i)
        o.light_paths[i].index += base;
      o.light_vertices.insert(o.light_vertices.end(), local_vertices[g].begin(), local_vertices[g].end());
    }
    for (uint32_t t = 0; t < local_bounces.size(); ++t) {
      o.stat_bounces_light += local_bounces[t];
      o.stat_splats += local_splats[t];
    }
  }

  film_commit_light(o, it.iteration);
  if (o.options.merge_vertices()) {
    build_grid(o);
  } else {
    o.grid = {};
  }

  auto light_vertices = make_array_view<VCMLightVertex>(o.light_vertices.data(), o.light_vertices.size());
  auto light_paths = make_array_view<VCMLightPath>(o.light_paths.data(), o.light_paths.size());
  std::vector<uint64_t> cam_bounces(std::max(1u, threads), 0);
  parallel_ranges(pixel_count, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t tid) {
    for (uint32_t pi = begin; pi < end; ++pi) {
      uint2 pixel = {};
      active_pixel(o, s, pi, it.iteration, pixel);  // the VCM's pixels never converge
      const auto& light_path = o.light_paths[pi];
      VCMPathState state = vcm_generate_camera_state(pixel, pi, scene, camera, it, light_path.spect);
      for (;;) {
        cam_bounces[tid] += 1;
        if (vcm_camera_step(scene, it, o.options, light_paths, light_vertices, state, o.rt, o.grid) == false)
          break;
      }
      state.merged *= it.vm_normalization;
      state.merged += (state.gathered / state.spect.sampling_pdf()).to_rgb();
      for_block(o, s, pixel, [&](const uint2& p) { film_accumulate_camera(o, p, state.merged); });
      o.camera_sampler_end[pi] = state.sampler.seed;
      o.camera_value[pi] = state.merged;
    }
    flush_thread_counters(o.counters);
  });
  for (auto b : cam_bounces)
    o.stat_bounces_camera += b;

  auto t1 = std::chrono::steady_clock::now();
  o.last_iteration_time = std::chrono::duration<double>(t1 - t0).count();
  o.total_time += o.last_iteration_time;
  o.completed += 1;
  it.iteration += 1;
}

// run_pt_iteration (oracle_vcm.cxx) over pixel_count() paths; estimate_noise_levels still runs over every pixel
void run_preview_pt_iteration(Oracle& o, uint32_t s, uint32_t threads) {
  auto t0 = std::chrono::steady_clock::now();
  const Scene& scene = o.scene;
  const Camera& camera = o.camera;
  const uint32_t pixel_count = reduced_count(o, s);
  const uint32_t iteration = o.iteration.iteration;
  o.camera_sampler_end.assign(pixel_count, 0u);
  o.camera_value.assign(pixel_count, float3{});
  std::vector<uint64_t> bounces(std::max(1u, threads), 0), processed(std::max(1u, threads), 0);
  parallel_ranges(pixel_count, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t tid) {
    for (uint32_t i = begin; i < end; ++i) {
      uint2 pixel = {};
      if (active_pixel(o, s, i, iteration, pixel) == false)
        continue;
      processed[tid] += 1;
      PTRayPayload payload = make_ray_payload(scene, camera, *o.film, pixel, i, iteration, scene.spectral(), o.pt_options.blue_noise);
      bounces[tid] += (payload.path_length <= scene.max_path_length) ? 1 : 0;
      while (run_path_iteration(scene, o.pt_options, o.rt, payload)) {
        bounces[tid] += (payload.path_length <= scene.max_path_length) ? 1 : 0;
      }
      auto normal = payload.view_normal;
      auto albedo = (payload.view_albedo / payload.spect.sampling_pdf()).to_rgb();
      auto color = (payload.accumulated / payload.spect.sampling_pdf()).to_rgb();
      if ((scene.radiance_clamp > 0.0f) && (payload.path_length > 1)) {
        float lum = luminance(color);
        if (lum > scene.radiance_clamp) {
          color *= scene.radiance_clamp / lum;
        }
      }
      for_block(o, s, pixel, [&](const uint2& p) { film_accumulate_pt(o, p, color, normal, albedo); });
      o.camera_sampler_end[i] = payload.smp.seed;
      o.camera_value[i] = color;
    }
    flush_thread_counters(o.counters);
  });
  o.pixels_processed = 0;
  for (uint32_t t = 0; t < bounces.size(); ++t) {
    o.stat_bounces_camera += bounces[t];
    o.pixels_processed += uint32_t(processed[t]);
  }
  film_estimate_noise_levels(o, iteration, scene.noise_threshold);
  auto t1 = std::chrono::steady_clock::now();
  o.last_iteration_time = std::chrono::duration<double>(t1 - t0).count();
  o.total_time += o.last_iteration_time;
  o.completed += 1;
  o.iteration.iteration += 1;
}

}  // namespace
}  // namespace etx

extern "C" {

void* oracle_create(const void* scene_blob, uint64_t scene_bytes, const void* camera_blob, uint64_t camera_bytes) {
  void* h = oracle_full_create(scene_blob, scene_bytes, camera_blob, camera_bytes);
  if (h)
    preview_of(h) = {};
  return h;
}

// Film::set_pixel_size (film.cxx:483-485): clamped, applied by the next oracle_begin
void oracle_set_film_pixel_size(void* h, uint32_t size) {
  preview_of(h).target_pixel_size = clamp(size, 1u, 1024u);
}

void oracle_begin(void* h, uint32_t first_iteration) {
  auto* o = static_cast<Oracle*>(h);
  PreviewFilm& p = preview_of(h);
  p.pixel_size = p.target_pixel_size;  // Film::clear (film.cxx:365)
  oracle_full_begin(h, first_iteration);
  o->active_pixels = reduced_count(*o, p.pixel_size);
}

double oracle_run_iterations(void* h, uint32_t count, uint32_t threads) {
  auto* o = static_cast<Oracle*>(h);
  const uint32_t s = preview_of(h).pixel_size;
  if (s == 1u)
    return oracle_full_run_iterations(h, count, threads);
  for (uint32_t i = 0; i < count; ++i) {
    if (o->integrator == ETXB_INTEGRATOR_PT) {
      run_preview_pt_iteration(*o, s, threads);
    } else {
      run_preview_iteration(*o, s, threads);
    }
  }
  return o->total_time;
}

// the per-light-path buffers hold pixel_count() entries at pixel size > 1; everything else is oracle_vcm.cxx's
int oracle_read_buffer(void* h, uint32_t id, void* dst, uint64_t dst_bytes, uint64_t* out_bytes) {
  auto* o = static_cast<Oracle*>(h);
  const bool light_path_buffer = (id == ETXB_BUF_LIGHT_PATH_COUNT) || (id == ETXB_BUF_LIGHT_PATH_OFFSET) || (id == ETXB_BUF_LIGHT_PATH_WAVELENGTH);
  if ((preview_of(h).pixel_size == 1u) || !light_path_buffer)
    return oracle_full_read_buffer(h, id, dst, dst_bytes, out_bytes);
  const size_t n = o->light_paths.size();
  std::vector<uint32_t> v(n);
  for (size_t i = 0; i < n; ++i) {
    const auto& lp = o->light_paths[i];
    if (id == ETXB_BUF_LIGHT_PATH_COUNT) {
      v[i] = lp.count;
    } else if (id == ETXB_BUF_LIGHT_PATH_OFFSET) {
      v[i] = lp.index;
    } else {
      memcpy(&v[i], &lp.spect.wavelength, 4);
    }
  }
  if (out_bytes)
    *out_bytes = n * 4u;
  if (dst == nullptr)
    return 0;
  if (dst_bytes < n * 4u)
    return -2;
  memcpy(dst, v.data(), n * 4u);
  return 0;
}

// pm::preview_offset of `count` (index, iteration) pairs — the definition the device calls
void oracle_preview_offset(const uint32_t* index, const uint32_t* iteration, uint32_t count, uint32_t size, uint32_t* dx, uint32_t* dy) {
  for (uint32_t k = 0; k < count; ++k)
    pm::preview_offset(index[k], iteration[k], size, dx[k], dy[k]);
}

}  // extern "C"
