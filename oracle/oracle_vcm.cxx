// TEST INFRASTRUCTURE — the CPU oracle for the VCM hot path.  Only tests/, __graft_entry__.smoke() and
// bench.py's cpu_baseline / --impl reference legs may load the library built from this file.
//
// What it is: the reference's OWN arithmetic — sources/etx/rt/shared/vcm_shared.hxx and every
// sources/etx/render/shared/*.hxx it pulls in, plus render/host/spectrum.cxx and thirdparty/bluenoise/
// bluenoise.cxx — compiled unmodified from /root/reference by oracle/build_oracle.sh, plus a restatement of
// the pieces that cannot be compiled here:
//   * etx::Raytracing (sources/etx/rt/rt.cxx:327-579; Embree 4 is not installed)  -> over etxb::Bvh, the
//     SAME tree + traversal routine the CUDA kernels use (etx_tracer_b200/csrc/bvh.h);
//   * the CPU VCM driver (sources/etx/rt/integrators/vcm_cpu.cxx:81-241; integrator.hxx -> util/options.hxx
//     is rejected by gcc)                                                           -> run_iteration();
//   * VCMSpatialGrid::construct (sources/etx/rt/integrators/vcm_shared.cxx:49-152)  -> build_grid(), with the
//     reference's `total = _cell_ends.back()` under-allocation fixed (sized by the full sum);
//   * the Film subset the VCM integrator touches (sources/etx/render/host/film.cxx:147-230,332-343,381-418);
//   * sample_blue_noise (sources/etx/rt/integrators/path_tracing.cxx:173-178);
//   * for the path tracer (SURVEY 8(f) N3; run_path_iteration itself is the reference's rt/shared/path_tracing_shared.hxx, compiled in place):
//     the CPUPathTracing driver (rt/integrators/path_tracing.cxx:50-110)            -> run_pt_iteration(), Film::sample (film.cxx:137-145),
//     Film::accumulate_camera_image with the normal / albedo / adaptive layers (:173-230) and Film::estimate_noise_levels (:233-330).
// Parity status: the reference ships no tests or golden vectors for this path (SURVEY.md §4); the pins are the
// known-answer vectors in tests/golden/ generated from these compiled headers.
#include <etx/core/core.hxx>
#include <etx/rt/rt.hxx>
#include <etx/render/host/film.hxx>
#include <etx/render/shared/scene_camera.hxx>
#include <etx/rt/shared/vcm_shared.hxx>

#include <bluenoise.hxx>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <chrono>
#include <cstring>
#include <thread>
#include <vector>

#include "bvh_build.h"
#include "../include/etx_b200.h"

namespace etx {

// ---------------------------------------------------------------------------------------------------
// Raytracing over etxb::Bvh (restates rt.cxx:250-579)
// ---------------------------------------------------------------------------------------------------
struct OracleCounters {
  std::atomic<uint64_t> rays_closest{0}, rays_shadow{0}, nodes{0}, tris{0};
};

struct RaytracingImpl {
  const etxb::Bvh* bvh = nullptr;
  const Scene* scene = nullptr;
  const Camera* camera = nullptr;
  OracleCounters* counters = nullptr;
};

// per-thread tallies, flushed into the shared atomics once per worker range (no cache-line ping-pong between threads)
struct ThreadCounters {
  uint64_t rays_closest = 0, rays_shadow = 0, nodes = 0, tris = 0;
};
static thread_local ThreadCounters g_thread_counters;
static void flush_thread_counters(OracleCounters& dst) {
  auto& t = g_thread_counters;
  dst.rays_closest += t.rays_closest;
  dst.rays_shadow += t.rays_shadow;
  dst.nodes += t.nodes;
  dst.tris += t.tris;
  t = {};
}

static thread_local const etxb::Bvh* g_pending_bvh = nullptr;
static thread_local OracleCounters* g_pending_counters = nullptr;

Raytracing::Raytracing() {
  static_assert(sizeof(_private_storage) >= sizeof(RaytracingImpl));
  _private = new (_private_storage) RaytracingImpl();
}
Raytracing::~Raytracing() {
}
void Raytracing::link_scene(const Scene& s) {
  _private->scene = &s;
}
void Raytracing::link_camera(const Camera& c) {
  _private->camera = &c;
}
const Scene& Raytracing::scene() const {
  return *_private->scene;
}
const Camera& Raytracing::camera() const {
  return *_private->camera;
}
void Raytracing::commit_changes() {
  _private->bvh = g_pending_bvh;
  _private->counters = g_pending_counters;
}

namespace {

struct HostNodeLoad {
  const etxb::BvhNode* nodes;
  etxb::BvhNode operator()(int32_t i) const {
    return nodes[i];
  }
};
struct HostTriLoad {
  const etxb::F4* pos;
  etxb::F4 operator()(uint32_t i) const {
    return pos[i];
  }
};

template <class Visitor>
void run_traversal(const RaytracingImpl* impl, const Ray& r, Visitor& v, bool shadow) {
  HostNodeLoad nl{impl->bvh->nodes.data()};
  HostTriLoad tl{impl->bvh->tri_pos.data()};
  etxb::TraverseStats st;
  etxb::traverse(nl, tl, r.o.x, r.o.y, r.o.z, r.d.x, r.d.y, r.d.z, r.min_t, r.max_t, v, impl->counters ? &st : nullptr);
  if (impl->counters) {
    g_thread_counters.nodes += st.nodes;
    g_thread_counters.tris += st.tris;
    (shadow ? g_thread_counters.rays_shadow : g_thread_counters.rays_closest) += 1;
  }
}

}  // namespace

// rt.cxx:428-466 — closest hit; one sampler draw per candidate via alpha_test_pass (scene_bsdf.hxx:128)
bool Raytracing::trace(const Scene& scene, const Ray& r, Intersection& result_intersection, Sampler& smp) const {
  IntersectionBase best = {{}, kInvalidIndex, 0.0f};
  auto visit = [&](uint32_t triangle_index, float u, float v, float t) -> int {
    const auto& tri = scene.triangles[triangle_index];
    const auto& mat = scene.materials[tri.material_index];
    if (mat.cls == Material::Class::Void)
      return etxb::kCandIgnore;
    if (alpha_test_pass(mat, tri, barycentrics({u, v}), scene, smp))
      return etxb::kCandIgnore;
    best = {{u, v}, triangle_index, t};
    return etxb::kCandAccept;
  };
  run_traversal(_private, r, visit, false);
  if (best.triangle_index == kInvalidIndex)
    return false;
  result_intersection = make_intersection(scene, r.d, best);
  return true;
}

// the rays trace_material and continuous_trace have traced on this thread: oracle_subsurface reports a gather's count as the device does
static thread_local uint32_t g_material_rays = 0;

// rt.cxx:327-371 — closest hit restricted to one material
bool Raytracing::trace_material(const Scene& scene, const Ray& r, const uint32_t material_id, Intersection& result_intersection, Sampler& smp) const {
  g_material_rays += 1;
  IntersectionBase best = {{}, kInvalidIndex, 0.0f};
  auto visit = [&](uint32_t triangle_index, float u, float v, float t) -> int {
    const auto& tri = scene.triangles[triangle_index];
    if ((material_id != kInvalidIndex) && (tri.material_index != material_id))
      return etxb::kCandIgnore;
    const auto& mat = scene.materials[tri.material_index];
    if (mat.cls == Material::Class::Void)
      return etxb::kCandIgnore;
    if (alpha_test_pass(mat, tri, barycentrics({u, v}), scene, smp))
      return etxb::kCandIgnore;
    best = {{u, v}, triangle_index, t};
    return etxb::kCandAccept;
  };
  run_traversal(_private, r, visit, false);
  if (best.triangle_index == kInvalidIndex)
    return false;
  result_intersection = make_intersection(scene, r.d, best);
  return true;
}

// rt.cxx:373-426 — collect up to N hits along the ray
uint32_t Raytracing::continuous_trace(const Scene& scene, const Ray& r, const ContinousTraceOptions& options, Sampler& smp) const {
  g_material_rays += 1;
  uint32_t count = 0;
  auto visit = [&](uint32_t triangle_index, float u, float v, float t) -> int {
    const auto& tri = scene.triangles[triangle_index];
    if ((options.material_id != kInvalidIndex) && (options.material_id != tri.material_index))
      return etxb::kCandIgnore;
    const auto& mat = scene.materials[tri.material_index];
    if (mat.cls == Material::Class::Void)
      return etxb::kCandIgnore;
    if (alpha_test_pass(mat, tri, barycentrics({u, v}), scene, smp))
      return etxb::kCandIgnore;
    if (count < options.max_intersections) {
      options.intersection_buffer[count] = {{u, v}, triangle_index, t};
      count += 1u;
    }
    return (count < options.max_intersections) ? etxb::kCandIgnore : etxb::kCandAccept;
  };
  run_traversal(_private, r, visit, false);
  return count;
}

// rt.cxx:468-579 — shadow ray through Boundary materials with per-segment medium transmittance
SpectralResponse Raytracing::trace_transmittance(const SpectralQuery spect, const Scene& scene, const float3& p0, const float3& p1, const Medium::Instance& medium,
  Sampler& smp) const {
  constexpr uint32_t kBufferSize = 63;
  struct Crossing {
    uint32_t primitive_id;
    float u, v, t;
  };
  Crossing crossings[kBufferSize + 1u];
  uint32_t crossing_count = 0;
  bool occluded = false;

  auto visit = [&](uint32_t triangle_index, float u, float v, float t) -> int {
    const auto& tri = scene.triangles[triangle_index];
    const auto& mat = scene.materials[tri.material_index];
    if (mat.cls == Material::Class::Void)
      return etxb::kCandIgnore;
    if (alpha_test_pass(mat, tri, barycentrics({u, v}), scene, smp))
      return etxb::kCandIgnore;
    if ((mat.cls != Material::Class::Boundary) || (crossing_count + 1u >= kBufferSize)) {
      occluded = true;
      return etxb::kCandTerminate;
    }
    crossings[crossing_count++] = {triangle_index, u, v, t};
    return etxb::kCandIgnore;
  };

  float3 direction = p1 - p0;
  float t_max = dot(direction, direction);
  if (t_max <= kRayEpsilon) {
    return {spect, 1.0f};
  }
  t_max = sqrtf(t_max);
  direction /= t_max;
  t_max -= fmaxf(kRayEpsilon, t_max * kRayEpsilon);

  Ray ray = {p0, direction, kRayEpsilon, t_max};
  run_traversal(_private, ray, visit, true);

  if (occluded) {
    return {spect, 0.0f};
  }

  for (uint32_t i = 0; i < crossing_count; ++i) {
    for (uint32_t j = i + 1; j < crossing_count; ++j) {
      if (crossings[i].t > crossings[j].t) {
        std::swap(crossings[i], crossings[j]);
      }
    }
  }
  crossings[crossing_count++] = {kInvalidIndex, 0.0f, 0.0f, t_max};

  float current_t = 0.0f;
  float3 origin = p0;
  SpectralResponse result = {spect, 1.0f};
  Medium::Instance current_medium = medium;
  for (uint32_t i = 0; i < crossing_count; ++i) {
    const auto& c = crossings[i];
    if (current_medium.valid()) {
      float dt = fmaxf(0.0f, c.t - current_t);
      if (current_medium.index != kInvalidIndex) {
        result *= medium_transmittance(scene, scene.mediums[current_medium.index], spect, smp, origin, direction, dt);
      } else {
        result *= medium_transmittance(current_medium, dt);
      }
    }
    if (c.primitive_id == kInvalidIndex)
      break;
    const auto& tri = scene.triangles[c.primitive_id];
    const auto& mat = scene.materials[tri.material_index];
    const bool entering = dot(tri.geo_n, direction) < 0.0f;
    current_medium = {.index = entering ? mat.int_medium : mat.ext_medium};
    current_t = c.t;
    origin = lerp_pos(scene.vertices, tri, barycentrics({c.u, c.v}));
  }
  return result;
}

// core/log.cxx is not compiled into the oracle; messages from spectrum.cxx go to stderr
void log::output(Color, const char* fmt, ...) {
  va_list args;
  va_start(args, fmt);
  vfprintf(stderr, fmt, args);
  fputc('\n', stderr);
  va_end(args);
}

// path_tracing.cxx:173-178
float2 sample_blue_noise(const uint2& pixel, const uint32_t total_samples, const uint32_t current_sample, uint32_t dimension) {
  auto smp = BNSampler(pixel.x, pixel.y, total_samples, current_sample);
  float u = smp.get(dimension + 0u);
  float v = smp.get(dimension + 1u);
  return {u, v};
}

// ---------------------------------------------------------------------------------------------------
// Film: the one member make_ray_payload calls (path_tracing_shared.hxx:245).  film.cxx itself cannot be compiled here (denoiser, task scheduler):
// the three members below restate film.cxx:104-121 (the dimensions only) and :137-145.
// ---------------------------------------------------------------------------------------------------
struct FilmImpl {
  uint2 dimensions = {};
};
Film::Film(TaskScheduler&) {
  _private = new (_private_storage) FilmImpl();
}
Film::~Film() {
}
void Film::allocate(const uint2& dim) {
  _private->dimensions = dim;
}
float2 Film::sample(const Scene& scene, const PixelFilter& sampler, const uint2& pixel, const float2& rnd) const {
  float2 jitter = rnd * 2.0f - 1.0f;
  if (sampler.image_index != kInvalidIndex) {
    jitter = scene.images[sampler.image_index].sample(rnd) * 2.0f - 1.0f;
  }
  float u = (float(pixel.x) + 0.5f + sampler.radius * jitter.x) / float(_private->dimensions.x) * 2.0f - 1.0f;
  float v = (float(pixel.y) + 0.5f + sampler.radius * jitter.y) / float(_private->dimensions.y) * 2.0f - 1.0f;
  return {u, v};
}

// ---------------------------------------------------------------------------------------------------
// Driver state
// ---------------------------------------------------------------------------------------------------
struct Oracle {
  Scene scene = {};
  Camera camera = {};
  etxb::Bvh bvh;
  Raytracing rt;
  OracleCounters counters;

  VCMOptions options = {};
  VCMIteration iteration = {};

  std::vector<VCMLightVertex> light_vertices;
  std::vector<VCMLightPath> light_paths;

  // grid storage (vcm_spatial_grid.hxx:15-23)
  VCMSpatialGridData grid = {};
  std::vector<uint32_t> cell_ends;
  std::vector<float3> g_positions, g_normals, g_w_in, g_throughput;
  std::vector<float> g_d_vcm, g_d_vm;
  std::vector<uint32_t> g_path_lengths;

  // film subset (film.cxx): y-flipped storage
  uint32_t width = 0, height = 0;
  std::vector<float3> film_camera, film_light, film_light_iteration;
  std::vector<uint32_t> film_samples;
  std::vector<float4> film_out;

  // path tracer: which integrator run_iterations drives, its options, the film members it alone touches (film.cxx:14-40)
  uint32_t integrator = ETXB_INTEGRATOR_VCM;
  PTOptions pt_options = {};
  uint64_t film_storage[(sizeof(Film) + 7) / 8] = {};
  Film* film = nullptr;
  std::vector<float3> film_normals, film_albedo, film_adaptive;
  std::vector<uint8_t> film_converged, film_tmp;
  std::vector<float> film_error;
  float noise_level = 0.0f;
  uint32_t active_pixels = 0, pixels_processed = 0;

  // debug taps
  std::vector<uint32_t> light_sampler_end, camera_sampler_end;
  std::vector<float3> camera_value;

  double total_time = 0.0;
  double last_iteration_time = 0.0;
  uint32_t completed = 0;
  uint64_t stat_bounces_light = 0, stat_bounces_camera = 0, stat_splats = 0;

  uint32_t pixel_count() const {
    return width * height;
  }
};

namespace {

void film_clear(Oracle& o) {
  uint32_t n = o.pixel_count();
  o.film_camera.assign(n, float3{});
  o.film_light.assign(n, float3{});
  o.film_light_iteration.assign(n, float3{});
  o.film_samples.assign(n, 0u);
  o.film_out.assign(n, float4{});
  o.film_normals.assign(n, float3{});
  o.film_albedo.assign(n, float3{});
  o.film_adaptive.assign(n, float3{});
  o.film_converged.assign(n, 0u);
  o.film_tmp.assign(n, 0u);
  o.film_error.assign(n, 0.0f);
  o.noise_level = 0.0f;
  o.active_pixels = n;
  o.pixels_processed = 0;
}

inline void atomic_add_f(float* ptr, float value) {
  auto* a = reinterpret_cast<std::atomic<uint32_t>*>(ptr);
  uint32_t old_bits = a->load(std::memory_order_relaxed);
  for (;;) {
    float old_value;
    memcpy(&old_value, &old_bits, 4);
    float new_value = old_value + value;
    uint32_t new_bits;
    memcpy(&new_bits, &new_value, 4);
    if (a->compare_exchange_weak(old_bits, new_bits, std::memory_order_relaxed))
      break;
  }
}

// film.cxx:147-171 (pixel_size == 1)
void film_add_light(Oracle& o, const float3& value, const float2& ndc, bool atomic) {
  if (dot(value, value) == 0.0f)
    return;
  float2 uv = ndc * 0.5f + 0.5f;
  uint32_t x = static_cast<uint32_t>(uv.x * o.width);
  uint32_t y = static_cast<uint32_t>(uv.y * o.height);
  if ((x >= o.width) || (y >= o.height))
    return;
  uint32_t i = x + (o.height - 1u - y) * o.width;
  float3& dst = o.film_light_iteration[i];
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

// film.cxx:173-230 (camera layer only; normal/albedo AOVs are passed as zero by the VCM integrator)
void film_accumulate_camera(Oracle& o, const uint2& pixel, const float3& color) {
  if ((pixel.x >= o.width) || (pixel.y >= o.height))
    return;
  uint32_t i = pixel.x + (o.height - 1u - pixel.y) * o.width;
  uint32_t sample_index = o.film_samples[i];
  double ds = double(sample_index);
  if (sample_index == 0) {
    o.film_camera[i] = color;
  } else {
    float t = float(ds / (ds + 1.0));
    o.film_camera[i] = {
      lerp(color.x, o.film_camera[i].x, t),
      lerp(color.y, o.film_camera[i].y, t),
      lerp(color.z, o.film_camera[i].z, t),
    };
  }
  o.film_samples[i] += 1u;
}

// film.cxx:332-343
void film_commit_light(Oracle& o, uint32_t iteration) {
  float t = float(double(iteration) / double(iteration + 1u));
  for (uint32_t i = 0, n = o.pixel_count(); i < n; ++i) {
    o.film_light[i] = (t == 0.0f) ? o.film_light_iteration[i] : lerp(o.film_light_iteration[i], o.film_light[i], t);
    o.film_light_iteration[i] = {};
  }
}

// vcm_shared.cxx:49-152, deterministic (vertex order) when threads == 1
void build_grid(Oracle& o) {
  o.grid = {};
  const auto& samples = o.light_vertices;
  uint64_t sample_count = samples.size();
  if (sample_count == 0)
    return;

  auto& data = o.grid;
  float radius = o.iteration.current_radius;
  data.radius_squared = radius * radius;
  data.inv_radius_squared = (data.radius_squared > 0.0f) ? 1.0f / data.radius_squared : 0.0f;
  data.cell_size = 2.0f * radius;
  data.bounding_box = {{kMaxFloat, kMaxFloat, kMaxFloat}, 0.0f, {-kMaxFloat, -kMaxFloat, -kMaxFloat}, 0.0f};
  for (const auto& p : samples) {
    if (p.is_medium)
      continue;
    data.bounding_box.p_min = min(data.bounding_box.p_min, p.pos);
    data.bounding_box.p_max = max(data.bounding_box.p_max, p.pos);
  }

  uint32_t hash_table_size = static_cast<uint32_t>(next_power_of_two(sample_count));
  data.hash_table_mask = hash_table_size - 1u;

  o.cell_ends.assign(hash_table_size, 0u);
  for (const auto& s : samples) {
    if (s.is_medium)
      continue;
    o.cell_ends[data.position_to_index(s.pos)] += 1u;
  }
  uint32_t sum = 0;
  for (auto& c : o.cell_ends) {
    uint32_t t = c;
    c = sum;
    sum += t;
  }
  uint32_t total = sum;  // reference uses _cell_ends.back() (under-allocates); see header comment
  o.g_positions.resize(total);
  o.g_normals.resize(total);
  o.g_w_in.resize(total);
  o.g_d_vcm.resize(total);
  o.g_d_vm.resize(total);
  o.g_path_lengths.resize(total);
  o.g_throughput.resize(total);
  for (const auto& s : samples) {
    if (s.is_medium)
      continue;
    uint32_t cell = data.position_to_index(s.pos);
    uint32_t dst = o.cell_ends[cell]++;
    o.g_positions[dst] = s.pos;
    o.g_normals[dst] = s.nrm;
    o.g_w_in[dst] = s.w_i;
    o.g_d_vcm[dst] = s.d_vcm;
    o.g_d_vm[dst] = s.d_vm;
    o.g_path_lengths[dst] = s.path_length;
    o.g_throughput[dst] = (s.throughput / s.throughput.sampling_pdf()).to_rgb();
  }
  data.cell_ends = make_array_view<uint32_t>(o.cell_ends.data(), o.cell_ends.size());
  data.positions = make_array_view<float3>(o.g_positions.data(), o.g_positions.size());
  data.normals = make_array_view<float3>(o.g_normals.data(), o.g_normals.size());
  data.w_in = make_array_view<float3>(o.g_w_in.data(), o.g_w_in.size());
  data.d_vcm = make_array_view<float>(o.g_d_vcm.data(), o.g_d_vcm.size());
  data.d_vm = make_array_view<float>(o.g_d_vm.data(), o.g_d_vm.size());
  data.path_lengths = make_array_view<uint32_t>(o.g_path_lengths.data(), o.g_path_lengths.size());
  data.throughput_rgb_div_pdf = make_array_view<float3>(o.g_throughput.data(), o.g_throughput.size());
}

// The reference hands pixel ranges to its workers dynamically (enkiTS task sets, render/host/tasks.cxx:57-66,91-96).  Same here: grains of
// kGrain pixels, pulled from a shared counter by `threads` workers, so that an expensive image region does not leave the other threads idle.
// fn(begin, end, grain index, thread index).
constexpr uint32_t kGrain = 256u;
inline uint32_t grain_count(uint32_t count, uint32_t threads) { return (threads <= 1) ? 1u : (count + kGrain - 1u) / kGrain; }
template <class F>
void parallel_ranges(uint32_t count, uint32_t threads, F&& fn) {
  if (threads <= 1) {
    fn(0u, count, 0u, 0u);
    return;
  }
  const uint32_t grains = grain_count(count, threads);
  std::atomic<uint32_t> next{0u};
  std::vector<std::thread> pool;
  for (uint32_t t = 0; t < threads; ++t) {
    pool.emplace_back([&fn, &next, grains, count, t]() {
      for (;;) {
        uint32_t g = next.fetch_add(1u, std::memory_order_relaxed);
        if (g >= grains) break;
        uint32_t b = g * kGrain, e = std::min(count, b + kGrain);
        fn(b, e, g, t);
      }
    });
  }
  for (auto& th : pool)
    th.join();
}

// start_next_iteration (vcm_cpu.cxx:95-124): merge radius and MIS weights of the iteration
void start_next_iteration(Oracle& o) {
  auto& it = o.iteration;
  float used_radius = o.options.initial_radius;
  if (used_radius == 0.0f) {
    uint32_t max_dim = max(o.width, o.height);
    used_radius = 5.0f * o.scene.bounding_sphere_radius / float(max_dim);
  }
  float radius_scale = 1.0f / (1.0f + float(it.iteration) / float(o.options.radius_decay));
  it.current_radius = used_radius * radius_scale;
  float eta_vcm = kPi * sqr(it.current_radius) * float(o.pixel_count());
  it.vc_weight = 1.0f / eta_vcm;
  it.vm_weight = o.options.enable_merging() ? eta_vcm : 0.0f;
  it.vm_normalization = 1.0f / eta_vcm;
}

// vcm_cpu.cxx:95-241, one full iteration (light pass, grid build, camera pass)
void run_iteration(Oracle& o, uint32_t threads) {
  auto t0 = std::chrono::steady_clock::now();
  const Scene& scene = o.scene;
  const Camera& camera = o.camera;
  auto& it = o.iteration;
  const uint32_t pixel_count = o.pixel_count();

  start_next_iteration(o);

  o.light_paths.assign(pixel_count, VCMLightPath{});
  o.light_vertices.clear();
  o.light_sampler_end.assign(pixel_count, 0u);
  o.camera_sampler_end.assign(pixel_count, 0u);
  o.camera_value.assign(pixel_count, float3{});

  // gather_light_vertices (:126-172); thread-local vectors are appended in thread order so that the vertex
  // pool is path-major regardless of the thread count
  const uint32_t grains = grain_count(pixel_count, threads);
  std::vector<std::vector<VCMLightVertex>> local_vertices(grains);  // per grain: appended in grain order below = path-major, whatever the thread count
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
            film_add_light(o, val, step.splat_uvs[k], threads > 1);
            local_splats[tid] += 1;
          }
        }
      }
      auto& lp = o.light_paths[i];
      lp.spect = state.spect;
      lp.index = path_begin;  // local; rebased below
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

  // complete_light_vertices (:209-225)
  film_commit_light(o, it.iteration);
  if (o.options.merge_vertices()) {
    build_grid(o);
  } else {
    o.grid = {};
  }

  // gather_camera_vertices (:174-207)
  auto light_vertices = make_array_view<VCMLightVertex>(o.light_vertices.data(), o.light_vertices.size());
  auto light_paths = make_array_view<VCMLightPath>(o.light_paths.data(), o.light_paths.size());
  std::vector<uint64_t> cam_bounces(std::max(1u, threads), 0);
  parallel_ranges(pixel_count, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t tid) {
    for (uint32_t pi = begin; pi < end; ++pi) {
      uint2 pixel = {pi % o.width, pi / o.width};  // Film::active_pixel with pixel_size == 1 (film.cxx:434-461)
      const auto& light_path = o.light_paths[pi];
      VCMPathState state = vcm_generate_camera_state(pixel, pi, scene, camera, it, light_path.spect);
      for (;;) {
        cam_bounces[tid] += 1;
        if (vcm_camera_step(scene, it, o.options, light_paths, light_vertices, state, o.rt, o.grid) == false)
          break;
      }
      state.merged *= it.vm_normalization;
      state.merged += (state.gathered / state.spect.sampling_pdf()).to_rgb();
      film_accumulate_camera(o, pixel, state.merged);
      o.camera_sampler_end[pi] = state.sampler.seed;
      o.camera_value[pi] = state.merged;
    }
    flush_thread_counters(o.counters);
  });
  for (auto b : cam_bounces)
    o.stat_bounces_camera += b;

  // complete_camera_vertices (:227-241)
  auto t1 = std::chrono::steady_clock::now();
  o.last_iteration_time = std::chrono::duration<double>(t1 - t0).count();
  o.total_time += o.last_iteration_time;
  o.completed += 1;
  it.iteration += 1;
}


// ---------------------------------------------------------------------------------------------------
// Path tracer (SURVEY 8(f) N3)
// ---------------------------------------------------------------------------------------------------
// film.cxx:173-230 with pixel_size == 1: colour, normal, albedo running means; the every-other-sample mean; the sample counter
void film_accumulate_pt(Oracle& o, const uint2& pixel, const float3& color, const float3& normal, const float3& albedo) {
  if ((pixel.x >= o.width) || (pixel.y >= o.height))
    return;
  uint32_t i = pixel.x + (o.height - 1u - pixel.y) * o.width;
  uint32_t sample_index = o.film_samples[i];
  double ds = double(sample_index);
  if (sample_index == 0) {
    o.film_camera[i] = color;
    o.film_normals[i] = normal;
    o.film_albedo[i] = albedo;
    o.film_adaptive[i] = color;
  } else {
    float t = float(ds / (ds + 1.0));
    o.film_camera[i] = {lerp(color.x, o.film_camera[i].x, t), lerp(color.y, o.film_camera[i].y, t), lerp(color.z, o.film_camera[i].z, t)};
    o.film_normals[i] = {lerp(normal.x, o.film_normals[i].x, t), lerp(normal.y, o.film_normals[i].y, t), lerp(normal.z, o.film_normals[i].z, t)};
    o.film_albedo[i] = {lerp(albedo.x, o.film_albedo[i].x, t), lerp(albedo.y, o.film_albedo[i].y, t), lerp(albedo.z, o.film_albedo[i].z, t)};
    if ((sample_index % 2) == 0) {
      t = float(ds / (ds + 2.0));
      o.film_adaptive[i] = {lerp(color.x, o.film_adaptive[i].x, t), lerp(color.y, o.film_adaptive[i].y, t), lerp(color.z, o.film_adaptive[i].z, t)};
    }
  }
  o.film_samples[i] += 1u;
}

// film.cxx:233-330, single-threaded (the reference's three parallel passes only ever clear flags inside a pass, so their result does not depend on the thread order;
// its float sum of error levels does, by rounding)
void film_estimate_noise_levels(Oracle& o, uint32_t sample_index, float threshold) {
  constexpr uint32_t kMinSamples = 32u;
  if ((threshold == 0.0f) || (sample_index < kMinSamples) || (sample_index % 2) != 0)
    return;
  const uint32_t n = o.pixel_count();
  uint32_t converged_now = 0;
  float total_noise = 0.0f;
  for (uint32_t i = 0; i < n; ++i) {
    if (o.film_converged[i])
      continue;
    const float3& v_i = o.film_camera[i];
    const float3& v_a = o.film_adaptive[i];
    float error_diff = dot(abs(v_i - v_a), 1.0f);
    float error_norm = dot(abs(v_i), 1.0f);
    float error_level = error_diff / (((error_norm < 1.0f) ? sqrtf(error_norm) : error_norm) + kEpsilon);
    uint8_t converged = error_level < threshold ? 1u : 0u;
    o.film_error[i] = error_level;
    o.film_converged[i] = converged;
    o.film_tmp[i] = converged;
    converged_now += converged;
    total_noise += error_level;
  }
  o.active_pixels = converged_now;
  o.noise_level = (converged_now > 0) ? (total_noise / float(converged_now)) : total_noise;
  constexpr uint32_t kBlockSize = 5u;
  const uint32_t w = o.width, h = o.height;
  for (uint32_t i = 0; i < n; ++i) {
    if (o.film_converged[i])
      continue;
    uint32_t x = i % w, y = i / w;
    uint32_t begin_x = x >= kBlockSize ? x - kBlockSize : 0u;
    uint32_t end_x = min(w, x + kBlockSize);
    for (uint32_t p = begin_x; p < end_x; ++p)
      o.film_tmp[p + y * w] = 0;
  }
  for (uint32_t i = 0; i < n; ++i) {
    if (o.film_tmp[i])
      continue;
    uint32_t x = i % w, y = i / w;
    uint32_t begin_y = y >= kBlockSize ? y - kBlockSize : 0u;
    uint32_t end_y = min(h, y + kBlockSize);
    for (uint32_t p = begin_y; p < end_y; ++p)
      o.film_converged[x + p * w] = 0;
  }
}

// CPUPathTracingImpl::execute_range over every pixel + update()'s bookkeeping (path_tracing.cxx:50-110)
void run_pt_iteration(Oracle& o, uint32_t threads) {
  auto t0 = std::chrono::steady_clock::now();
  const Scene& scene = o.scene;
  const Camera& camera = o.camera;
  const uint32_t pixel_count = o.pixel_count();
  const uint32_t iteration = o.iteration.iteration;
  o.camera_sampler_end.assign(pixel_count, 0u);
  o.camera_value.assign(pixel_count, float3{});
  std::vector<uint64_t> bounces(std::max(1u, threads), 0), processed(std::max(1u, threads), 0);
  parallel_ranges(pixel_count, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t tid) {
    for (uint32_t i = begin; i < end; ++i) {
      uint2 pixel = {i % o.width, i / o.width};  // Film::active_pixel with pixel_size == 1 (film.cxx:434-461)
      uint32_t fi = pixel.x + (o.height - 1u - pixel.y) * o.width;
      if (o.film_converged[fi])
        continue;
      processed[tid] += 1;
      PTRayPayload payload = make_ray_payload(scene, camera, *o.film, pixel, i, iteration, scene.spectral(), o.pt_options.blue_noise);
      // a call that gets past the length test (:486) traces a ray and handles one event: that is what the device counts as a bounce
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
      film_accumulate_pt(o, pixel, color, normal, albedo);
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

// ---------------------------------------------------------------------------------------------------
// C API (loaded with ctypes by tests / bench)
// ---------------------------------------------------------------------------------------------------
using namespace etx;

extern "C" {

void* oracle_create(const void* scene_blob, uint64_t scene_bytes, const void* camera_blob, uint64_t camera_bytes) {
  if ((scene_bytes != sizeof(Scene)) || (camera_bytes != sizeof(Camera)))
    return nullptr;
  auto* o = new Oracle();
  memcpy(&o->scene, scene_blob, sizeof(Scene));
  memcpy(&o->camera, camera_blob, sizeof(Camera));
  o->width = o->camera.film_size.x;
  o->height = o->camera.film_size.y;
  etxb::build_bvh(reinterpret_cast<const float*>(o->scene.vertices.a), sizeof(Vertex), reinterpret_cast<const uint32_t*>(o->scene.triangles.a), sizeof(Triangle),
    uint32_t(o->scene.triangles.count), o->bvh);
  o->rt.link_scene(o->scene);
  o->rt.link_camera(o->camera);
  g_pending_bvh = &o->bvh;
  g_pending_counters = &o->counters;
  o->rt.commit_changes();
  o->options = {};
  o->options.options = VCMOptions::DefaultOptions;
  o->options.radius_decay = 256u;
  o->options.initial_radius = 0.0f;
  o->options.kernel = VCMOptions::Epanechnikov;
  o->options.blue_noise = true;
  o->film = new (o->film_storage) Film(*reinterpret_cast<TaskScheduler*>(o->film_storage));  // the scheduler reference is never used
  o->film->allocate({o->width, o->height});
  film_clear(*o);
  return o;
}

void oracle_destroy(void* h) {
  delete static_cast<Oracle*>(h);
}

void oracle_set_options(void* h, const etxb_vcm_options* opt) {
  auto* o = static_cast<Oracle*>(h);
  o->options.options = opt->options;
  o->options.radius_decay = opt->radius_decay;
  o->options.kernel = opt->kernel;
  o->options.initial_radius = opt->initial_radius;
  o->options.blue_noise = opt->blue_noise != 0;
}

void oracle_set_integrator(void* h, uint32_t integrator) {
  static_cast<Oracle*>(h)->integrator = integrator;
}

void oracle_pt_set_options(void* h, const etxb_pt_options* opt) {
  auto* o = static_cast<Oracle*>(h);
  o->pt_options.nee = opt->nee != 0;
  o->pt_options.direct = opt->direct != 0;
  o->pt_options.mis = opt->mis != 0;
  o->pt_options.blue_noise = opt->blue_noise != 0;
}

void oracle_pt_get_status(void* h, etxb_pt_status* out) {
  auto* o = static_cast<Oracle*>(h);
  out->pixels_processed = o->pixels_processed;
  out->active_pixels = o->active_pixels;
  out->noise_level = o->noise_level;
  out->max_sample_count = o->scene.samples;
}

void oracle_set_scene_settings(void* h, float noise_threshold, float radiance_clamp) {
  auto* o = static_cast<Oracle*>(h);
  o->scene.noise_threshold = noise_threshold;
  o->scene.radiance_clamp = radiance_clamp;
}

void oracle_begin(void* h, uint32_t first_iteration) {
  auto* o = static_cast<Oracle*>(h);
  film_clear(*o);
  o->iteration = {};
  o->iteration.iteration = first_iteration;
  o->total_time = 0.0;
  o->completed = 0;
  o->stat_bounces_light = o->stat_bounces_camera = o->stat_splats = 0;
  o->counters.rays_closest = 0;
  o->counters.rays_shadow = 0;
  o->counters.nodes = 0;
  o->counters.tris = 0;
}

double oracle_run_iterations(void* h, uint32_t count, uint32_t threads) {
  auto* o = static_cast<Oracle*>(h);
  for (uint32_t i = 0; i < count; ++i) {
    if (o->integrator == ETXB_INTEGRATOR_PT) {
      run_pt_iteration(*o, threads);
    } else {
      run_iteration(*o, threads);
    }
  }
  return o->total_time;
}

int oracle_read_film(void* h, uint32_t layer, float* dst, uint64_t dst_bytes) {
  auto* o = static_cast<Oracle*>(h);
  uint32_t n = o->pixel_count();
  if (dst_bytes < uint64_t(n) * 16u)
    return -1;
  auto* out = reinterpret_cast<float4*>(dst);
  for (uint32_t i = 0; i < n; ++i) {
    float3 v = {};
    switch (layer) {
      case ETXB_FILM_RESULT:
        v = max(float3{}, o->film_camera[i] + o->film_light[i]);  // film.cxx:398-405
        break;
      case ETXB_FILM_CAMERA:
        v = o->film_camera[i];
        break;
      case ETXB_FILM_LIGHT:
        v = o->film_light[i];
        break;
      case ETXB_FILM_NORMALS:
        v = o->film_normals[i] * 0.5f + 0.5f;  // film.cxx:409
        break;
      case ETXB_FILM_ALBEDO:
        v = o->film_albedo[i];
        break;
      case ETXB_FILM_CAMERA_ADAPTIVE:
        v = o->film_adaptive[i];
        break;
      default:
        v = o->film_light_iteration[i];
        break;
    }
    out[i] = {v.x, v.y, v.z, 1.0f};
  }
  return 0;
}

int oracle_read_buffer(void* h, uint32_t id, void* dst, uint64_t dst_bytes, uint64_t* out_bytes) {
  auto* o = static_cast<Oracle*>(h);
  uint32_t n = o->pixel_count();
  std::vector<uint8_t> tmp;
  auto put = [&](const void* p, uint64_t bytes) {
    tmp.resize(bytes);
    memcpy(tmp.data(), p, bytes);
  };
  switch (id) {
    case ETXB_BUF_LIGHT_PATH_COUNT: {
      std::vector<uint32_t> v(n);
      for (uint32_t i = 0; i < n; ++i)
        v[i] = o->light_paths[i].count;
      put(v.data(), v.size() * 4);
      break;
    }
    case ETXB_BUF_LIGHT_PATH_OFFSET: {
      std::vector<uint32_t> v(n);
      for (uint32_t i = 0; i < n; ++i)
        v[i] = o->light_paths[i].index;
      put(v.data(), v.size() * 4);
      break;
    }
    case ETXB_BUF_LIGHT_PATH_WAVELENGTH: {
      std::vector<float> v(n);
      for (uint32_t i = 0; i < n; ++i)
        v[i] = o->light_paths[i].spect.wavelength;
      put(v.data(), v.size() * 4);
      break;
    }
    case ETXB_BUF_LIGHT_SAMPLER:
      put(o->light_sampler_end.data(), o->light_sampler_end.size() * 4);
      break;
    case ETXB_BUF_CAMERA_SAMPLER:
      put(o->camera_sampler_end.data(), o->camera_sampler_end.size() * 4);
      break;
    case ETXB_BUF_LV_POS: {
      std::vector<float3> v(o->light_vertices.size());
      for (size_t i = 0; i < v.size(); ++i)
        v[i] = o->light_vertices[i].pos;
      put(v.data(), v.size() * 12);
      break;
    }
    case ETXB_BUF_LV_THROUGHPUT: {
      std::vector<float3> v(o->light_vertices.size());
      for (size_t i = 0; i < v.size(); ++i) {
        const auto& t = o->light_vertices[i].throughput;
        v[i] = t.spectral() ? float3{t.value, t.value, t.value} : t.integrated;
      }
      put(v.data(), v.size() * 12);
      break;
    }
    case ETXB_BUF_LV_MIS: {
      std::vector<float3> v(o->light_vertices.size());
      for (size_t i = 0; i < v.size(); ++i)
        v[i] = {o->light_vertices[i].d_vcm, o->light_vertices[i].d_vc, o->light_vertices[i].d_vm};
      put(v.data(), v.size() * 12);
      break;
    }
    case ETXB_BUF_CAMERA_GATHERED:
      put(o->camera_value.data(), o->camera_value.size() * 12);
      break;
    case ETXB_BUF_PIXEL_INFO: {
      std::vector<uint32_t> v(n);
      for (uint32_t i = 0; i < n; ++i)
        v[i] = (o->film_samples[i] & 0x3fffffffu) | (o->film_converged[i] ? (1u << 30u) : 0u) | (o->film_tmp[i] ? (1u << 31u) : 0u);
      put(v.data(), v.size() * 4);
      break;
    }
    case ETXB_BUF_PIXEL_ERROR:
      put(o->film_error.data(), o->film_error.size() * 4);
      break;
    default:
      return -1;
  }
  if (out_bytes)
    *out_bytes = tmp.size();
  if (dst == nullptr)
    return 0;
  if (dst_bytes < tmp.size())
    return -2;
  memcpy(dst, tmp.data(), tmp.size());
  return 0;
}

void oracle_get_counters(void* h, etxb_counters* out) {
  auto* o = static_cast<Oracle*>(h);
  memset(out, 0, sizeof(*out));
  out->rays_closest = o->counters.rays_closest;
  out->rays_shadow = o->counters.rays_shadow;
  out->nodes_visited = o->counters.nodes;
  out->tris_tested = o->counters.tris;
  out->bounces_light = o->stat_bounces_light;
  out->bounces_camera = o->stat_bounces_camera;
  out->light_vertices = o->light_vertices.size();
  out->splats = o->stat_splats;
}

// rays: {o.xyz, min_t, d.xyz, max_t}; hits_uv_t: {u, v, t} per ray; hits_tri: triangle index or 0xffffffff
void oracle_trace(void* h, const float* rays, uint32_t* seeds, uint32_t count, float* hits_uv_t, uint32_t* hits_tri) {
  auto* o = static_cast<Oracle*>(h);
  for (uint32_t i = 0; i < count; ++i) {
    const float* r = rays + size_t(i) * 8;
    Ray ray = {{r[0], r[1], r[2]}, {r[4], r[5], r[6]}, r[3], r[7]};
    Sampler smp(seeds[i]);
    Intersection isect = {};
    bool hit = o->rt.trace(o->scene, ray, isect, smp);
    seeds[i] = smp.seed;
    hits_tri[i] = hit ? isect.triangle_index : kInvalidIndex;
    hits_uv_t[size_t(i) * 3 + 0] = hit ? isect.barycentric.y : 0.0f;
    hits_uv_t[size_t(i) * 3 + 1] = hit ? isect.barycentric.z : 0.0f;
    hits_uv_t[size_t(i) * 3 + 2] = hit ? isect.t : 0.0f;
  }
  flush_thread_counters(o->counters);
}

void oracle_bvh_info(void* h, uint32_t* node_count, uint32_t* slot_count) {
  auto* o = static_cast<Oracle*>(h);
  *node_count = uint32_t(o->bvh.nodes.size());
  *slot_count = uint32_t(o->bvh.tri_index.size());
}

// The reference's own BSDF evaluation for etxb_closure_query records (include/etx_b200.h), as the VCM consumers call it
// (vcm_shared.hxx:708-713,738-748,852-857): bsdf::evaluate, then bsdf::reverse_pdf on the same sampler where the evaluation is valid.
// Repetition r runs on Sampler(seed, r); the statistics are those etxb_debug_closure_eval returns.  Queries are spread over `threads`.
static_assert(sizeof(etxb_closure_query) == 96);
void oracle_bsdf_eval(void* h, const etxb_closure_query* queries, uint32_t count, uint32_t repetitions, uint32_t threads, double* out) {
  auto* o = static_cast<Oracle*>(h);
  const Scene& scene = o->scene;
  parallel_ranges(count, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t) {
    for (uint32_t i = begin; i < end; ++i) {
      const etxb_closure_query& q = queries[i];
      Vertex v = {};
      v.nrm = {q.nrm[0], q.nrm[1], q.nrm[2]};
      v.tan = {q.tan[0], q.tan[1], q.tan[2]};
      v.btn = {q.btn[0], q.btn[1], q.btn[2]};
      v.tex = {q.uv[0], q.uv[1]};
      const float3 w_i = {q.w_i[0], q.w_i[1], q.w_i[2]}, w_o = {q.w_o[0], q.w_o[1], q.w_o[2]};
      const SpectralQuery spect = scene.spectral() ? SpectralQuery{q.wavelength, SpectralQuery::Spectral} : SpectralQuery::sample();
      const BSDFData data(spect, kInvalidIndex, static_cast<PathSource>(q.path_source), v, w_i);
      const Material& mat = scene.materials[q.material];
      double mean[8] = {}, m2[8] = {};
      double* dst = out + size_t(i) * ETXB_CLOSURE_STATS;
      uint32_t finite = 0, nonfinite = 0, negative = 0, unsupported = 0;
      for (uint32_t r = 0; r < repetitions; ++r) {
        Sampler smp(q.seed, r);
        BSDFEval e = bsdf::evaluate(data, w_o, mat, scene, smp);
        float rev = e.valid() ? bsdf::reverse_pdf(data, w_o, mat, scene, smp) : 0.0f;
        const float3 f = e.func.spectral() ? float3{e.func.value, e.func.value, e.func.value} : e.func.integrated;
        const float3 b = e.bsdf.spectral() ? float3{e.bsdf.value, e.bsdf.value, e.bsdf.value} : e.bsdf.integrated;
        const float val[8] = {f.x, f.y, f.z, b.x, b.y, b.z, e.pdf, rev};
        if (r == 0) {
          for (uint32_t k = 0; k < 8; ++k)
            dst[16 + k] = val[k];
        }
        bool ok = true;
        for (uint32_t k = 0; k < 8; ++k)
          ok = ok && std::isfinite(val[k]);
        negative += ((e.pdf < 0.0f) || (rev < 0.0f)) ? 1u : 0u;
        unsupported += ((e.pdf == 0.0f) && ((f.x != 0.0f) || (f.y != 0.0f) || (f.z != 0.0f) || (b.x != 0.0f) || (b.y != 0.0f) || (b.z != 0.0f))) ? 1u : 0u;
        if (!ok) {
          nonfinite += 1u;
          continue;
        }
        finite += 1u;
        for (uint32_t k = 0; k < 8; ++k) {
          const double delta = double(val[k]) - mean[k];
          mean[k] += delta / double(finite);
          m2[k] += delta * (double(val[k]) - mean[k]);
        }
      }
      for (uint32_t k = 0; k < 8; ++k) {
        dst[k] = mean[k];
        dst[8 + k] = (finite > 0) ? m2[k] / double(finite) : 0.0;
      }
      dst[24] = double(nonfinite);
      dst[25] = double(negative);
      dst[26] = double(unsupported);
      for (uint32_t k = 27; k < ETXB_CLOSURE_STATS; ++k)
        dst[k] = 0.0;
    }
  });
}

// The reference's own bsdf::sample for etxb_sample_query records (include/etx_b200.h), with the fixed values a bounce pushes
// (vcm_shared.hxx:1013-1027: rnd_bsdf, rnd_connection, rnd_support, push_fixed, sample, pop_fixed) in mode 0 or the query's own in
// mode 1.  One etxb_sample_result per (query, repetition r), repetition r on Sampler(seed, r), as etxb_debug_bsdf_sample writes them.
static_assert(sizeof(etxb_sample_query) == 96);
static_assert(sizeof(etxb_sample_result) == 48);
void oracle_bsdf_sample(void* h, const etxb_sample_query* queries, uint32_t count, uint32_t repetitions, uint32_t threads, etxb_sample_result* out) {
  auto* o = static_cast<Oracle*>(h);
  const Scene& scene = o->scene;
  parallel_ranges(count * repetitions, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t) {
    for (uint32_t t = begin; t < end; ++t) {
      const etxb_sample_query& q = queries[t / repetitions];
      Vertex v = {};
      v.nrm = {q.nrm[0], q.nrm[1], q.nrm[2]};
      v.tan = {q.tan[0], q.tan[1], q.tan[2]};
      v.btn = {q.btn[0], q.btn[1], q.btn[2]};
      v.tex = {q.uv[0], q.uv[1]};
      const float3 w_i = {q.w_i[0], q.w_i[1], q.w_i[2]};
      const SpectralQuery spect = scene.spectral() ? SpectralQuery{q.wavelength, SpectralQuery::Spectral} : SpectralQuery::sample();
      const BSDFData data(spect, q.medium, static_cast<PathSource>(q.path_source), v, w_i);
      Sampler smp(q.seed, t % repetitions);
      etxb_sample_result& dst = out[t];
      dst.seed_start = smp.seed;
      if (q.mode == 0u) {
        const float2 rnd_bsdf = smp.next_2d();
        smp.next_2d();  // rnd_connection
        const float2 rnd_support = smp.next_2d();
        smp.push_fixed(rnd_bsdf.x, rnd_bsdf.y, rnd_support.x);
      } else {
        smp.push_fixed(q.fixed[0], q.fixed[1], q.fixed[2]);
      }
      const BSDFSample s = bsdf::sample(data, scene.materials[q.material], scene, smp);
      smp.pop_fixed();
      const float3 w = s.weight.spectral() ? float3{s.weight.value, s.weight.value, s.weight.value} : s.weight.integrated;
      dst.w_o[0] = s.w_o.x;
      dst.w_o[1] = s.w_o.y;
      dst.w_o[2] = s.w_o.z;
      dst.pdf = s.pdf;
      dst.weight[0] = w.x;
      dst.weight[1] = w.y;
      dst.weight[2] = w.z;
      dst.eta = s.eta;
      dst.properties = s.properties;
      dst.medium_index = s.medium_index;
      dst.seed_end = smp.seed;
    }
  });
}

// The reference's own emitter routines (scene_emitters.hxx) for etxb_emitter_query records (include/etx_b200.h): sample_emitter_index and
// emitter_discrete_pdf (op 0), sample_emitter (op 1), sample_emission on Sampler(seed, r) (op 2), emitter_get_radiance with the
// EmitterRadianceQuery the query describes (op 3).  One etxb_emitter_result per (query, repetition r), as etxb_debug_emitter writes them.
static_assert(sizeof(etxb_emitter_query) == 80);
static_assert(sizeof(etxb_emitter_result) == 104);
void oracle_emitter(void* h, const etxb_emitter_query* queries, uint32_t count, uint32_t repetitions, uint32_t threads, etxb_emitter_result* out) {
  auto* o = static_cast<Oracle*>(h);
  const Scene& scene = o->scene;
  parallel_ranges(count * repetitions, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t) {
    for (uint32_t t = begin; t < end; ++t) {
      const etxb_emitter_query& q = queries[t / repetitions];
      const SpectralQuery spect = scene.spectral() ? SpectralQuery{q.wavelength, SpectralQuery::Spectral} : SpectralQuery::sample();
      const float3 source = {q.source[0], q.source[1], q.source[2]};
      etxb_emitter_result dst = {};
      EmitterSample s = {};
      if (q.op == ETXB_EMITTER_SELECT) {
        s.emitter_index = sample_emitter_index(scene, q.rnd[0]);
        s.pdf_sample = emitter_discrete_pdf(scene.emitter_instances[s.emitter_index], scene.emitters_distribution);
      } else if (q.op == ETXB_EMITTER_SAMPLE_IN) {
        s = sample_emitter(spect, q.emitter, {q.rnd[0], q.rnd[1]}, source, scene);
      } else if (q.op == ETXB_EMITTER_EMISSION) {
        Sampler smp(q.seed, t % repetitions);
        dst.seed_start = smp.seed;
        s = sample_emission(scene, spect, smp);
        dst.seed_end = smp.seed;
      } else {
        EmitterRadianceQuery rq = {
          .source_position = source,
          .target_position = {q.target[0], q.target[1], q.target[2]},
          .direction = {q.direction[0], q.direction[1], q.direction[2]},
          .uv = {q.uv[0], q.uv[1]},
          .directly_visible = q.directly_visible != 0u,
        };
        s.emitter_index = q.emitter;
        s.value = emitter_get_radiance(scene.emitter_instances[q.emitter], spect, rq, s.pdf_area, s.pdf_dir, s.pdf_dir_out, scene);
      }
      const float3 v = s.value.spectral() ? float3{s.value.value, s.value.value, s.value.value} : s.value.integrated;
      const auto put = [](float* d, const float3& a) {
        d[0] = a.x;
        d[1] = a.y;
        d[2] = a.z;
      };
      put(dst.value, v);
      put(dst.origin, s.origin);
      put(dst.normal, s.normal);
      put(dst.direction, s.direction);
      put(dst.barycentric, s.barycentric);
      dst.pdf_sample = s.pdf_sample;
      dst.pdf_area = s.pdf_area;
      dst.pdf_dir = s.pdf_dir;
      dst.pdf_dir_out = s.pdf_dir_out;
      dst.emitter_index = s.emitter_index;
      dst.triangle_index = s.triangle_index;
      dst.medium_index = s.medium_index;
      dst.flags = (s.is_delta ? 1u : 0u) | (s.is_distant ? 2u : 0u);
      out[t] = dst;
    }
  });
}

// The reference's own media routines (scene_medium.hxx, compiled in place: medium_intersects_bounds and medium_sample_density_internal lie
// in its anonymous namespace, visible in this translation unit) for etxb_medium_query records (include/etx_b200.h), and for op 5
// Raytracing::trace_transmittance above with Medium::Instance{.index = medium}.  One etxb_medium_result per (query, repetition r) on
// Sampler(seed, r), as etxb_debug_medium writes them.  The caller keeps to the hook's checks (a valid index, max_t >= kRayEpsilon for op 3).
static_assert(sizeof(etxb_medium_query) == 96);
static_assert(sizeof(etxb_medium_result) == 64);
void oracle_medium(void* h, const etxb_medium_query* queries, uint32_t count, uint32_t repetitions, uint32_t threads, etxb_medium_result* out) {
  auto* o = static_cast<Oracle*>(h);
  const Scene& scene = o->scene;
  parallel_ranges(count * repetitions, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t) {
    for (uint32_t t = begin; t < end; ++t) {
      const etxb_medium_query& q = queries[t / repetitions];
      const SpectralQuery spect = scene.spectral() ? SpectralQuery{q.wavelength, SpectralQuery::Spectral} : SpectralQuery::sample();
      const float3 origin = {q.origin[0], q.origin[1], q.origin[2]}, direction = {q.direction[0], q.direction[1], q.direction[2]};
      const auto put = [](float* d, const float3& a) {
        d[0] = a.x;
        d[1] = a.y;
        d[2] = a.z;
      };
      const auto put_spectral = [&](float* d, const SpectralResponse& s) { put(d, s.spectral() ? float3{s.value, s.value, s.value} : s.integrated); };
      etxb_medium_result dst = {};
      Sampler smp(q.seed, t % repetitions);
      dst.seed_start = smp.seed;
      if (q.op == ETXB_MEDIUM_BOUNDS) {
        float3 pos = origin, dir = direction;
        dst.flag = medium_intersects_bounds(scene.mediums[q.medium], origin, direction, q.max_t, pos, dir, dst.t_min, dst.t_max) ? 1u : 0u;
        put(dst.pos, pos);
        put(dst.dir, dir);
      } else if (q.op == ETXB_MEDIUM_DENSITY) {
        dst.value[0] = medium_sample_density_internal(scene.mediums[q.medium], origin);
      } else if (q.op == ETXB_MEDIUM_TRANSMITTANCE) {
        put_spectral(dst.value, medium_transmittance(scene, scene.mediums[q.medium], spect, smp, origin, direction, q.max_t));
      } else if (q.op == ETXB_MEDIUM_SAMPLE) {
        const SpectralResponse throughput =
          scene.spectral() ? SpectralResponse{spect, q.throughput[0]} : SpectralResponse{spect, float3{q.throughput[0], q.throughput[1], q.throughput[2]}};
        const Medium::Sample s = sample_medium(scene, scene.mediums[q.medium], spect, throughput, smp, origin, direction, q.max_t);
        put_spectral(dst.value, s.weight);
        put(dst.pos, s.pos);
        dst.t = s.sampled_medium_t;
      } else if (q.op == ETXB_MEDIUM_PHASE) {
        dst.value[0] = phase_function(direction, {q.w_o[0], q.w_o[1], q.w_o[2]}, q.g);
        put(dst.dir, sample_phase_function(direction, q.g, {q.rnd[0], q.rnd[1]}));
      } else {
        const SpectralResponse tr = o->rt.trace_transmittance(spect, scene, origin, {q.end[0], q.end[1], q.end[2]}, Medium::Instance{.index = q.medium}, smp);
        put_spectral(dst.value, tr);
      }
      dst.seed_end = smp.seed;
      out[t] = dst;
    }
  });
}

// The reference's own subsurface routines (scene_bssrdf_subsurface.hxx and subsurface::gather of path_tracing_shared.hxx, compiled in
// place) for etxb_subsurface_query records (include/etx_b200.h), with Raytracing::trace_material and continuous_trace above for ops 0 and
// 1.  Entries are make_intersection(scene, dir, {{u, v}, triangle, 0}), as etxb_debug_subsurface builds them.  One etxb_subsurface_result
// per (query, repetition r) on Sampler(seed, r).  The caller keeps to the hook's checks, except that a zero direction is traced as given.
static_assert(sizeof(etxb_subsurface_query) == 128);
static_assert(sizeof(etxb_subsurface_result) == 1920);
void oracle_subsurface(void* h, const etxb_subsurface_query* queries, uint32_t count, uint32_t repetitions, uint32_t threads, etxb_subsurface_result* out) {
  auto* o = static_cast<Oracle*>(h);
  const Scene& scene = o->scene;
  parallel_ranges(count * repetitions, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t) {
    for (uint32_t t = begin; t < end; ++t) {
      const etxb_subsurface_query& q = queries[t / repetitions];
      const SpectralQuery spect = scene.spectral() ? SpectralQuery{q.wavelength, SpectralQuery::Spectral} : SpectralQuery::sample();
      const float3 origin = {q.origin[0], q.origin[1], q.origin[2]}, direction = {q.dir[0], q.dir[1], q.dir[2]};
      const auto put = [](float* d, const float3& a) {
        d[0] = a.x;
        d[1] = a.y;
        d[2] = a.z;
      };
      const auto put_spectral = [&](float* d, const SpectralResponse& s) { put(d, s.spectral() ? float3{s.value, s.value, s.value} : s.integrated); };
      const auto put_probe = [&](etxb_subsurface_probe& d, const subsurface::Sample& s) {
        put(d.o, s.ray.o);
        put(d.d, s.ray.d);
        d.min_t = s.ray.min_t;
        d.max_t = s.ray.max_t;
        put(d.u, s.u);
        put(d.v, s.v);
        put(d.w, s.w);
        put(d.basis_prob, s.basis_prob);
        d.sampled_radius = s.sampled_radius;
      };
      etxb_subsurface_result& dst = out[t];
      dst = {};
      Sampler smp(q.seed, t % repetitions);
      dst.seed_start = smp.seed;
      const Ray ray = {origin, direction, q.t_min, q.t_max};
      if (q.op == ETXB_SUBSURFACE_TRACE_MATERIAL) {
        Intersection i;
        const bool found = o->rt.trace_material(scene, ray, q.material, i, smp);
        dst.count = found ? 1u : 0u;
        dst.hits[0].tri = kInvalidIndex;
        if (found) {
          dst.hits[0] = {i.barycentric.y, i.barycentric.z, i.t, i.triangle_index};
        }
      } else if (q.op == ETXB_SUBSURFACE_CONTINUOUS_TRACE) {
        IntersectionBase buffer[subsurface::kIntersectionsPerDirection] = {};
        dst.count = o->rt.continuous_trace(scene, ray, ContinousTraceOptions{buffer, q.max_count, q.material}, smp);
        for (uint32_t k = 0; k < dst.count; ++k)
          dst.hits[k] = {buffer[k].barycentric.x, buffer[k].barycentric.y, buffer[k].t, buffer[k].triangle_index};
      } else if (q.op == ETXB_SUBSURFACE_REMAP) {
        for (uint32_t k = 0; k < 3u; ++k)
          subsurface::remap_channel(q.color[k], q.distances[k], dst.albedo[k], dst.extinction[k], dst.scattering[k]);
      } else {
        const Intersection in = make_intersection(scene, direction, IntersectionBase{{q.u, q.v}, q.triangle, 0.0f});
        const auto& sss = scene.materials[in.material_index].subsurface;
        if (q.op == ETXB_SUBSURFACE_PROFILE) {
          dst.s_r = subsurface::sample_s_r(q.rnd);
          put_spectral(dst.eval, subsurface::evaluate(spect, scene, in, sss, q.radius));
          const subsurface::Sample s = subsurface::sample(spect, scene, in, sss, q.direction, smp);
          put_probe(dst.probes[0], s);
          dst.geometric_weight = subsurface::geometric_weigth({q.normal[0], q.normal[1], q.normal[2]}, s);
        } else {
          if (sss.cls == SubsurfaceMaterial::Class::ChristensenBurley) {  // the gather's three probes are its first draws
            Sampler probe_smp = smp;
            for (uint32_t d = 0; d < subsurface::kIntersectionDirections; ++d)
              put_probe(dst.probes[d], subsurface::sample(spect, scene, in, sss, d, probe_smp));
          }
          subsurface::Gather g = {};
          const uint32_t rays_before = g_material_rays;
          dst.flag = (subsurface::gather(spect, scene, in, o->rt, smp, g) == subsurface::GatherResult::Succeedded) ? 1u : 0u;
          dst.rays = g_material_rays - rays_before;
          if (dst.flag) {
            dst.count = g.intersection_count;
            dst.selected = g.selected_intersection;
            dst.selected_sample_weight = g.selected_sample_weight;
            dst.total_weight = g.total_weight;
            for (uint32_t k = 0; k < g.intersection_count; ++k) {
              const Intersection& e = g.intersections[k];
              etxb_subsurface_hit& hk = dst.hits[k];
              hk.u = e.barycentric.y;
              hk.v = e.barycentric.z;
              hk.t = e.t;
              hk.tri = e.triangle_index;
              put(hk.w_i, e.w_i);
              put_spectral(hk.weight, g.weights[k]);
              put(hk.pos, e.pos);
              put(hk.nrm, e.nrm);
            }
          }
        }
      }
      dst.seed_end = smp.seed;
    }
  });
}

// The reference's own photon gather (VCMSpatialGridData::gather, vcm_shared.hxx:886-924) for etxb_debug_merge's inputs: the light-vertex
// records (device layout, 96 B) become o.light_vertices and build_grid runs on them at the current iteration; each query becomes the
// Intersection make_intersection builds for its hit (as oracle_trace does) and a VCMPathState, and is gathered `repetitions` times on
// Sampler(seed, r).  out = double[8] per query: the mean and the (population) variance of the merged rgb over the repetitions, the sampler
// state after repetition 0, 0.  grid_out = bbox min, bbox max, cell size, radius squared, hash table mask, photon count.
struct MergeRecord {
  float thr[3], d_vcm, w_i[3], d_vc, bc[3], d_vm, pos[3];
  uint32_t tri;
  float nrm[3];
  uint32_t material, medium, path_length, path_index, ordinal;
};
static_assert(sizeof(MergeRecord) == 96);
static_assert(sizeof(etxb_merge_query) == 64);
void oracle_merge(void* h, const void* records, uint32_t record_count, const float* light_wavelengths, const etxb_merge_query* queries, uint32_t count,
                  uint32_t repetitions, uint32_t threads, double* out, double* grid_out) {
  auto* o = static_cast<Oracle*>(h);
  const Scene& scene = o->scene;
  const bool spectral = scene.spectral();
  auto response = [spectral](float wavelength, const float* v) {
    return spectral ? SpectralResponse{SpectralQuery{wavelength, SpectralQuery::Spectral}, v[0]} : SpectralResponse{SpectralQuery::sample(), float3{v[0], v[1], v[2]}};
  };
  start_next_iteration(*o);
  o->light_vertices.assign(record_count, VCMLightVertex{});
  const auto* recs = static_cast<const MergeRecord*>(records);
  for (uint32_t k = 0; k < record_count; ++k) {
    const MergeRecord& r = recs[k];
    VCMLightVertex& v = o->light_vertices[k];
    v.throughput = response(light_wavelengths[r.path_index], r.thr);
    v.w_i = {r.w_i[0], r.w_i[1], r.w_i[2]};
    v.d_vcm = r.d_vcm;
    v.bc = {r.bc[0], r.bc[1], r.bc[2]};
    v.d_vc = r.d_vc;
    v.pos = {r.pos[0], r.pos[1], r.pos[2]};
    v.d_vm = r.d_vm;
    v.nrm = {r.nrm[0], r.nrm[1], r.nrm[2]};
    v.triangle_index = r.tri;
    v.material_index = r.material;
    v.medium_index = r.medium;
    v.is_medium = (r.tri == kInvalidIndex);
    v.path_length = r.path_length;
    v.path_index = r.path_index;
  }
  if (o->options.merge_vertices()) {
    build_grid(*o);
  } else {
    o->grid = {};
  }
  const VCMSpatialGridData& grid = o->grid;
  const double g[10] = {grid.bounding_box.p_min.x, grid.bounding_box.p_min.y, grid.bounding_box.p_min.z, grid.bounding_box.p_max.x, grid.bounding_box.p_max.y,
    grid.bounding_box.p_max.z, grid.cell_size, grid.radius_squared, double(grid.hash_table_mask), double(grid.positions.count)};
  for (uint32_t k = 0; k < 10; ++k)
    grid_out[k] = g[k];
  parallel_ranges(count, threads, [&](uint32_t begin, uint32_t end, uint32_t, uint32_t) {
    for (uint32_t i = begin; i < end; ++i) {
      const etxb_merge_query& q = queries[i];
      const float3 w_i = {q.w_i[0], q.w_i[1], q.w_i[2]};
      const Intersection isect = make_intersection(scene, w_i, IntersectionBase{{q.u, q.v}, q.tri, 0.0f});
      double mean[3] = {}, m2[3] = {};
      double* dst = out + size_t(i) * 8u;
      for (uint32_t r = 0; r < repetitions; ++r) {
        VCMPathState state = {};
        state.throughput = response(q.wavelength, q.throughput);
        state.spect = state.throughput;
        state.ray.d = w_i;
        state.d_vcm = q.d_vcm;
        state.d_vm = q.d_vm;
        state.total_path_depth = q.total_path_depth;
        state.medium_index = q.medium;
        state.sampler = Sampler(q.seed, r);
        const float3 m = grid.gather(scene, state, o->options, isect, o->iteration.vc_weight);
        const double v[3] = {m.x, m.y, m.z};
        for (uint32_t k = 0; k < 3; ++k) {
          const double delta = v[k] - mean[k];
          mean[k] += delta / double(r + 1u);
          m2[k] += delta * (v[k] - mean[k]);
        }
        if (r == 0)
          dst[6] = double(state.sampler.seed);
      }
      for (uint32_t k = 0; k < 3; ++k) {
        dst[k] = mean[k];
        dst[3 + k] = m2[k] / double(std::max(repetitions, 1u));
      }
      dst[7] = 0.0;
    }
  });
}

// ---- known-answer helpers straight from the reference headers ----------------------------------------
void oracle_sampler(const uint32_t* a, const uint32_t* b, uint32_t count, uint32_t draws, uint32_t* out_seed, float* out_values) {
  for (uint32_t i = 0; i < count; ++i) {
    Sampler s(a[i], b[i]);
    out_seed[size_t(i) * (draws + 1u)] = s.seed;
    for (uint32_t d = 0; d < draws; ++d) {
      out_values[size_t(i) * draws + d] = s.next();
      out_seed[size_t(i) * (draws + 1u) + d + 1u] = s.seed;
    }
  }
}

// fn ids shared with etxb_debug_math (etx_tracer_b200/csrc/debug_ids.h)
void oracle_math(uint32_t fn, const float* x, const float* y, uint32_t count, float* out) {
  for (uint32_t i = 0; i < count; ++i) {
    float a = x[i], b = y ? y[i] : 0.0f;
    float r = 0.0f;
    switch (fn) {
      case 0: r = sinf(a); break;
      case 1: r = cosf(a); break;
      case 2: r = expf(a); break;
      case 3: r = logf(a); break;
      case 4: r = powf(a, b); break;
      case 5: r = acosf(a); break;
      case 6: r = atan2f(a, b); break;
      case 7: r = SpectralQuery::spectral_sample(a).wavelength; break;
      case 8: r = SpectralQuery{a, SpectralQuery::Spectral}.sampling_pdf(); break;
      case 9: r = SpectralResponse{SpectralQuery{a, SpectralQuery::Spectral}, 1.0f}.to_rgb().x; break;
      case 10: r = SpectralResponse{SpectralQuery{a, SpectralQuery::Spectral}, 1.0f}.to_rgb().y; break;
      case 11: r = SpectralResponse{SpectralQuery{a, SpectralQuery::Spectral}, 1.0f}.to_rgb().z; break;
      case 12: r = atanf(a); break;
      case 13: r = asinf(a); break;
      case 14: r = sample_blue_noise({uint32_t(a) & 127u, uint32_t(a) >> 7}, 256u, uint32_t(b), 0).x; break;
      case 15: r = sample_blue_noise({uint32_t(a) & 127u, uint32_t(a) >> 7}, 256u, uint32_t(b), 4).y; break;
      default: break;
    }
    out[i] = r;
  }
}

void oracle_offset_ray(const float* p, const float* n, float* out) {
  float3 r = offset_ray({p[0], p[1], p[2]}, {n[0], n[1], n[2]});
  out[0] = r.x;
  out[1] = r.y;
  out[2] = r.z;
}

uint32_t oracle_grid_cell_index(uint32_t mask, int32_t x, int32_t y, int32_t z) {
  VCMSpatialGridData g = {};
  g.hash_table_mask = mask;
  return g.cell_index(x, y, z);
}

// ---- scene-building helpers (reference host code: render/host/spectrum.cxx) --------------------------
void oracle_spectrum_rgb_reflectance(const float* rgb, void* out_spd) {
  auto s = SpectralDistribution::rgb_reflectance({rgb[0], rgb[1], rgb[2]});
  memcpy(out_spd, &s, sizeof(s));
}
void oracle_spectrum_rgb_luminance(const float* rgb, void* out_spd) {
  auto s = SpectralDistribution::rgb_luminance({rgb[0], rgb[1], rgb[2]});
  memcpy(out_spd, &s, sizeof(s));
}
void oracle_spectrum_constant(float value, void* out_spd) {
  auto s = SpectralDistribution::constant(value);
  memcpy(out_spd, &s, sizeof(s));
}
void oracle_spectrum_blackbody(float temperature, float scale, int normalized, void* out_spd) {
  auto s = normalized ? SpectralDistribution::from_normalized_black_body(temperature, scale) : SpectralDistribution::from_black_body(temperature, scale);
  memcpy(out_spd, &s, sizeof(s));
}
int oracle_spectrum_load_ior(const char* file_name, void* out_eta, void* out_k) {
  SpectralDistribution eta, k;
  auto cls = RefractiveIndex::load_from_file(file_name, eta, k, nullptr);
  memcpy(out_eta, &eta, sizeof(eta));
  memcpy(out_k, &k, sizeof(k));
  return int(cls);
}
float oracle_spectrum_luminance(const void* spd) {
  SpectralDistribution s;
  memcpy(&s, spd, sizeof(s));
  return s.luminance();
}
void oracle_color_tables(float* xyz_441x3, float* rgb_response_391x3, float* y_integral) {
  for (uint32_t i = 0; i < spectrum::WavelengthCount; ++i) {
    float3 v = spectrum::spectral_xyz(i);
    xyz_441x3[i * 3 + 0] = v.x;
    xyz_441x3[i * 3 + 1] = v.y;
    xyz_441x3[i * 3 + 2] = v.z;
  }
  for (uint32_t i = 0; i < spectrum::RGBResponseWavelengthCount; ++i) {
    SpectralQuery q = {float(i + spectrum::RGBResponseShortestWavelength), SpectralQuery::Spectral};
    rgb_response_391x3[i * 3 + 0] = rgb_response(q, {1.0f, 0.0f, 0.0f}).value;
    rgb_response_391x3[i * 3 + 1] = rgb_response(q, {0.0f, 1.0f, 0.0f}).value;
    rgb_response_391x3[i * 3 + 2] = rgb_response(q, {0.0f, 0.0f, 1.0f}).value;
  }
  *y_integral = spectrum::kYIntegral();
}
void oracle_build_camera(void* camera_blob, const float* origin, const float* target, const float* up, uint32_t w, uint32_t h, float fov) {
  // scene_representation.cxx:579-598 (build_camera) restated
  Camera camera;
  memcpy(&camera, camera_blob, sizeof(Camera));
  float3 o = {origin[0], origin[1], origin[2]}, t = {target[0], target[1], target[2]}, u = {up[0], up[1], up[2]};
  float4x4 view = look_at(o, t, u);
  float4x4 proj = perspective(fov * kPi / 180.0f, w, h, camera.clip_near, camera.clip_far);
  float4x4 inv_view = inverse(view);
  camera.target = t;
  camera.position = {inv_view.col[3].x, inv_view.col[3].y, inv_view.col[3].z};
  camera.side = {view.col[0].x, view.col[1].x, view.col[2].x};
  camera.up = {view.col[0].y, view.col[1].y, view.col[2].y};
  camera.direction = {-view.col[0].z, -view.col[1].z, -view.col[2].z};
  camera.tan_half_fov = 1.0f / std::abs(proj.col[0].x);
  camera.aspect = proj.col[1].y / proj.col[0].x;
  camera.view_proj = proj * view;
  float plane_w = 2.0f * camera.tan_half_fov;
  float plane_h = 2.0f * camera.tan_half_fov / camera.aspect;
  camera.area = plane_w * plane_h;
  camera.film_size = {w, h};
  camera.image_plane = float(camera.film_size.x) / (2.0f * camera.tan_half_fov);
  memcpy(camera_blob, &camera, sizeof(Camera));
}

// sizeof table checked against include/etx_b200.h by tests/test_layout.py
uint32_t oracle_sizeof(uint32_t id) {
  switch (id) {
    case 0: return sizeof(Scene);
    case 1: return sizeof(Camera);
    case 2: return sizeof(Vertex);
    case 3: return sizeof(Triangle);
    case 4: return sizeof(Material);
    case 5: return sizeof(EmitterProfile);
    case 6: return sizeof(Emitter);
    case 7: return sizeof(SpectralDistribution);
    case 8: return sizeof(Image);
    case 9: return sizeof(Medium);
    case 10: return sizeof(Distribution);
    case 11: return sizeof(VCMPathState);
    case 12: return sizeof(VCMLightVertex);
    default: return 0;
  }
}

}  // extern "C"
