// module.cu — C ABI (include/etx_b200.h) over the wavefront kernels: context, scene upload, iteration driver.
// Host-side counterpart of CPUVCMImpl (sources/etx/rt/integrators/vcm_cpu.cxx:30-241) and of
// Raytracing::commit_changes (sources/etx/rt/rt.cxx:58-88).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <deque>
#include <string>
#include <utility>
#include <vector>

#include <dlfcn.h>
#include <nccl.h>

#include "bvh_build.h"
#include "bvh_build_device.h"
#include "kernels.cuh"
#include "kernels_pt.cuh"
#include "kernels_denoise.cuh"

using namespace etxb;

#if defined(ETXB_PARITY) && ETXB_PARITY
static const char* kFlavor = "parity";
#else
static const char* kFlavor = "fast";
#endif

namespace {

enum KernelId : uint32_t {
  K_LIGHT_BEGIN,
  K_TRACE_LIGHT,
  K_LIGHT_BOUNCE,
  K_LV_SCAN,
  K_LV_REORDER,
  K_GRID_BBOX,
  K_GRID_KEYS,
  K_GRID_SORT,
  K_GRID_BUILD,
  K_CAMERA_BEGIN,
  K_TRACE_CAMERA,
  K_CAMERA_SHADE,
  K_CAMERA_CONNECT,
  K_SHADOW_TRACE,
  K_QUEUE_SORT,
  K_CAMERA_MERGE_SORT,
  K_CAMERA_MERGE,
  K_CAMERA_MERGE_GENERIC,
  K_CAMERA_CONTINUE,
  K_FILM_COMMIT,
  K_COMM_LIGHT_IMAGE,
  K_COMM_PHOTONS,
  K_PT_BEGIN,
  K_PT_SHADE,
  K_PT_ACCUMULATE,
  K_FILM_NOISE,
  K_BVH_BUILD,
  K_BVH_WIDE,
  K_FILM_ADAPTIVE,
  K_DENOISE_VARIANCE,
  K_DENOISE_SMOOTH,
  K_DENOISE_NLM,
  K_COMM_PT_MASK,
  K_COMM_PT_COUNT,
  K_COUNT
};
const char* kKernelNames[K_COUNT] = {"light_begin", "trace_closest(light)", "light_bounce", "lv_scan", "lv_reorder", "grid_bbox", "grid_keys", "grid_sort", "grid_build",
  "camera_begin", "trace_closest(camera)", "camera_shade", "camera_connect", "shadow_trace", "queue_sort", "camera_merge_sort", "camera_merge", "camera_merge_generic", "camera_continue", "film_commit_light", "nccl_allreduce_light_image", "nccl_allgather_photons",
  "pt_begin", "pt_shade", "pt_accumulate", "film_noise_levels", "bvh_build", "bvh_collapse_wide",
  "film_adaptive_vcm", "denoise_variance", "denoise_smooth", "denoise_nlm", "nccl_allreduce_pt_mask", "nccl_allreduce_pt_count"};

// Queue sizes from which a pass takes its large-queue branches (the context's `thresholds`; etxb_debug_set_thresholds overrides them):
//   merge_sort_min_queries  the gather queue is sorted by its merge keys (below it, a latency-bound tail, the sort launches cost more than they save)
//   merge_min_warps_per_sm  the gather gives each warp up to 32 queries while the queue still fills this many warps per SM
//   tail_queue              vertex connections go through the host-sized, material-pair-sorted list, and the queue count is read every bounce
//   sort_queue_min          path queues and connection lists are grouped by material (scenes with stochastic BSDFs)
constexpr etxb_debug_thresholds kDefaultThresholds = {16384u, 32u, 8192u, 1024u, 0u};

// A device allocation with one owner: it is freed when the buffer is destroyed, on the device that is current then.
template <class T>
struct DevBuf {
  T* ptr = nullptr;
  size_t count = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : ptr(std::exchange(o.ptr, nullptr)), count(std::exchange(o.count, size_t(0))) {}
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      release();
      ptr = std::exchange(o.ptr, nullptr);
      count = std::exchange(o.count, size_t(0));
    }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t alloc(size_t n) {
    release();
    count = n;
    if (n == 0) return cudaSuccess;
    return cudaMalloc(&ptr, n * sizeof(T));
  }
  // alloc that keeps the allocation when it already holds n elements; counts the allocations it makes
  cudaError_t ensure(size_t n, uint32_t& allocations) {
    if (ptr && (count == n)) return cudaSuccess;
    allocations += 1;
    return alloc(n);
  }
  void release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    count = 0;
  }
  size_t bytes() const { return count * sizeof(T); }
};

struct TimedLaunch {
  uint32_t kernel;
  cudaEvent_t start, stop;
};

// 128-bit content hash of a byte range, chained through `seed`: four independent 64-bit multiply-rotate lanes over 32-byte stripes (the
// round of xxHash64), a zero-padded tail, and two differently mixed 64-bit digests of the lanes and the length.  It detects edits, not
// adversaries.
struct Hash128 {
  uint64_t lo = 0, hi = 0;
  bool operator==(const Hash128& o) const { return (lo == o.lo) && (hi == o.hi); }
};
constexpr uint64_t kHashP1 = 0x9E3779B185EBCA87ull, kHashP2 = 0xC2B2AE3D27D4EB4Full, kHashP3 = 0x165667B19E3779F9ull, kHashP4 = 0x85EBCA77C2B2AE63ull;
inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
inline uint64_t hash_round(uint64_t acc, uint64_t w) { return rotl64(acc + w * kHashP2, 31) * kHashP1; }
inline uint64_t hash_mix(uint64_t h) {
  h ^= h >> 33;
  h *= kHashP2;
  h ^= h >> 29;
  h *= kHashP3;
  return h ^ (h >> 32);
}
Hash128 hash128(const void* data, size_t bytes, Hash128 seed) {
  const uint8_t* p = static_cast<const uint8_t*>(data);
  uint64_t v[4] = {seed.lo + kHashP1 + kHashP2, seed.hi + kHashP2, seed.lo ^ kHashP3, seed.hi - kHashP1};
  size_t i = 0;
  for (; i + 32 <= bytes; i += 32) {
    uint64_t w[4];
    memcpy(w, p + i, 32);
    for (int k = 0; k < 4; ++k) v[k] = hash_round(v[k], w[k]);
  }
  uint64_t tail[4] = {0, 0, 0, 0};
  if (bytes > i) memcpy(tail, p + i, bytes - i);
  for (int k = 0; k < 4; ++k) v[k] = hash_round(v[k], tail[k]);
  const uint64_t a = rotl64(v[0], 1) + rotl64(v[1], 7) + rotl64(v[2], 12) + rotl64(v[3], 18);
  const uint64_t b = (v[0] * kHashP4) ^ rotl64(v[1], 29) ^ (v[2] * kHashP3) ^ rotl64(v[3], 43);
  return {hash_mix(a ^ (uint64_t(bytes) * kHashP4)), hash_mix(b + uint64_t(bytes) * kHashP1)};
}

// what the last upload / update of a context copied, by content (etxb_update_scene keeps what did not change)
struct SceneHashes {
  bool valid = false;  // set once the whole scene is on the device
  Hash128 geometry;    // vertex array + triangle array: device vertices, triangles, BVH2 (+ the 4-wide tree)
  std::vector<Hash128> images, grids;  // per image; per medium (zero for media without a density grid)
};

}  // namespace

struct etxb_ctx {
  int device = 0;
  uint32_t sm_count = 132;  // the device's multiprocessors (set at creation): persistent and grid-stride launches are sized by it
  cudaStream_t stream = nullptr;
  std::string error;
  bool scene_ready = false;
  bool spectral = false;
  bool profile = false;
  bool has_stochastic_merge = false;  // some material that can be merged at is not Lambert (needs the generic gather)
  bool plain_scene = false;           // set at upload: no media, Boundary surfaces or subsurface (the bounce kernels' PLAIN instantiation)
  bool opaque_scene = false;          // set at upload: no alpha test can reject a hit (every opacity 1, no alpha images), no Boundary surfaces / media

  // scene in HBM
  DevBuf<DVertex> vertices;
  DevBuf<DTriangle> triangles;
  DevBuf<uint32_t> tri_emitter;
  DevBuf<etxb_material> materials;
  DevBuf<etxb_emitter_profile> profiles;
  DevBuf<etxb_emitter> emitters;
  DevBuf<DSpectrum> spectra;
  DevBuf<DImage> images;
  DevBuf<DMedium> mediums;
  std::vector<DevBuf<float>> medium_density;
  std::vector<DevBuf<uint8_t>> image_pixels, image_dists;
  DevBuf<etxb_distribution_entry> emitter_dist;
  DevBuf<BvhNode> bvh_nodes;
  DevBuf<WideNode> wide_nodes;
  bool wide_rejected = false;         // the committed geometry's 4-wide tree exceeds kWideStackSize (the scene walks the BVH2)
  bool debug_trace_wide = false;      // etxb_debug_select_tree: etxb_debug_trace walks the 4-wide tree when the scene has one
  DevBuf<float4> bvh_tris;
  DevBuf<float> xyz_table, rgb_response_table;
  DevBuf<uint8_t> bn_sobol, bn_scrambling, bn_ranking;
  float y_integral = 0.0f;
  DeviceScene dscene = {};
  double bvh_build_seconds = 0.0;
  SceneHashes hashes;

  // per-path state + queues.  path_count = W * H sizes the film and every path-indexed buffer; launch_count = Film::pixel_count() is the
  // number of paths an iteration traces: W * H at pixel size 1, ceil(W / s) * ceil(H / s) in the coarse preview
  uint32_t width = 0, height = 0, path_count = 0, launch_count = 0;
  uint32_t pixel_size = 1, target_pixel_size = 1;  // Film::pixel_size, and the one etxb_set_film_pixel_size stored for the next etxb_begin
  DevBuf<float4> ray_o, ray_d, thr, mis, hit, gathered, merged, camera_value, bs_weight_pdf, bs_wo_eta;
  DevBuf<uint4> misc;
  DevBuf<uint2> bs_props;
  DevBuf<float> wavelength;
  DevBuf<uint32_t> queue_sorted, queue_keys, queue_keys_sorted;  // path queue grouped by hit material (scenes with stochastic BSDFs)
  DevBuf<uint2> conn_list_sorted;
  DevBuf<uint32_t> lv_count, lp_offset, queue_a, queue_b, queue_counts, sampler_end_light, sampler_end_camera, merge_key, conn_count;
  DevBuf<float4> conn_rec;  // product build, scenes with a connection stage: kConnRecRows rows per path (kernels.cuh)
  DevBuf<uint2> conn_list, shadow_span;
  DevBuf<float4> shadow_p0, shadow_p1, shadow_value;
  DevBuf<uint32_t> shadow_result, shadow_count, trace_cursor;  // trace_cursor: work cursor of k_shadow_resolve
  // light vertices + grid
  uint32_t lv_capacity = 0, max_light_vertices_cfg = 0;
  DevBuf<LightVertexRec> lv_tmp, lv_final;
  DevBuf<uint32_t> lv_tmp_count, overflow, grid_bbox, keys_in, keys_out, vals_in, vals_out;
  DevBuf<uint2> cell_range;
  DevBuf<float4> g_pos, g_nrm, g_win, g_thr;
  DevBuf<uint8_t> cub_temp;
  DevBuf<DeviceCounters> counters;
  // film
  DevBuf<float4> film_camera, film_light, film_light_iteration, film_out;

  // unidirectional path tracer (SURVEY 8(f) N3): the same context renders with CPUPathTracing's algorithm once etxb_set_integrator selects it
  uint32_t integrator = ETXB_INTEGRATOR_VCM;
  etxb_pt_options pt_options = {1u, 1u, 1u, 1u};
  DevBuf<float4> film_normals, film_albedo, film_adaptive;  // Film's Normals / Albedo / CameraAdaptive layers (allocated with the first PT run;
                                                           // CameraAdaptive also with the first VCM camera pass)
  DevBuf<float4> film_denoised;                             // Film's Denoised layer: the last etxb_denoise, zeros before it (StorageDenoised)
  DevBuf<float4> denoise_u, denoise_var_raw, denoise_var;   // etxb_denoise scratch: colour with its flags, variance, smoothed variance
  DevBuf<uint32_t> denoise_flag;                            // set by k_denoise_variance where a pixel has fewer than two samples
  DevBuf<uint32_t> film_ldr;                                 // the tone-mapped RGBA8 frame of etxb_read_film_ldr
  DevBuf<uint32_t> pt_info;                                  // InternalData (sample count, converged, tmp)
  DevBuf<uint32_t> pt_mask;                                  // the noise estimate's active mask + kNoiseStats (kernels_pt.cuh)
  DevBuf<float> pt_error;
  uint32_t pixel_sampler_image = 0xffffffffu;
  float pixel_sampler_radius = 1.0f, noise_threshold = 0.0f, radiance_clamp = 0.0f;
  uint32_t scene_samples = 0;
  uint32_t pt_pixels_processed = 0, pt_active_pixels = 0;  // active pixels of the last iteration; Film::active_pixel_count (over all ranks
                                                           // on a context with a communicator)
  float pt_noise_level = 0.0f;                             // Film::noise_level

  etxb_vcm_options options = {};
  uint32_t iteration = 0;            // absolute iteration index (VCMIteration::iteration)
  bool external_iteration = false;   // etxb_set_next_iteration: the caller sets every iteration's index, it does not advance by itself
  uint32_t completed = 0;            // iterations finished since etxb_begin
  uint32_t rank = 0, world = 1;
  bool group_lane = false;           // a lane of an etxb_group (etxb_group_create)
  bool light_full = false;           // camera-split iterations (etxb_group replicas): the partition applies to the camera pass only, the light pass traces every path
  uint32_t last_light_vertices = 0;
  uint32_t overflow_flag = 0;
  double last_iteration_time = 0.0, total_time = 0.0;
  uint64_t kernel_launches = 0;
  GridData grid = {};
  // queue sizes from which a pass takes its large-queue branches (etxb_debug_set_thresholds; 0 = always, 0xffffffff = never), and what ran
  etxb_debug_thresholds thresholds = kDefaultThresholds;
  etxb_debug_branch_counts branch_counts = {};

  // pixel-tile sharding across processes (one per GPU): NCCL communicator over NVLink, created by etxb_comm_init
  ncclComm_t comm = nullptr;
  cudaStream_t comm_stream = nullptr;  // highest priority: a collective's few CTAs start as soon as ANY slot frees up instead of queueing behind the
                                       // tens of thousands of blocks of another lane's kernel (measured, 2 GPUs x 4 lanes: 43 ms per all-reduce waiting otherwise)
  cudaEvent_t comm_ev_in = nullptr, comm_ev_out = nullptr;
  DevBuf<uint32_t> comm_counts;   // [world] stored light vertices per rank (all-gathered every iteration)
  DevBuf<float4> film_reduced;    // rank 0: sum of every rank's camera tiles (etxb_comm_reduce_film)
  double comm_ms = 0.0;           // device time of the collectives of the iterations since etxb_begin

  // etxb_enqueue_iteration is asynchronous (CPUVCM::update returns at once, vcm_cpu.cxx:264-276): the iteration's host loop — it reads queue
  // sizes back between bounces — runs on this context's own worker thread; etxb_poll never blocks, etxb_wait drains
  std::thread worker;
  std::mutex worker_m;
  std::condition_variable worker_cv, worker_idle;
  uint32_t worker_queued = 0;
  bool worker_busy = false, worker_quit = false;
  int worker_error = ETXB_OK;

  cudaEvent_t ev_iter_start = nullptr, ev_iter_stop = nullptr;
  std::vector<TimedLaunch> timed;
  std::vector<cudaEvent_t> event_pool;
  size_t event_cursor = 0;
  float kernel_ms[K_COUNT] = {};
  uint32_t kernel_count[K_COUNT] = {};

  // frees the device buffers; a C++ symbol, kept out of the library's exports (the interface is etxb_destroy)
  __attribute__((visibility("hidden"))) ~etxb_ctx() = default;
};

// ---------------------------------------------------------------------------------------------------------------------
// Iterations in flight (etxb_group): L contexts on one device, one host thread each, pulling iteration indices from per-lane
// queues (WorkPlan).  VCM iterations are independent (vcm_cpu.cxx:95-113: the index only sets the merge radius and the sampler seeds), and
// the bounce loop of one iteration ends in a long latency-bound tail (a few thousand paths, ~50 bounces); with several iterations in
// flight that tail overlaps the full-width head of another iteration.  The film is the mean of the lanes' films weighted by the
// iterations each lane finished — the same set of iterations, hence the same estimate, as one context running them in sequence.
// ---------------------------------------------------------------------------------------------------------------------
extern "C" {  // the film-combine kernels keep unmangled names in the module
constexpr uint32_t kMaxLanes = 9;  // 8 whole-iteration lanes + the camera-split lane of the replica mode
struct FilmLanes {
  const float4* camera[kMaxLanes];
  const float4* light[kMaxLanes];
  float weight[kMaxLanes];        // camera layer
  float weight_light[kMaxLanes];  // light layer (differs from `weight` only for a camera-split lane that is not part 0)
  float weight_count[kMaxLanes];  // raw mode: what the lane adds to .w
  uint32_t lanes, layer, pixels;
  uint32_t raw;  // 1: no clamp, alpha = sum of the weights (a partial sum that another stage finishes)
};
__global__ void __launch_bounds__(256) k_film_combine(FilmLanes f, float4* out) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f.pixels) return;
  float x = 0.0f, y = 0.0f, z = 0.0f;
  for (uint32_t l = 0; l < f.lanes; ++l) {
    float4 c = (f.layer != ETXB_FILM_LIGHT) ? f.camera[l][i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    float4 g = (f.layer != ETXB_FILM_CAMERA) ? f.light[l][i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    x += f.weight[l] * c.x + f.weight_light[l] * g.x;
    y += f.weight[l] * c.y + f.weight_light[l] * g.y;
    z += f.weight[l] * c.z + f.weight_light[l] * g.z;
  }
  if (f.raw) {
    float w = 0.0f;
    for (uint32_t l = 0; l < f.lanes; ++l) w += f.weight_count[l];
    out[i] = make_float4(x, y, z, w);
    return;
  }
  if (f.layer == ETXB_FILM_RESULT) {  // Film::layer(Result): max(0, camera + light) (film.cxx:381-418)
    x = fmaxf(0.0f, x);
    y = fmaxf(0.0f, y);
    z = fmaxf(0.0f, z);
  }
  out[i] = make_float4(x, y, z, 1.0f);
}
// rank 0 of a replica run: the reduced sum of (iterations x mean film) over the ranks -> the mean over all iterations (.w carries the count)
__global__ void __launch_bounds__(256) k_film_finish_mean(const float4* sum, float4* out, uint32_t pixels, uint32_t clamp) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pixels) return;
  float4 v = sum[i];
  float inv = (v.w > 0.0f) ? 1.0f / v.w : 0.0f;
  float x = v.x * inv, y = v.y * inv, z = v.z * inv;
  if (clamp) {
    x = fmaxf(0.0f, x);
    y = fmaxf(0.0f, y);
    z = fmaxf(0.0f, z);
  }
  out[i] = make_float4(x, y, z, 1.0f);
}
}  // extern "C"

// Which lane renders which iteration of an etxb_group.  etxb_group_enqueue deals the new ordinals into queues (plan_enqueue, the one place
// that reads the mode); lane l pops queues[lane_queue[l]], whatever the mode.
//   local     one GPU: every lane reads queue 0, which holds the ordinals in order, so a free lane takes the next one
//   tiles     etxb_group_comm_init, world >= 2: lane l reads queue l, which holds the ordinals l, l + L, l + 2L, ... on EVERY rank (lane l of every
//             rank shares a communicator; one shared queue would pair different iterations across ranks)
//   replicas  etxb_group_comm_init_replicas, world >= 2: replica_plan deals the job's ordinals; whole frames go to queue 0, which every lane but
//             the split lane reads, and camera-split parts to the split lane's own queue
// The split lane reads its own queue in every mode, which only the replica mode fills; tile mode and a split lane refuse each other.
struct WorkItem {
  uint32_t ordinal;      // of the iteration within the job
  uint32_t part, parts;  // parts == 1: the whole frame; else the camera pass of part `part` (tile % parts == part), light pass in full
};
enum class GroupMode : uint32_t { local = 0, tiles = 1, replicas = 2 };  // the values etxb_debug_group_plan takes
struct WorkPlan {
  GroupMode mode = GroupMode::local;
  uint32_t world = 1, rank = 0;
  uint32_t enqueued = 0;                     // iterations enqueued since etxb_group_begin: the next ordinal
  uint32_t split_lane = 0xffffffffu;         // the lane reserved for camera-split iterations (etxb_group_reserve_split_lane), or none
  uint32_t split_part = 0, split_parts = 0;  // the (part, parts) that lane's film is made of; 0 parts = not used yet
  std::vector<std::deque<WorkItem>> queues;  // one per lane
  std::vector<uint32_t> lane_queue;
};

struct etxb_group {
  std::vector<etxb_ctx*> lanes;
  std::vector<std::thread> workers;
  std::mutex m;
  std::condition_variable cv_work, cv_idle;
  uint32_t first_iteration = 0, taken = 0;  // the k-th iteration handed out renders index first + k
  uint32_t in_flight = 0;
  WorkPlan plan;
  bool quit = false;
  int error = ETXB_OK;
  std::string error_text;
  std::chrono::steady_clock::time_point busy_since;
  double busy_seconds = 0.0;   // wall time with at least one iteration queued or in flight
  double last_iteration_seconds = 0.0;
  DevBuf<float4> combined;
  int device = 0;
  ncclComm_t reduce_comm = nullptr;  // the frame reduce has its own communicator: the lanes' ones are busy with iterations in flight
  cudaStream_t stream = nullptr;
  DevBuf<float4> combined_light, reduced;
};

namespace {

// NCCL is bound at run time: a single-GPU host needs no libnccl, and a torch host that already loaded its bundled libnccl.so.2 shares it.
struct NcclApi {
  void* handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Reduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
};
NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return;
    bool ok = true;
    auto bind = [&](auto& fn, const char* name) {
      fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, name));
      ok = ok && (fn != nullptr);
    };
    bind(api.GetUniqueId, "ncclGetUniqueId");
    bind(api.CommInitRank, "ncclCommInitRank");
    bind(api.CommDestroy, "ncclCommDestroy");
    bind(api.AllReduce, "ncclAllReduce");
    bind(api.AllGather, "ncclAllGather");
    bind(api.Reduce, "ncclReduce");
    bind(api.Broadcast, "ncclBroadcast");
    bind(api.GroupStart, "ncclGroupStart");
    bind(api.GroupEnd, "ncclGroupEnd");
    bind(api.GetErrorString, "ncclGetErrorString");
    if (ok) api.handle = h;
  });
  return api.handle ? &api : nullptr;
}

int fail(etxb_ctx* ctx, int code, const char* fmt, ...) {
  char buf[1024];
  va_list args;
  va_start(args, fmt);
  vsnprintf(buf, sizeof(buf), fmt, args);
  va_end(args);
  if (ctx) ctx->error = buf;
  return code;
}

#define CUDA_OK(ctx, call)                                                                                   \
  do {                                                                                                       \
    cudaError_t err__ = (call);                                                                              \
    if (err__ != cudaSuccess) {                                                                              \
      return fail(ctx, (err__ == cudaErrorMemoryAllocation) ? ETXB_ERR_OUT_OF_MEMORY : ETXB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(err__), \
        __FILE__, __LINE__);                                                                                 \
    }                                                                                                        \
  } while (0)

#define NCCL_OK(ctx, call)                                                                                                 \
  do {                                                                                                                     \
    ncclResult_t res__ = (call);                                                                                           \
    if (res__ != ncclSuccess) return fail(ctx, ETXB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, nccl_api()->GetErrorString(res__), __FILE__, __LINE__); \
  } while (0)

// Joins rank `rank` of a `world`-rank communicator on the current device; `id` holds the ncclUniqueId rank 0 made.  Collective.
int comm_init_rank(etxb_ctx* ctx, ncclComm_t* comm, uint32_t world, uint32_t rank, const void* id) {
  NcclApi* n = nccl_api();
  if (!n) return fail(ctx, ETXB_ERR_NOT_READY, "libnccl.so.2 could not be loaded");
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  NCCL_OK(ctx, n->CommInitRank(comm, int(world), uid, int(rank)));
  return ETXB_OK;
}

// A stream at the device's highest priority, so that its few blocks do not queue behind the lanes' large kernels
cudaError_t create_priority_stream(cudaStream_t* stream) {
  int prio_low = 0, prio_high = 0;
  if (cudaError_t err = cudaDeviceGetStreamPriorityRange(&prio_low, &prio_high)) return err;
  return cudaStreamCreateWithPriority(stream, cudaStreamNonBlocking, prio_high);
}

template <class T>
int upload(etxb_ctx* ctx, DevBuf<T>& buf, const T* host, size_t n) {
  CUDA_OK(ctx, buf.alloc(std::max<size_t>(n, 1)));
  if (n) CUDA_OK(ctx, cudaMemcpyAsync(buf.ptr, host, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  return ETXB_OK;
}

cudaEvent_t next_event(etxb_ctx* ctx) {
  if (ctx->event_cursor == ctx->event_pool.size()) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    ctx->event_pool.push_back(e);
  }
  return ctx->event_pool[ctx->event_cursor++];
}

struct LaunchTimer {
  etxb_ctx* ctx;
  TimedLaunch t;
  LaunchTimer(etxb_ctx* c, uint32_t kernel) : ctx(c) {
    ctx->kernel_launches += 1;
    ctx->kernel_count[kernel] += 1;
    if (ctx->profile) {
      t.kernel = kernel;
      t.start = next_event(ctx);
      t.stop = next_event(ctx);
      cudaEventRecord(t.start, ctx->stream);
    }
  }
  ~LaunchTimer() {
    if (ctx->profile) {
      cudaEventRecord(t.stop, ctx->stream);
      ctx->timed.push_back(t);
    }
  }
};

bool material_class_supported_host(uint32_t cls) { return cls <= ETXB_MAT_VOID; }

// A Distribution over `size` items holds size + 1 entries (DistributionBuilder allocates the closing {0, 0, 1} entry, distribution_builder.hxx:8-14,
// 52) while `values.count` says `size` (the reference's loader) or size + 1 (hosts that count the closing entry): both are accepted, and the
// device always gets the size + 1 entries.
bool distribution_covers(uint64_t count, uint64_t size) { return (count == size) || (count == size + 1u); }

uint32_t next_pow2(uint64_t v) {
  // next_power_of_two (math.hxx:1001-1010)
  v--;
  v |= v >> 1;
  v |= v >> 2;
  v |= v >> 4;
  v |= v >> 8;
  v |= v >> 16;
  v |= v >> 32;
  v++;
  return uint32_t(v);
}

// Film::dimensions() (film.cxx:373-379)
uint32_t film_dims_x(const etxb_ctx* ctx) { return (ctx->width + ctx->pixel_size - 1u) / ctx->pixel_size; }
uint32_t film_dims_y(const etxb_ctx* ctx) { return (ctx->height + ctx->pixel_size - 1u) / ctx->pixel_size; }

LaunchParams make_params(etxb_ctx* ctx) {
  LaunchParams p = {};
  p.scene = ctx->dscene;
  p.paths = {ctx->ray_o.ptr, ctx->ray_d.ptr, ctx->thr.ptr, ctx->mis.ptr, ctx->misc.ptr, ctx->hit.ptr, ctx->gathered.ptr, ctx->merged.ptr, ctx->wavelength.ptr,
    ctx->lv_count.ptr, ctx->bs_weight_pdf.ptr, ctx->bs_wo_eta.ptr, ctx->bs_props.ptr, ctx->merge_key.ptr, ctx->conn_rec.ptr};
  p.film = {ctx->film_camera.ptr, ctx->film_light.ptr, ctx->film_light_iteration.ptr, ctx->width, ctx->height, ctx->pixel_size, film_dims_x(ctx), film_dims_y(ctx)};
  p.grid = ctx->grid;
  p.lv_tmp = ctx->lv_tmp.ptr;
  p.lv_final = ctx->lv_final.ptr;
  p.lv_tmp_count = ctx->lv_tmp_count.ptr;
  p.lv_capacity = ctx->lv_capacity;
  p.lp_offset = ctx->lp_offset.ptr;
  p.overflow = ctx->overflow.ptr;
  p.counters = ctx->counters.ptr;
  p.sampler_end_light = ctx->sampler_end_light.ptr;
  p.sampler_end_camera = ctx->sampler_end_camera.ptr;
  p.camera_value = ctx->camera_value.ptr;
  p.path_count = ctx->launch_count;
  p.rank = ctx->rank;
  p.world = ctx->world;
  p.light_world = ctx->light_full ? 1u : ctx->world;
  p.camera_sample_index = ctx->completed;
  p.conn_list = ctx->conn_list.ptr;
  p.conn_count = ctx->conn_count.ptr;
  p.conn_capacity = ctx->lv_capacity;
  p.conn_key = (ctx->has_stochastic_merge && ctx->conn_list_sorted.count) ? ctx->keys_in.ptr : nullptr;  // keys_in / vals_in are free after the grid build
  p.paths.shadow_span = ctx->shadow_span.ptr;
  p.shadow_p0 = ctx->shadow_p0.ptr;
  p.shadow_p1 = ctx->shadow_p1.ptr;
  p.shadow_value = ctx->shadow_value.ptr;
  p.shadow_result = ctx->shadow_result.ptr;
  p.shadow_count = ctx->shadow_count.ptr;
  p.shadow_capacity = uint32_t(ctx->shadow_p0.count);
  p.shadow_stage = (ctx->dscene.deferred_shadow_rays && ctx->shadow_p0.count) ? 1u : 0u;
#if defined(ETXB_PARITY) && ETXB_PARITY
  p.shadow_atomic = 0;
#else
  p.shadow_atomic = (!p.shadow_stage && ctx->opaque_scene && ctx->plain_scene && ctx->has_stochastic_merge && ctx->shadow_p0.count) ? 1u : 0u;
#endif
  p.merge_material_major = ctx->has_stochastic_merge ? 1u : 0u;
#if defined(ETXB_PARITY) && ETXB_PARITY
  p.connect_stage = 0;
#else
  p.connect_stage = ctx->has_stochastic_merge ? 1u : 0u;
#endif
  // start_next_iteration (vcm_cpu.cxx:95-113): the radius from dimensions() * pixel_size() (wider than the film when a side is not a multiple
  // of the pixel size), eta_vcm from pixel_count()
  VcmParams& v = p.vcm;
  v.options = ctx->options.options;
  v.kernel = ctx->options.kernel;
  v.blue_noise = (ctx->options.blue_noise != 0) && ctx->dscene.has_blue_noise;
  v.iteration = ctx->iteration;
  float used_radius = ctx->options.initial_radius;
  if (used_radius == 0.0f) {
    uint32_t max_dim = std::max(film_dims_x(ctx) * ctx->pixel_size, film_dims_y(ctx) * ctx->pixel_size);
    used_radius = 5.0f * ctx->dscene.bounding_sphere_radius / float(max_dim);
  }
  float radius_scale = 1.0f / (1.0f + float(ctx->iteration) / float(ctx->options.radius_decay));
  v.current_radius = used_radius * radius_scale;
  float eta_vcm = kPi * (v.current_radius * v.current_radius) * float(ctx->launch_count);
  v.vc_weight = 1.0f / eta_vcm;
  v.vm_weight = (ctx->options.options & ETXB_VCM_ENABLE_MERGING) ? eta_vcm : 0.0f;
  v.vm_normalization = 1.0f / eta_vcm;
  return p;
}

uint32_t blocks_for(uint32_t n, uint32_t block) { return (n + block - 1u) / block; }

int read_u32(etxb_ctx* ctx, const uint32_t* dptr, uint32_t& out) {
  CUDA_OK(ctx, cudaMemcpyAsync(&out, dptr, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  return ETXB_OK;
}

// Size of the next bounce's queue.  A long queue is read back every bounce (the grids are sized by it).  In the tail of a pass the
// queue only shrinks and every kernel guards on the device-side count, so the previous size stays a valid upper bound for the launch
// grids: the host then enqueues several bounces back to back and reads the count only every kTailBatch bounces.  A tail starts below
// thresholds.tail_queue.
constexpr uint32_t kTailBatch = 4u;
int next_queue_size(etxb_ctx* ctx, const uint32_t* dptr, uint32_t& active, uint32_t& unsynced) {
  if ((active < ctx->thresholds.tail_queue) && (unsynced + 1u < kTailBatch)) {
    unsynced += 1u;
    return ETXB_OK;
  }
  unsynced = 0;
  return read_u32(ctx, dptr, active);
}

// Scenes with stochastic BSDFs: the bounce kernels spend their time in the BSDF class of the surface that was hit, and a warp that holds
// several classes runs them one after the other.  k_trace_closest leaves one key per queue slot (material index; 0xff = miss; 0x100 = slot
// past the device-side count); a stable 9-bit radix sort groups the queue, slots past the count stay at the end.  Returns the queue the
// rest of the bounce must use.  Short queues (the tail of a pass, below thresholds.sort_queue_min) are latency bound and skip it.
inline bool sorts_queue(const etxb_ctx* ctx, uint32_t active) { return ctx->has_stochastic_merge && (active >= ctx->thresholds.sort_queue_min) && ctx->queue_sorted.count; }
int sort_queue_by_material(etxb_ctx* ctx, const uint32_t* queue, uint32_t active, const uint32_t** sorted) {
  ctx->branch_counts.queue_sorts += 1;
  size_t temp_bytes = ctx->cub_temp.bytes();
  CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(ctx->cub_temp.ptr, temp_bytes, ctx->queue_keys.ptr, ctx->queue_keys_sorted.ptr, queue, ctx->queue_sorted.ptr, int(active), 0, 9,
                 ctx->stream));
  *sorted = ctx->queue_sorted.ptr;
  return ETXB_OK;
}

// closest hits of a queue, one ray per thread: the 4-wide quantised tree where the scene has one (dwide.cuh), the BVH2 otherwise
int launch_trace_closest(etxb_ctx* ctx, const LaunchParams& p, const uint32_t* queue, const uint32_t* count, uint32_t* keys, uint32_t active) {
  if (p.scene.wide_nodes != nullptr) {
    k_trace_closest_wide<<<blocks_for(active, 256), 256, 0, ctx->stream>>>(p, queue, count, keys, active);
  } else {
    k_trace_closest<<<blocks_for(active, 256), 256, 0, ctx->stream>>>(p, queue, count, keys, active);
  }
  return ETXB_OK;
}
// the bounce's shadow segments (ShadowBatch, atomic mode): traced and added to their targets
int launch_shadow_resolve(etxb_ctx* ctx, const LaunchParams& p, uint32_t active) {
  CUDA_OK(ctx, cudaMemsetAsync(ctx->trace_cursor.ptr, 0, 4, ctx->stream));
  const uint32_t blocks = std::min<uint32_t>(blocks_for(std::min<uint64_t>(uint64_t(active) * 4ull, 0x7fffffffull), kTraversalBlock), ctx->sm_count);
  if (p.scene.wide_nodes != nullptr) {
    k_shadow_resolve<true><<<blocks, kTraversalBlock, 0, ctx->stream>>>(p, ctx->trace_cursor.ptr);
  } else {
    k_shadow_resolve<false><<<blocks, kTraversalBlock, 0, ctx->stream>>>(p, ctx->trace_cursor.ptr);
  }
  return ETXB_OK;
}

// The wavefront bounce loop of a pass.  `begin(queue, count)` launches the pass's first kernel, which fills the first queue and its
// device-side count.  Every bounce traces the closest hits of the queue (timer `trace_kernel`), groups the queue by material when it is
// long enough, clears the next count and calls `bounce(q, count, next_queue, next_count, active)` for the rest: its stages read queue `q`
// and the count, and write the surviving paths to the next queue and count.  `active` is an upper bound of the count (kTailBatch), exact
// whenever active >= thresholds.tail_queue.  The first count is stored to `first_active` when it is given.
template <class Begin, class Bounce>
int run_bounces(etxb_ctx* ctx, const LaunchParams& p, uint32_t trace_kernel, Begin&& begin, Bounce&& bounce, uint32_t* first_active = nullptr) {
  uint32_t* counts = ctx->queue_counts.ptr;  // [cur] = this bounce's queue, [cur ^ 1] = the next one's
  CUDA_OK(ctx, cudaMemsetAsync(counts, 0, 8, ctx->stream));
  uint32_t* qin = ctx->queue_a.ptr;
  uint32_t* qout = ctx->queue_b.ptr;
  if (int rc = begin(qin, counts + 0)) return rc;
  uint32_t active = 0;
  if (int rc = read_u32(ctx, counts + 0, active)) return rc;
  if (first_active) *first_active = active;
  uint32_t cur = 0, unsynced = 0;
  while (active > 0) {
    const bool sorted = sorts_queue(ctx, active);
    const uint32_t* q = qin;  // the queue every stage of this bounce reads
    {
      LaunchTimer t(ctx, trace_kernel);
      if (int rc = launch_trace_closest(ctx, p, qin, counts + cur, sorted ? ctx->queue_keys.ptr : nullptr, active)) return rc;
    }
    if (sorted) {
      LaunchTimer t(ctx, K_QUEUE_SORT);
      if (int rc = sort_queue_by_material(ctx, qin, active, &q)) return rc;
    }
    CUDA_OK(ctx, cudaMemsetAsync(counts + (cur ^ 1u), 0, 4, ctx->stream));
    if (int rc = bounce(q, counts + cur, qout, counts + (cur ^ 1u), active)) return rc;
    cur ^= 1u;
    std::swap(qin, qout);
    if (int rc = next_queue_size(ctx, counts + cur, active, unsynced)) return rc;
  }
  CUDA_OK(ctx, cudaGetLastError());
  return ETXB_OK;
}

template <bool SP, bool PLAIN>
int run_light_pass(etxb_ctx* ctx) {
  LaunchParams p = make_params(ctx);
  auto begin = [&](uint32_t* queue, uint32_t* count) -> int {
    CUDA_OK(ctx, cudaMemsetAsync(ctx->lv_tmp_count.ptr, 0, 4, ctx->stream));
    LaunchTimer t(ctx, K_LIGHT_BEGIN);
    k_light_begin<SP><<<blocks_for(ctx->launch_count, 128), 128, 0, ctx->stream>>>(p, queue, count);
    return ETXB_OK;
  };
  auto bounce = [&](const uint32_t* q, const uint32_t* count, uint32_t* next_queue, uint32_t* next_count, uint32_t active) -> int {
    if (p.shadow_atomic) CUDA_OK(ctx, cudaMemsetAsync(ctx->shadow_count.ptr, 0, 8, ctx->stream));
    {
      LaunchTimer t(ctx, K_LIGHT_BOUNCE);
      k_light_bounce<SP, PLAIN><<<blocks_for(active, 128), 128, 0, ctx->stream>>>(p, q, count, next_queue, next_count);
    }
    if (p.shadow_atomic) {
      // the light-to-camera connections of this bounce: segments -> splats (light image)
      LaunchTimer t(ctx, K_SHADOW_TRACE);
      if (int rc = launch_shadow_resolve(ctx, p, active)) return rc;
    }
    return ETXB_OK;
  };
  if (int rc = run_bounces(ctx, p, K_TRACE_LIGHT, begin, bounce)) return rc;

  // path-major vertex pool: offsets = exclusive scan of per-path counts (VCMLightPath::index)
  uint32_t total = 0;
  if (int rc = read_u32(ctx, ctx->lv_tmp_count.ptr, total)) return rc;
  uint32_t ovf = 0;
  if (int rc = read_u32(ctx, ctx->overflow.ptr, ovf)) return rc;
  ctx->overflow_flag |= ovf;
  total = std::min(total, ctx->lv_capacity);
  {
    LaunchTimer t(ctx, K_LV_SCAN);
    size_t temp_bytes = ctx->cub_temp.bytes();
    CUDA_OK(ctx, cub::DeviceScan::ExclusiveSum(ctx->cub_temp.ptr, temp_bytes, ctx->lv_count.ptr, ctx->lp_offset.ptr, int(ctx->launch_count), ctx->stream));
  }
  if (total > 0) {
    LaunchTimer t(ctx, K_LV_REORDER);
    k_lv_reorder<<<blocks_for(total, 256), 256, 0, ctx->stream>>>(p, total);
  }
  ctx->last_light_vertices = total;
  CUDA_OK(ctx, cudaGetLastError());
  return ETXB_OK;
}

template <bool SP>
int run_grid_build(etxb_ctx* ctx, const LightVertexRec* records, uint32_t count) {
  ctx->grid = {};
  LaunchParams p = make_params(ctx);
  {
    // complete_light_vertices -> Film::commit_light_iteration(iteration) (vcm_cpu.cxx:209-211); with pixel tiles over several GPUs
    // comm_exchange has all-reduced the per-iteration light image across ranks before this call
    LaunchTimer t(ctx, K_FILM_COMMIT);
    // the running mean counts the iterations THIS context has accumulated since etxb_begin (= the absolute index in the reference's flow,
    // which always starts at 0; after etxb_begin(ctx, k != 0) or with interleaved iterations the absolute index would scale the first
    // commit by 1/(k+1) against a cleared film)
    k_film_commit_light<<<blocks_for(ctx->path_count, 256), 256, 0, ctx->stream>>>(p.film, ctx->completed);
    if (ctx->pixel_size != 1u) CUDA_OK(ctx, cudaMemsetAsync(ctx->film_light_iteration.ptr, 0, size_t(ctx->launch_count) * 16u, ctx->stream));
  }
  bool merging = (ctx->options.options & ETXB_VCM_ENABLE_MERGING) && (ctx->options.options & ETXB_VCM_MERGE_VERTICES);
  if (!merging || (count == 0)) return ETXB_OK;
  p.lv_final = const_cast<LightVertexRec*>(records);
  float radius = p.vcm.current_radius;
  uint32_t init[6];
  for (int k = 0; k < 3; ++k) {
    init[k] = 0xffffffffu;
    init[3 + k] = 0u;
  }
  CUDA_OK(ctx, cudaMemcpyAsync(ctx->grid_bbox.ptr, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
  {
    LaunchTimer t(ctx, K_GRID_BBOX);
    k_grid_bbox<<<std::min<uint32_t>(blocks_for(count, 256), ctx->sm_count * 8u), 256, 0, ctx->stream>>>(records, count, ctx->grid_bbox.ptr);
  }
  uint32_t table_size = next_pow2(count);
  uint32_t mask = table_size - 1u;
  float cell_size = 2.0f * radius;
  {
    LaunchTimer t(ctx, K_GRID_KEYS);
    k_grid_keys<<<blocks_for(count, 256), 256, 0, ctx->stream>>>(records, count, ctx->grid_bbox.ptr, cell_size, mask, ctx->keys_in.ptr, ctx->vals_in.ptr);
  }
  {
    LaunchTimer t(ctx, K_GRID_SORT);
    size_t temp_bytes = ctx->cub_temp.bytes();
    int end_bit = 1;
    while ((1ull << end_bit) < table_size) end_bit++;
    if (ctx->dscene.medium_count) end_bit = 32;  // medium vertices carry the key 0xffffffff and must sort behind every cell
    CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(ctx->cub_temp.ptr, temp_bytes, ctx->keys_in.ptr, ctx->keys_out.ptr, ctx->vals_in.ptr, ctx->vals_out.ptr, int(count), 0,
                   end_bit, ctx->stream));
  }
  CUDA_OK(ctx, cudaMemsetAsync(ctx->cell_range.ptr, 0, size_t(table_size) * sizeof(uint2), ctx->stream));
  {
    LaunchTimer t(ctx, K_GRID_BUILD);
    k_grid_build<SP><<<blocks_for(count, 256), 256, 0, ctx->stream>>>(p, ctx->keys_out.ptr, ctx->vals_out.ptr, count, ctx->cell_range.ptr, ctx->g_pos.ptr, ctx->g_nrm.ptr,
      ctx->g_win.ptr, ctx->g_thr.ptr);
  }
  uint32_t bbox[6];
  CUDA_OK(ctx, cudaMemcpyAsync(bbox, ctx->grid_bbox.ptr, sizeof(bbox), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  GridData& g = ctx->grid;
  g.cell_range = ctx->cell_range.ptr;
  g.pos_dvcm = ctx->g_pos.ptr;
  g.nrm_dvm = ctx->g_nrm.ptr;
  g.win_len = ctx->g_win.ptr;
  g.thr_rgb = ctx->g_thr.ptr;
  g.bbox_min = {ordered_to_float(bbox[0]), ordered_to_float(bbox[1]), ordered_to_float(bbox[2])};
  g.bbox_max = {ordered_to_float(bbox[3]), ordered_to_float(bbox[4]), ordered_to_float(bbox[5])};
  g.hash_table_mask = mask;
  g.photon_count = count;
  g.cell_size = cell_size;
  g.radius_squared = radius * radius;
  g.inv_radius_squared = (g.radius_squared > 0.0f) ? 1.0f / g.radius_squared : 0.0f;
  CUDA_OK(ctx, cudaGetLastError());
  return ETXB_OK;
}

// The photon gather of a bounce over queue `q` (`active` slots, device-side count at `count`); merge_key holds one key per slot.  The parity
// build runs the serial, reference-ordered gather; the product build the warp-cooperative Lambert gather and, in scenes with stochastic
// BSDFs, the closure gather.  `active` must be the exact count when the queue is sorted here: a stale slot past the count would be sorted in.
template <bool SP>
int launch_merge(etxb_ctx* ctx, const LaunchParams& p, const uint32_t* q, const uint32_t* count, uint32_t active) {
#if defined(ETXB_PARITY) && ETXB_PARITY
  LaunchTimer t(ctx, K_CAMERA_MERGE_GENERIC);
  k_camera_merge_serial<SP><<<blocks_for(active, 128), 128, 0, ctx->stream>>>(p, q, count);
  ctx->branch_counts.merge_launches[0] += 1;
#else
  if (!ctx->grid.photon_count) return ETXB_OK;
  const etxb_debug_thresholds& th = ctx->thresholds;
  const uint32_t* ids = q;
  const uint32_t* keys = ctx->merge_key.ptr;
  if (active >= th.merge_sort_min_queries) {
    // queries sorted by the Morton code of their base cell: neighbours in the queue read the same photon cells.  A short queue
    // (the tail of the pass) is latency bound, not bandwidth bound: it goes in queue order and saves the sort launches.
    LaunchTimer t(ctx, K_CAMERA_MERGE_SORT);
    size_t temp_bytes = ctx->cub_temp.bytes();
    CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(ctx->cub_temp.ptr, temp_bytes, ctx->merge_key.ptr, ctx->keys_out.ptr, q, ctx->vals_out.ptr, int(active), 0, 32,
                   ctx->stream));
    ids = ctx->vals_out.ptr;
    keys = ctx->keys_out.ptr;
    ctx->branch_counts.merge_sorts += 1;
  }
  // queries per warp: 32 while that still fills the machine, fewer for short queues (a warp serialises its queries)
  uint32_t qpw = 32u;
  while ((qpw > 1u) && (uint64_t(active / qpw) < uint64_t(th.merge_min_warps_per_sm) * ctx->sm_count)) qpw >>= 1;
  if (th.merge_qpw) qpw = th.merge_qpw;
  const uint32_t merge_blocks = blocks_for(blocks_for(active, qpw), kMergeWarpsPerBlock);
  {
    LaunchTimer t(ctx, K_CAMERA_MERGE);
    k_camera_merge_coop<SP><<<merge_blocks, kMergeWarpsPerBlock * 32, 0, ctx->stream>>>(p, ids, keys, count, qpw);
  }
  if (ctx->has_stochastic_merge) {
    LaunchTimer t(ctx, K_CAMERA_MERGE_GENERIC);
    const uint32_t closure_blocks = blocks_for(blocks_for(active, qpw), kClosureWarpsPerBlock);
    k_camera_merge_closure<SP><<<closure_blocks, kClosureWarpsPerBlock * 32, 0, ctx->stream>>>(p, ids, keys, count, qpw);
  }
  ctx->branch_counts.merge_launches[__builtin_ctz(qpw)] += 1;
#endif
  return ETXB_OK;
}

int film_ensure_adaptive(etxb_ctx* ctx);

template <bool SP, bool PLAIN>
int run_camera_pass(etxb_ctx* ctx) {
  LaunchParams p = make_params(ctx);
  const bool merging = (ctx->options.options & ETXB_VCM_ENABLE_MERGING) && (ctx->options.options & ETXB_VCM_MERGE_VERTICES);
  auto begin = [&](uint32_t* queue, uint32_t* count) -> int {
    LaunchTimer t(ctx, K_CAMERA_BEGIN);
    k_camera_begin<SP><<<blocks_for(ctx->launch_count, 128), 128, 0, ctx->stream>>>(p, queue, count);
    return ETXB_OK;
  };
  auto bounce = [&](const uint32_t* q, const uint32_t* count, uint32_t* next_queue, uint32_t* next_count, uint32_t active) -> int {
    if (p.connect_stage) CUDA_OK(ctx, cudaMemsetAsync(ctx->conn_count.ptr, 0, 4, ctx->stream));
    if (p.shadow_stage || p.shadow_atomic) CUDA_OK(ctx, cudaMemsetAsync(ctx->shadow_count.ptr, 0, 8, ctx->stream));
    {
      LaunchTimer t(ctx, K_CAMERA_SHADE);
      k_camera_shade<SP, PLAIN><<<blocks_for(active, 128), 128, 0, ctx->stream>>>(p, q, count);
    }
    if (p.shadow_stage && (ctx->options.options & ETXB_VCM_CONNECT_VERTICES)) {
      // one thread per (camera vertex, light vertex) pair of the bounce, grid-stride over the reserved shadow slots (count on the device)
      LaunchTimer t(ctx, K_CAMERA_CONNECT);
      uint32_t blocks = std::min<uint32_t>(ctx->sm_count * 16u, blocks_for(std::min<uint64_t>(uint64_t(active) * 8ull, 0x7fffffffull), 128));
      k_camera_connect_deferred<SP><<<blocks, 128, 0, ctx->stream>>>(p);
    }
    if (p.shadow_stage) {
      // persistent warps over the bounce's deferred shadow rays (the number of rays stays on the device)
      LaunchTimer t(ctx, K_SHADOW_TRACE);
      uint32_t blocks = std::min<uint32_t>(ctx->sm_count * 8u, blocks_for(std::min<uint64_t>(uint64_t(active) * 32ull, 0x7fffffffull), 256));
      k_shadow_trace<<<blocks, 256, 0, ctx->stream>>>(p);
    }
#if !(defined(ETXB_PARITY) && ETXB_PARITY)  // make_params: the parity build has no connection stage
    if (p.connect_stage && (ctx->options.options & ETXB_VCM_CONNECT_VERTICES)) {
      if (active < ctx->thresholds.tail_queue) {
        // tail of the pass: the pair count stays on the device (k_camera_connect is grid-stride), no host round trip per bounce
        LaunchTimer t(ctx, K_CAMERA_CONNECT);
        const uint32_t blocks = std::min<uint32_t>(ctx->sm_count * 4u, blocks_for(active * 4u, 128));
        k_camera_connect<SP, PLAIN><<<blocks, 128, 0, ctx->stream>>>(p, ctx->conn_list.ptr);
      } else {
        uint32_t pending = 0;
        if (int rc = read_u32(ctx, ctx->conn_count.ptr, pending)) return rc;
        pending = std::min(pending, ctx->lv_capacity);
        if (pending) {
          const uint2* list = ctx->conn_list.ptr;
          if (p.conn_key && (pending >= ctx->thresholds.sort_queue_min)) {
            // connections grouped by (camera vertex material, light vertex material): one pair of BSDF classes per warp
            LaunchTimer t(ctx, K_QUEUE_SORT);
            size_t temp_bytes = ctx->cub_temp.bytes();
            CUDA_OK(ctx, cub::DeviceRadixSort::SortPairs(ctx->cub_temp.ptr, temp_bytes, ctx->keys_in.ptr, ctx->vals_in.ptr, reinterpret_cast<const unsigned long long*>(ctx->conn_list.ptr),
                           reinterpret_cast<unsigned long long*>(ctx->conn_list_sorted.ptr), int(pending), 0, 16, ctx->stream));
            list = ctx->conn_list_sorted.ptr;
            ctx->branch_counts.pair_sorts += 1;
          }
          ctx->branch_counts.connect_launches += 1;
          LaunchTimer t(ctx, K_CAMERA_CONNECT);
          k_camera_connect<SP, PLAIN><<<blocks_for(pending, 128), 128, 0, ctx->stream>>>(p, list);
        }
      }
    }
#endif
    if (p.shadow_atomic) {
      // emitter-sample and vertex-connection segments of this bounce: traced, the unoccluded ones added to their paths' gathered sums
      LaunchTimer t(ctx, K_SHADOW_TRACE);
      if (int rc = launch_shadow_resolve(ctx, p, active)) return rc;
    }
    if (merging) {
      if (int rc = launch_merge<SP>(ctx, p, q, count, active)) return rc;
    }
    LaunchTimer t(ctx, K_CAMERA_CONTINUE);
    k_camera_continue<SP><<<blocks_for(active, 128), 128, 0, ctx->stream>>>(p, q, count, next_queue, next_count);
    return ETXB_OK;
  };
  if (int rc = run_bounces(ctx, p, K_TRACE_CAMERA, begin, bounce)) return rc;
  if (ctx->pixel_size != 1u) {
    LaunchTimer t(ctx, K_CAMERA_CONTINUE);
    k_film_fill_blocks<false><<<blocks_for(ctx->path_count, 256), 256, 0, ctx->stream>>>(p, PtFilm{}, ctx->iteration);
  }
  if ((p.camera_sample_index % 2u) == 0u) {
    // CameraAdaptive, the even-sample mean the denoiser's variance estimate reads (an odd sample leaves it as it is)
    if (int rc = film_ensure_adaptive(ctx)) return rc;
    LaunchTimer t(ctx, K_FILM_ADAPTIVE);
    k_film_adaptive_vcm<<<blocks_for(ctx->path_count, 256), 256, 0, ctx->stream>>>(p, ctx->film_adaptive.ptr);
  }
  CUDA_OK(ctx, cudaGetLastError());
  return ETXB_OK;
}

// Pixel-tile sharding (SURVEY 8(e), north star): between the light pass and the grid build of an iteration the ranks exchange what is global —
//   (a) the light-tracing splats land on ANY pixel (vcm_cpu.cxx:147-154): all-reduce(sum) of the per-iteration light image, after which every
//       rank commits the same running mean (film.cxx:332-343);
//   (b) merging queries the photon map of ALL light paths (vcm_cpu.cxx:219-221): all-gather of the path-major vertex records (96 B each, block
//       sizes differ per rank: counts first, then one broadcast per owner inside a group call = an uneven all-gather), into the allocation-order
//       pool, which is free once the path-major pool exists; every rank then builds the same grid.
// Camera tiles are disjoint: they meet only when a frame is wanted (etxb_comm_reduce_film).  With merging on, `records` / `count` are set to
// the gathered pool; otherwise they are left as they are.
int comm_exchange(etxb_ctx* ctx, const LightVertexRec** records, uint32_t* count) {
  NcclApi* n = nccl_api();
  // the collectives run on the context's high-priority stream, fenced against its work stream by events on both sides
  cudaStream_t cs = ctx->comm_stream;
  auto fence_out = [&]() -> cudaError_t {
    cudaError_t e = cudaEventRecord(ctx->comm_ev_out, cs);
    return (e == cudaSuccess) ? cudaStreamWaitEvent(ctx->stream, ctx->comm_ev_out, 0) : e;
  };
  {
    LaunchTimer t(ctx, K_COMM_LIGHT_IMAGE);
    CUDA_OK(ctx, cudaEventRecord(ctx->comm_ev_in, ctx->stream));
    CUDA_OK(ctx, cudaStreamWaitEvent(cs, ctx->comm_ev_in, 0));
    NCCL_OK(ctx, n->AllReduce(ctx->film_light_iteration.ptr, ctx->film_light_iteration.ptr, size_t(ctx->path_count) * 4u, ncclFloat, ncclSum, ctx->comm, cs));
    CUDA_OK(ctx, fence_out());
  }
  const bool merging = (ctx->options.options & ETXB_VCM_ENABLE_MERGING) && (ctx->options.options & ETXB_VCM_MERGE_VERTICES);
  if (!merging) return ETXB_OK;
  const uint32_t world = ctx->world, rank = ctx->rank;
  std::vector<uint32_t> counts(world, 0u);
  {
    LaunchTimer t(ctx, K_COMM_PHOTONS);
    uint32_t mine = ctx->last_light_vertices;
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->comm_counts.ptr + rank, &mine, 4, cudaMemcpyHostToDevice, cs));
    NCCL_OK(ctx, n->AllGather(ctx->comm_counts.ptr + rank, ctx->comm_counts.ptr, 1, ncclUint32, ctx->comm, cs));
    CUDA_OK(ctx, cudaMemcpyAsync(counts.data(), ctx->comm_counts.ptr, size_t(world) * 4u, cudaMemcpyDeviceToHost, cs));
    CUDA_OK(ctx, cudaStreamSynchronize(cs));
    uint64_t total = 0;
    std::vector<uint64_t> offsets(world, 0u);
    for (uint32_t r = 0; r < world; ++r) {
      offsets[r] = total;
      total += counts[r];
    }
    if (total > ctx->lv_capacity) return fail(ctx, ETXB_ERR_OVERFLOW, "gathered photon count %llu exceeds the pool capacity %u", (unsigned long long)total, ctx->lv_capacity);
    constexpr size_t kRecordFloats = sizeof(LightVertexRec) / 4u;
    NCCL_OK(ctx, n->GroupStart());
    for (uint32_t r = 0; r < world; ++r) {
      if (counts[r] == 0u) continue;
      ncclResult_t res = n->Broadcast(ctx->lv_final.ptr, ctx->lv_tmp.ptr + offsets[r], size_t(counts[r]) * kRecordFloats, ncclFloat, int(r), ctx->comm, cs);
      if (res != ncclSuccess) {
        n->GroupEnd();
        return fail(ctx, ETXB_ERR_CUDA, "ncclBroadcast failed: %s", n->GetErrorString(res));
      }
    }
    NCCL_OK(ctx, n->GroupEnd());
    CUDA_OK(ctx, fence_out());
    *records = ctx->lv_tmp.ptr;
    *count = uint32_t(total);
  }
  return ETXB_OK;
}

void resolve_timers(etxb_ctx* ctx) {
  for (auto& t : ctx->timed) {
    float ms = 0.0f;
    if (cudaEventElapsedTime(&ms, t.start, t.stop) == cudaSuccess) ctx->kernel_ms[t.kernel] += ms;
  }
  ctx->timed.clear();
  ctx->event_cursor = 0;
}

int finish_iteration(etxb_ctx* ctx) {
  CUDA_OK(ctx, cudaEventRecord(ctx->ev_iter_stop, ctx->stream));
  CUDA_OK(ctx, cudaEventSynchronize(ctx->ev_iter_stop));
  float ms = 0.0f;
  CUDA_OK(ctx, cudaEventElapsedTime(&ms, ctx->ev_iter_start, ctx->ev_iter_stop));
  ctx->last_iteration_time = double(ms) * 1e-3;
  ctx->total_time += ctx->last_iteration_time;
  resolve_timers(ctx);
  ctx->completed += 1;
  if (!ctx->external_iteration) ctx->iteration += 1;
  return ETXB_OK;
}

// ---- unidirectional path tracer (SURVEY 8(f) N3) -----------------------------------------------------------------------------------------
// CameraAdaptive (film.cxx:173-230): written by both integrators, allocated (as zeros) with the first pass that writes it at this film size
int film_ensure_adaptive(etxb_ctx* ctx) {
  const size_t n = ctx->path_count;
  if (ctx->film_adaptive.count == n) return ETXB_OK;
  CUDA_OK(ctx, ctx->film_adaptive.alloc(n));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->film_adaptive.ptr, 0, n * 16, ctx->stream));
  return ETXB_OK;
}

// The film layers and the per-pixel history only CPUPathTracing touches (film.cxx:14-40, 104-121), allocated with the first run.
int pt_ensure_film(etxb_ctx* ctx) {
  const size_t n = ctx->path_count;
  if (ctx->film_normals.count == n) return ETXB_OK;
  DevBuf<float4>* f4[] = {&ctx->film_normals, &ctx->film_albedo};
  for (auto* b : f4) {
    CUDA_OK(ctx, b->alloc(n));
    CUDA_OK(ctx, cudaMemsetAsync(b->ptr, 0, n * 16, ctx->stream));
  }
  if (int rc = film_ensure_adaptive(ctx)) return rc;
  CUDA_OK(ctx, ctx->pt_info.alloc(n));
  CUDA_OK(ctx, ctx->pt_error.alloc(n));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->pt_info.ptr, 0, n * 4, ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->pt_error.ptr, 0, n * 4, ctx->stream));
  return ETXB_OK;
}

PtFilm make_pt_film(etxb_ctx* ctx) { return {ctx->film_normals.ptr, ctx->film_albedo.ptr, ctx->film_adaptive.ptr, ctx->pt_info.ptr, ctx->pt_error.ptr}; }

// The buffers one rank's noise estimate reads and writes: its film, its history, the mask (+ kNoiseStats) and its place in the tile rule
struct NoiseView {
  FilmBuffers film;
  PtFilm pf;
  uint32_t* mask;
  uint32_t rank, world;
};

uint32_t noise_mask_words(uint32_t width, uint32_t height) { return height * noise_mask_words_per_row(width); }

int noise_level_pass(etxb_ctx* ctx, const NoiseView& v, float threshold) {
  const uint32_t words = noise_mask_words(v.film.width, v.film.height);
  CUDA_OK(ctx, cudaMemsetAsync(v.mask + words, 0, kNoiseStats * 4u, ctx->stream));
  LaunchTimer t(ctx, K_FILM_NOISE);
  k_film_noise_level<<<blocks_for(words * 32u, 256), 256, 0, ctx->stream>>>(v.film, v.pf, threshold, v.rank, v.world, v.mask, v.mask + words);
  return ETXB_OK;
}

int noise_dilate_pass(etxb_ctx* ctx, const NoiseView& v) {
  LaunchTimer t(ctx, K_FILM_NOISE);
  k_film_noise_dilate<<<blocks_for(noise_mask_words(v.film.width, v.film.height) * 32u, 256), 256, 0, ctx->stream>>>(v.film.width, v.film.height, v.rank, v.world,
                                                                                                                         v.mask, v.pf.info);
  return ETXB_OK;
}

// The path tracer's only collective, on the context's high-priority stream fenced by events like comm_exchange: with `mask`, the active mask
// with the converged count and pixels_processed (uint32 sums: the words of different ranks are disjoint) and the error sum (float); without,
// pixels_processed alone.
int comm_noise_exchange(etxb_ctx* ctx, uint32_t words, bool mask) {
  NcclApi* n = nccl_api();
  cudaStream_t cs = ctx->comm_stream;
  uint32_t* m = ctx->pt_mask.ptr;
  LaunchTimer t(ctx, mask ? K_COMM_PT_MASK : K_COMM_PT_COUNT);
  CUDA_OK(ctx, cudaEventRecord(ctx->comm_ev_in, ctx->stream));
  CUDA_OK(ctx, cudaStreamWaitEvent(cs, ctx->comm_ev_in, 0));
  if (mask) {
    NCCL_OK(ctx, n->GroupStart());
    ncclResult_t res = n->AllReduce(m, m, size_t(words) + kNoiseStatProcessed + 1u, ncclUint32, ncclSum, ctx->comm, cs);
    if (res == ncclSuccess) res = n->AllReduce(m + words + kNoiseStatError, m + words + kNoiseStatError, 1, ncclFloat, ncclSum, ctx->comm, cs);
    ncclResult_t end = n->GroupEnd();
    NCCL_OK(ctx, (res != ncclSuccess) ? res : end);
  } else {
    NCCL_OK(ctx, n->AllReduce(m + words + kNoiseStatProcessed, m + words + kNoiseStatProcessed, 1, ncclUint32, ncclSum, ctx->comm, cs));
  }
  CUDA_OK(ctx, cudaEventRecord(ctx->comm_ev_out, cs));
  CUDA_OK(ctx, cudaStreamWaitEvent(ctx->stream, ctx->comm_ev_out, 0));
  return ETXB_OK;
}

// Film::estimate_noise_levels (film.cxx:233-330) after iteration `sample_index`, on this context's pixels.  On a context with a communicator this
// is also where the ranks agree on what update() reads: every iteration all-reduces pixels_processed, one with an estimate the mask and the
// stats as well.  Which collectives a rank issues thus depends on the iteration index, the noise threshold and Scene::samples alone.
constexpr uint32_t kFilmMinSamples = 32u;
int pt_estimate_noise_levels(etxb_ctx* ctx, uint32_t sample_index) {
  const float threshold = ctx->noise_threshold;
  const bool estimate = (threshold != 0.0f) && (sample_index >= kFilmMinSamples) && ((sample_index % 2u) == 0u);
  const bool comm = ctx->comm != nullptr;
  if (!estimate && !comm) return ETXB_OK;
  const uint32_t words = noise_mask_words(ctx->width, ctx->height);
  if (ctx->pt_mask.count != size_t(words) + kNoiseStats) CUDA_OK(ctx, ctx->pt_mask.alloc(size_t(words) + kNoiseStats));
  uint32_t* stats = ctx->pt_mask.ptr + words;
  const NoiseView v = {{ctx->film_camera.ptr, ctx->film_light.ptr, ctx->film_light_iteration.ptr, ctx->width, ctx->height}, make_pt_film(ctx), ctx->pt_mask.ptr,
                       ctx->rank, ctx->world};
  if (estimate) {
    if (int rc = noise_level_pass(ctx, v, threshold)) return rc;
  }
  if (comm) {
    const uint32_t processed = ctx->pt_pixels_processed;
    CUDA_OK(ctx, cudaMemcpyAsync(stats + kNoiseStatProcessed, &processed, 4, cudaMemcpyHostToDevice, ctx->stream));
    if (int rc = comm_noise_exchange(ctx, words, estimate)) return rc;
  }
  if (estimate) {
    if (int rc = noise_dilate_pass(ctx, v)) return rc;
  }
  uint32_t host[kNoiseStats] = {};
  CUDA_OK(ctx, cudaMemcpyAsync(host, stats, sizeof(host), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  if (comm) ctx->pt_pixels_processed = host[kNoiseStatProcessed];
  if (estimate) {
    float total = 0.0f;
    memcpy(&total, &host[kNoiseStatError], 4);
    ctx->pt_active_pixels = host[kNoiseStatConverged];
    ctx->pt_noise_level = (host[kNoiseStatConverged] > 0u) ? (total / float(host[kNoiseStatConverged])) : total;
  }
  return ETXB_OK;
}

// One CPUPathTracingImpl task (path_tracing.cxx:50-83) followed by update()'s bookkeeping (:85-110): every active pixel's path, the film update,
// the noise estimate.
template <bool SP, bool PLAIN>
int run_pt_iteration(etxb_ctx* ctx) {
  CUDA_OK(ctx, cudaEventRecord(ctx->ev_iter_start, ctx->stream));
  if (int rc = pt_ensure_film(ctx)) return rc;
  LaunchParams p = make_params(ctx);
  p.connect_stage = 0;
  p.shadow_stage = 0;  // the slot-ordered deferred shadow rays belong to the VCM camera step; the path tracer uses the atomic list or traces inline
  PtParams pt = {};
  pt.nee = ctx->pt_options.nee;
  pt.direct = ctx->pt_options.direct;
  pt.mis = ctx->pt_options.mis;
  pt.blue_noise = (ctx->pt_options.blue_noise != 0u) && ctx->dscene.has_blue_noise;
  pt.iteration = ctx->iteration;
  pt.pixel_sampler_image = ctx->pixel_sampler_image;
  pt.pixel_sampler_radius = ctx->pixel_sampler_radius;
  pt.radiance_clamp = ctx->radiance_clamp;
  PtFilm pf = make_pt_film(ctx);
  auto begin = [&](uint32_t* queue, uint32_t* count) -> int {
    LaunchTimer t(ctx, K_PT_BEGIN);
    k_pt_begin<SP><<<blocks_for(ctx->launch_count, 128), 128, 0, ctx->stream>>>(p, pt, pf, queue, count);
    return ETXB_OK;
  };
  auto bounce = [&](const uint32_t* q, const uint32_t* count, uint32_t* next_queue, uint32_t* next_count, uint32_t active) -> int {
    if (p.shadow_atomic) CUDA_OK(ctx, cudaMemsetAsync(ctx->shadow_count.ptr, 0, 8, ctx->stream));
    {
      LaunchTimer t(ctx, K_PT_SHADE);
      k_pt_shade<SP, PLAIN><<<blocks_for(active, 128), 128, 0, ctx->stream>>>(p, pt, q, count, next_queue, next_count);
    }
    if (p.shadow_atomic) {
      LaunchTimer t(ctx, K_SHADOW_TRACE);
      if (int rc = launch_shadow_resolve(ctx, p, active)) return rc;
    }
    return ETXB_OK;
  };
  if (int rc = run_bounces(ctx, p, K_TRACE_CAMERA, begin, bounce, &ctx->pt_pixels_processed)) return rc;
  {
    LaunchTimer t(ctx, K_PT_ACCUMULATE);
    k_pt_accumulate<SP><<<blocks_for(ctx->launch_count, 256), 256, 0, ctx->stream>>>(p, pt, pf);
    if (ctx->pixel_size != 1u) k_film_fill_blocks<true><<<blocks_for(ctx->path_count, 256), 256, 0, ctx->stream>>>(p, pf, ctx->iteration);
  }
  if (int rc = pt_estimate_noise_levels(ctx, ctx->iteration)) return rc;
  CUDA_OK(ctx, cudaGetLastError());
  return finish_iteration(ctx);
}

// ---- scene upload / update ------------------------------------------------------------------------------------------------------------------
// etxb_upload_scene and etxb_update_scene run the same stages: validate_scene makes every check and touches nothing on the device,
// prepare_scene hashes the bulk arrays (prepare_bvh uploads a new geometry and builds its BVH2 on the device), commit_scene commits to the device.  An
// update keeps the device copies whose content hashes did not change; everything small is derived from the PODs again on every call.
struct SceneClass {
  bool stochastic = false;  // has_stochastic_merge
  bool boundaries = false, subsurface = false, deferred = false, opaque = false, plain = false;
};

struct ScenePrep {
  SceneClass cls;
  SceneHashes hashes;
  double fingerprint_seconds = 0.0, bvh_seconds = 0.0;
  uint64_t bytes_hashed = 0;
  // a new geometry's device copies and BVH2 (prepare_bvh: built once, copied into each context that commits it)
  DevBuf<DVertex> vertices;
  DevBuf<DTriangle> triangles;
  DevBuf<BvhNode> bvh_nodes;
  DevBuf<float4> bvh_tris;
  uint32_t max_depth = 0;
  bool have_bvh = false;
  DevBuf<WideNode> wide;  // the 4-wide tree collapsed from the first committing context's BVH2
  uint32_t max_stack = 0;
  bool have_wide = false;
};

double seconds_since(std::chrono::steady_clock::time_point t0) { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); }

bool image_has_table(const etxb_image& im) {
  return (im.y_distribution.values.a != nullptr) && distribution_covers(im.y_distribution.values.count, im.isize[1]) && (im.x_distributions.count == im.isize[1]);
}
size_t image_pixel_bytes(const etxb_image& im) { return size_t(im.isize[0]) * im.isize[1] * (im.format == 1u ? 16 : 4); }

int check_scene_args(etxb_ctx* ctx, uint64_t scene_bytes, uint64_t camera_bytes) {
  if (scene_bytes != sizeof(etxb_scene) || camera_bytes != sizeof(etxb_camera))
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "scene/camera size mismatch: got %llu/%llu, expected %zu/%zu", (unsigned long long)scene_bytes,
      (unsigned long long)camera_bytes, sizeof(etxb_scene), sizeof(etxb_camera));
  if (!ctx->xyz_table.ptr) return fail(ctx, ETXB_ERR_NOT_READY, "etxb_upload_color_tables must be called before etxb_upload_scene");
  return ETXB_OK;
}

// Every check of the upload but the BVH depth (prepare_bvh), and the scene-class flags.  What the device path does not cover yet fails
// loudly (no CPU fallback); every index the host builder and the kernels follow is checked: a malformed scene is an error, not an
// out-of-bounds read.
int validate_scene(etxb_ctx* ctx, const etxb_scene& s, const etxb_camera& cam, SceneClass& c) {
  if (cam.cls > 1u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "unknown camera class %u", cam.cls);
  if (cam.lens_image != ETXB_INVALID_INDEX) {
    if (cam.lens_image >= s.images.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "camera lens image index out of range");
    const auto& lens = static_cast<const etxb_image*>(s.images.a)[cam.lens_image];
    if (!distribution_covers(lens.y_distribution.values.count, lens.isize[1])) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "camera lens image has no sampling table");
  }
  const auto* mats = static_cast<const etxb_material*>(s.materials.a);
  for (uint64_t i = 0; i < s.materials.count; ++i) {
    const etxb_material& m = mats[i];
    if (!material_class_supported_host(m.cls)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "material %llu: class %u is not supported on the device yet", (unsigned long long)i, m.cls);
    if (m.diffuse_variation > 2u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: unknown diffuse_variation %u", (unsigned long long)i, m.diffuse_variation);
    if (m.subsurface.cls > 2u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: unknown subsurface class %u", (unsigned long long)i, m.subsurface.cls);
    if (m.subsurface.cls != 0) {
      if (s.subsurface_exit_material >= s.materials.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu uses subsurface scattering but scene.subsurface_exit_material is not set", (unsigned long long)i);
      if ((m.subsurface.image_index != ETXB_INVALID_INDEX) && (m.subsurface.image_index >= s.images.count))
        return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: subsurface image index out of range", (unsigned long long)i);
    }
    uint32_t imgs[] = {m.reflectance.image_index, m.scattering.image_index, m.emission.image_index, m.roughness.image_index, m.normal_image_index, m.thinfilm.thickness_image};
    for (uint32_t im : imgs)
      if ((im != ETXB_INVALID_INDEX) && (im >= s.images.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: image index %u out of range", (unsigned long long)i, im);
    if (((m.int_medium != ETXB_INVALID_INDEX) && (m.int_medium >= s.mediums.count)) || ((m.ext_medium != ETXB_INVALID_INDEX) && (m.ext_medium >= s.mediums.count)))
      return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "material %llu: medium index out of range", (unsigned long long)i);
  }
  c = {};
  for (uint64_t i = 0; i < s.materials.count; ++i) {
    const etxb_material& m = mats[i];
    bool lambert = (m.cls == ETXB_MAT_DIFFUSE) && (m.diffuse_variation == 0);
    bool smooth = (std::max(m.roughness.value[0], m.roughness.value[1]) <= 1.0e-4f) && (m.roughness.image_index == ETXB_INVALID_INDEX);
    bool always_delta = (((m.cls == ETXB_MAT_DIELECTRIC) || (m.cls == ETXB_MAT_CONDUCTOR)) && smooth) || (m.cls == ETXB_MAT_THINFILM) || (m.cls == ETXB_MAT_MIRROR) ||
                        (m.cls == ETXB_MAT_VOID);
    if (!lambert && !always_delta) c.stochastic = true;
  }
  const auto* emitters = static_cast<const etxb_emitter*>(s.emitter_instances.a);
  for (uint64_t i = 0; i < s.emitter_instances.count; ++i) {
    if (emitters[i].cls > 2u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter %llu: unknown class %u", (unsigned long long)i, emitters[i].cls);
    if (emitters[i].cls == 1u) {
      const auto& prof = static_cast<const etxb_emitter_profile*>(s.emitter_profiles.a)[emitters[i].profile];
      if (prof.emission.image_index >= s.images.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "environment emitter %llu has no image", (unsigned long long)i);
      const auto& img = static_cast<const etxb_image*>(s.images.a)[prof.emission.image_index];
      if (!distribution_covers(img.y_distribution.values.count, img.isize[1])) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "environment emitter %llu: image has no sampling table", (unsigned long long)i);
    }
  }
  // media (medium.hxx:8-47)
  const auto* meds = static_cast<const etxb_medium*>(s.mediums.a);
  for (uint64_t i = 0; i < s.mediums.count; ++i) {
    const etxb_medium& md = meds[i];
    if (md.cls == 1u) {
      size_t n = size_t(md.dimensions[0]) * md.dimensions[1] * md.dimensions[2];
      if ((n == 0) || (md.density.count != n)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium %llu: density grid does not match its dimensions", (unsigned long long)i);
    } else if (md.cls != 0u) {
      return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "medium %llu: unknown class %u", (unsigned long long)i, md.cls);
    }
  }
  for (uint64_t i = 0; i < s.materials.count; ++i) {
    if (mats[i].cls == ETXB_MAT_BOUNDARY) c.boundaries = true;
    if (mats[i].subsurface.cls != 0) c.subsurface = true;
  }
  if ((cam.medium_index != ETXB_INVALID_INDEX) && (cam.medium_index >= s.mediums.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "camera medium index out of range");
  // deferred shadow rays (ShadowBatch, dvcm.cuh) need: no alpha test that can reject, no Boundary surfaces / media (transmittance is 0 or 1),
  // no BSDF whose evaluation draws from the sampler, no subsurface exits
  c.plain = !c.boundaries && !c.subsurface && (s.mediums.count == 0) && (cam.medium_index == ETXB_INVALID_INDEX);
  bool no_alpha = true;
  const auto* all_images = static_cast<const etxb_image*>(s.images.a);
  for (uint64_t i = 0; no_alpha && (i < s.materials.count); ++i) {
    if (mats[i].opacity != 1.0f) no_alpha = false;
    uint32_t im = mats[i].scattering.image_index;
    if ((im != ETXB_INVALID_INDEX) && (all_images[im].options & kImageHasAlpha)) no_alpha = false;
  }
  c.opaque = c.plain && no_alpha;
  c.deferred = c.opaque && !c.stochastic;
  // images: pixels + flattened row/column CDFs (image.hxx:8-50)
  for (uint64_t i = 0; i < s.images.count; ++i) {
    const etxb_image& im = all_images[i];
    if ((im.format != 1u) && (im.format != 2u)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "image %llu: unknown pixel format %u", (unsigned long long)i, im.format);
    if (size_t(im.isize[0]) * im.isize[1] == 0) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "image %llu is empty", (unsigned long long)i);
    if (image_has_table(im)) {
      const auto* rows = static_cast<const etxb_distribution*>(im.x_distributions.a);
      for (uint32_t y = 0; y < im.isize[1]; ++y)
        if (!distribution_covers(rows[y].values.count, im.isize[0])) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "image %llu: row %u distribution has %llu entries", (unsigned long long)i, y, (unsigned long long)rows[y].values.count);
    }
  }
  if (s.emitter_instances.count == 0) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "scene has no emitters");
  const auto* spectra = static_cast<const etxb_spectrum*>(s.spectrums.a);
  for (uint64_t i = 0; i < s.spectrums.count; ++i) {
    const etxb_spectrum& sp = spectra[i];
    if (sp.entry_count != 441) return fail(ctx, ETXB_ERR_UNSUPPORTED, "spectrum %llu has %u entries; the loader's 441-entry 390..830 nm grid is required", (unsigned long long)i, sp.entry_count);
    for (uint32_t k = 0; k < 441; ++k)
      if (sp.entries[k].wavelength != float(390 + k)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "spectrum %llu is not on the integer 390..830 nm grid", (unsigned long long)i);
  }
  // geometry
  const auto* tris = static_cast<const etxb_triangle*>(s.triangles.a);
  for (uint64_t i = 0; i < s.triangles.count; ++i) {
    const etxb_triangle& t = tris[i];
    if ((t.i[0] >= s.vertices.count) || (t.i[1] >= s.vertices.count) || (t.i[2] >= s.vertices.count))
      return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "triangle %llu: vertex index out of range", (unsigned long long)i);
    if (t.material_index >= s.materials.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "triangle %llu: material index %u out of range", (unsigned long long)i, t.material_index);
  }
  if (s.triangle_to_emitter.count != s.triangles.count)
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "triangle_to_emitter has %llu entries for %llu triangles", (unsigned long long)s.triangle_to_emitter.count, (unsigned long long)s.triangles.count);
  const auto* t2e = static_cast<const uint32_t*>(s.triangle_to_emitter.a);
  for (uint64_t i = 0; i < s.triangle_to_emitter.count; ++i)
    if ((t2e[i] != ETXB_INVALID_INDEX) && (t2e[i] >= s.emitter_instances.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "triangle %llu: emitter index out of range", (unsigned long long)i);
  for (uint64_t i = 0; i < s.emitter_instances.count; ++i) {
    if (emitters[i].profile >= s.emitter_profiles.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter %llu: profile index out of range", (unsigned long long)i);
    if ((emitters[i].cls == 0u) && (emitters[i].triangle_index >= s.triangles.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "area emitter %llu: triangle index out of range", (unsigned long long)i);
  }
  if (!distribution_covers(s.emitters_distribution.values.count, s.emitter_instances.count))
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter distribution has %llu entries for %llu emitters", (unsigned long long)s.emitters_distribution.values.count, (unsigned long long)s.emitter_instances.count);
  if ((s.pixel_sampler_image != 0xffffffffu) && (s.pixel_sampler_image >= s.images.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "pixel sampler image out of range");
  if (size_t(cam.film_size[0]) * cam.film_size[1] == 0) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "empty film");
  return ETXB_OK;
}

// validate_scene + the content hashes of the arrays commit_scene may keep on the device: the vertices and triangles (one geometry
// hash), each image (pixels, sampling tables, scalar fields) and each density grid (values and dimensions)
int prepare_scene(etxb_ctx* ctx, const etxb_scene& s, const etxb_camera& cam, ScenePrep& p) {
  if (int rc = validate_scene(ctx, s, cam, p.cls)) return rc;
  auto t0 = std::chrono::steady_clock::now();
  SceneHashes& h = p.hashes;
  auto hash = [&p](const void* data, size_t bytes, Hash128 seed) {
    p.bytes_hashed += bytes;
    return hash128(data, bytes, seed);
  };
  h.geometry = hash(s.vertices.a, s.vertices.count * sizeof(etxb_vertex), {});
  h.geometry = hash(s.triangles.a, s.triangles.count * sizeof(etxb_triangle), h.geometry);
  h.images.assign(s.images.count, {});
  const auto* imgs = static_cast<const etxb_image*>(s.images.a);
  for (uint64_t i = 0; i < s.images.count; ++i) {
    const etxb_image& im = imgs[i];
    const bool table = image_has_table(im);
    const float fields[] = {im.fsize[0], im.fsize[1], im.offset[0], im.offset[1], im.scale[0], im.scale[1], im.normalization};
    const uint32_t ifields[] = {im.isize[0], im.isize[1], im.options, im.format, table ? 1u : 0u};
    Hash128 x = hash(fields, sizeof(fields), {});
    x = hash(ifields, sizeof(ifields), x);
    x = hash(im.pixels.a, image_pixel_bytes(im), x);
    if (table) {
      x = hash(im.y_distribution.values.a, (size_t(im.isize[1]) + 1u) * sizeof(etxb_distribution_entry), x);
      const auto* rows = static_cast<const etxb_distribution*>(im.x_distributions.a);
      for (uint32_t y = 0; y < im.isize[1]; ++y) x = hash(rows[y].values.a, (size_t(im.isize[0]) + 1u) * sizeof(etxb_distribution_entry), x);
    }
    h.images[i] = x;
  }
  h.grids.assign(s.mediums.count, {});
  const auto* meds = static_cast<const etxb_medium*>(s.mediums.a);
  for (uint64_t i = 0; i < s.mediums.count; ++i) {
    if (meds[i].cls != 1u) continue;
    h.grids[i] = hash(meds[i].dimensions, sizeof(meds[i].dimensions), {});
    h.grids[i] = hash(meds[i].density.a, meds[i].density.count * sizeof(float), h.grids[i]);
  }
  h.valid = true;
  p.fingerprint_seconds = seconds_since(t0);
  return ETXB_OK;
}

// takes ownership of a cudaMalloc'd array of n elements
template <class T>
void adopt(DevBuf<T>& buf, T* ptr, size_t n) {
  buf.release();
  buf.ptr = ptr;
  buf.count = n;
}

// a device-to-device copy into `dst`, sized as `src`
template <class T>
int copy_device(etxb_ctx* ctx, DevBuf<T>& dst, const DevBuf<T>& src) {
  CUDA_OK(ctx, dst.alloc(src.count));
  if (src.count) CUDA_OK(ctx, cudaMemcpyAsync(dst.ptr, src.ptr, src.bytes(), cudaMemcpyDeviceToDevice, ctx->stream));
  return ETXB_OK;
}

// A new geometry's vertices and triangles on the device, its BVH2 built there (bvh_build_device.cu: the tree of build_bvh), and the check of
// its depth against the traversal stack.  Everything goes into the prep's own buffers: a refusal or a CUDA error leaves the committed scene as it was.
int prepare_bvh(etxb_ctx* ctx, const etxb_scene& s, ScenePrep& p) {
  if (p.have_bvh) return ETXB_OK;
  auto t0 = std::chrono::steady_clock::now();
  const auto* verts = static_cast<const etxb_vertex*>(s.vertices.a);
  std::vector<DVertex> dverts(s.vertices.count);
  for (uint64_t i = 0; i < s.vertices.count; ++i) {
    const etxb_vertex& v = verts[i];
    dverts[i].pos_u = make_float4(v.pos[0], v.pos[1], v.pos[2], v.tex[0]);
    dverts[i].nrm_v = make_float4(v.nrm[0], v.nrm[1], v.nrm[2], v.tex[1]);
    dverts[i].tan = make_float4(v.tan[0], v.tan[1], v.tan[2], 0.0f);
    dverts[i].btn = make_float4(v.btn[0], v.btn[1], v.btn[2], 0.0f);
  }
  if (int rc = upload(ctx, p.vertices, dverts.data(), dverts.size())) return rc;
  if (int rc = upload(ctx, p.triangles, reinterpret_cast<const DTriangle*>(s.triangles.a), size_t(s.triangles.count))) return rc;
  const auto b0 = std::chrono::steady_clock::now();
  DeviceBvhOut out;
  CUDA_OK(ctx, build_bvh_device(reinterpret_cast<const float*>(p.vertices.ptr), sizeof(DVertex), reinterpret_cast<const uint32_t*>(p.triangles.ptr), sizeof(DTriangle),
    uint32_t(s.triangles.count), false, ctx->stream, out));
  adopt(p.bvh_nodes, out.nodes, out.node_count);
  adopt(p.bvh_tris, reinterpret_cast<float4*>(out.tri_pos), size_t(out.slot_count) * 3u);
  p.max_depth = out.max_depth;
  ctx->bvh_build_seconds = seconds_since(b0);
  ctx->kernel_ms[K_BVH_BUILD] += float(ctx->bvh_build_seconds * 1.0e3);
  ctx->kernel_count[K_BVH_BUILD] += 1;
  p.bvh_seconds += seconds_since(t0);
  p.have_bvh = true;
  if (p.max_depth >= uint32_t(kBvhStackSize)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "BVH depth %u exceeds the traversal stack (%d)", p.max_depth, kBvhStackSize);
  return ETXB_OK;
}

bool geometry_kept(const etxb_ctx* ctx, const ScenePrep& p, bool reuse) { return reuse && ctx->hashes.valid && (ctx->hashes.geometry == p.hashes.geometry); }

// The device side of an upload (reuse = false: every buffer is allocated and copied again) or of an update (reuse = true: what the
// hashes show unchanged stays, path-state buffers of the same size stay).  Runs after prepare_scene, so only CUDA errors remain: they
// leave the scene not ready.  Ends with etxb_begin(ctx, 0).
int commit_scene(etxb_ctx* ctx, const etxb_scene& s, const etxb_camera& cam, ScenePrep& p, bool reuse, etxb_update_info* info) {
  const bool keep_geometry = geometry_kept(ctx, p, reuse);
  if (!keep_geometry)
    if (int rc = prepare_bvh(ctx, s, p)) return rc;
  const SceneHashes old = std::move(ctx->hashes);
  ctx->hashes = {};
  ctx->scene_ready = false;
  etxb_update_info st = {};
  ctx->has_stochastic_merge = p.cls.stochastic;
  ctx->plain_scene = p.cls.plain;
  ctx->opaque_scene = p.cls.opaque;
  DeviceScene& d = ctx->dscene;
  const auto* mats = static_cast<const etxb_material*>(s.materials.a);

  // ---- media: dense density grids go to HBM as they are ---------------------------------------------------------------------------------
  {
    const auto* meds = static_cast<const etxb_medium*>(s.mediums.a);
    std::vector<DMedium> dmeds(s.mediums.count);
    ctx->medium_density.resize(s.mediums.count);
    for (uint64_t i = 0; i < s.mediums.count; ++i) {
      const etxb_medium& md = meds[i];
      DMedium& dm = dmeds[i];
      dm = {};
      dm.bounds_min = {md.bounds_min[0], md.bounds_min[1], md.bounds_min[2]};
      dm.bounds_max = {md.bounds_max[0], md.bounds_max[1], md.bounds_max[2]};
      dm.cls = md.cls;
      dm.enable_explicit_connections = md.enable_explicit_connections;
      dm.absorption_index = md.absorption_index;
      dm.scattering_index = md.scattering_index;
      dm.phase_function_g = md.phase_function_g;
      dm.max_sigma = md.max_sigma;
      dm.dim_x = md.dimensions[0];
      dm.dim_y = md.dimensions[1];
      dm.dim_z = md.dimensions[2];
      DevBuf<float>& grid = ctx->medium_density[i];
      if (md.cls == 1u) {
        size_t n = size_t(dm.dim_x) * dm.dim_y * dm.dim_z;
        if (reuse && old.valid && (i < old.grids.size()) && (old.grids[i] == p.hashes.grids[i]) && (grid.count == n)) {
          st.grids_kept += 1;
        } else {
          CUDA_OK(ctx, grid.alloc(n));
          CUDA_OK(ctx, cudaMemcpyAsync(grid.ptr, md.density.a, n * 4, cudaMemcpyHostToDevice, ctx->stream));
          st.grids_uploaded += 1;
        }
        dm.density = grid.ptr;
      } else {
        grid.release();
      }
    }
    if (int rc = upload(ctx, ctx->mediums, dmeds.data(), dmeds.size())) return rc;
    d.mediums = ctx->mediums.ptr;
    d.medium_count = uint32_t(dmeds.size());
    d.has_boundaries = p.cls.boundaries ? 1 : 0;
    d.has_subsurface = p.cls.subsurface ? 1 : 0;
    d.subsurface_exit_material = s.subsurface_exit_material;
    d.deferred_shadow_rays = p.cls.deferred ? 1u : 0u;
  }
  // ---- images: pixels + flattened row/column CDFs (image.hxx:8-50) ---------------------------------------------------------------
  {
    const auto* imgs = static_cast<const etxb_image*>(s.images.a);
    std::vector<DImage> dimgs(s.images.count);
    ctx->image_pixels.resize(s.images.count);
    ctx->image_dists.resize(s.images.count * 2);
    for (uint64_t i = 0; i < s.images.count; ++i) {
      const etxb_image& im = imgs[i];
      DImage& di = dimgs[i];
      di = {};
      const size_t bytes = image_pixel_bytes(im);
      const bool table = image_has_table(im);
      DevBuf<uint8_t>& pixels = ctx->image_pixels[i];
      DevBuf<uint8_t>& x_dist = ctx->image_dists[i * 2];
      DevBuf<uint8_t>& y_dist = ctx->image_dists[i * 2 + 1];
      if (reuse && old.valid && (i < old.images.size()) && (old.images[i] == p.hashes.images[i]) && (pixels.count == bytes)) {
        st.images_kept += 1;
      } else {
        CUDA_OK(ctx, pixels.alloc(bytes));
        CUDA_OK(ctx, cudaMemcpyAsync(pixels.ptr, im.pixels.a, bytes, cudaMemcpyHostToDevice, ctx->stream));
        x_dist.release();
        y_dist.release();
        if (table) {
          size_t nx = size_t(im.isize[0]) + 1u, ny = size_t(im.isize[1]) + 1u;
          std::vector<etxb_distribution_entry> flat(nx * im.isize[1]);
          const auto* rows = static_cast<const etxb_distribution*>(im.x_distributions.a);
          for (uint32_t y = 0; y < im.isize[1]; ++y) memcpy(flat.data() + size_t(y) * nx, rows[y].values.a, nx * sizeof(etxb_distribution_entry));
          CUDA_OK(ctx, x_dist.alloc(flat.size() * sizeof(etxb_distribution_entry)));
          CUDA_OK(ctx, cudaMemcpy(x_dist.ptr, flat.data(), flat.size() * sizeof(etxb_distribution_entry), cudaMemcpyHostToDevice));
          CUDA_OK(ctx, y_dist.alloc(ny * sizeof(etxb_distribution_entry)));
          CUDA_OK(ctx, cudaMemcpy(y_dist.ptr, im.y_distribution.values.a, ny * sizeof(etxb_distribution_entry), cudaMemcpyHostToDevice));
        }
        st.images_uploaded += 1;
      }
      di.pixels_f32 = (im.format == 1u) ? reinterpret_cast<const float4*>(pixels.ptr) : nullptr;
      di.pixels_u8 = (im.format == 2u) ? reinterpret_cast<const uchar4*>(pixels.ptr) : nullptr;
      di.fsize_x = im.fsize[0]; di.fsize_y = im.fsize[1];
      di.offset_x = im.offset[0]; di.offset_y = im.offset[1];
      di.scale_x = im.scale[0]; di.scale_y = im.scale[1];
      di.isize_x = im.isize[0]; di.isize_y = im.isize[1];
      di.normalization = im.normalization;
      di.options = im.options;
      di.format = im.format;
      if (table) {
        di.x_dist = reinterpret_cast<const etxb_distribution_entry*>(x_dist.ptr);
        di.y_dist = reinterpret_cast<const etxb_distribution_entry*>(y_dist.ptr);
        di.has_distribution = 1;
      }
    }
    if (int rc = upload(ctx, ctx->images, dimgs.data(), dimgs.size())) return rc;
    d.images = ctx->images.ptr;
    d.image_count = uint32_t(dimgs.size());
  }
  const auto* spectra = static_cast<const etxb_spectrum*>(s.spectrums.a);
  std::vector<DSpectrum> dspec(s.spectrums.count);
  for (uint64_t i = 0; i < s.spectrums.count; ++i) {
    for (uint32_t k = 0; k < 441; ++k) dspec[i].power[k] = spectra[i].entries[k].power;
    memcpy(dspec[i].rgb, spectra[i].integrated, 12);
  }

  // ---- geometry ------------------------------------------------------------------------------------------------------
  static_assert(sizeof(DTriangle) == sizeof(etxb_triangle), "triangle layout");
  if (!keep_geometry) {
    if (int rc = copy_device(ctx, ctx->vertices, p.vertices)) return rc;
    if (int rc = copy_device(ctx, ctx->triangles, p.triangles)) return rc;
  }
  if (int rc = upload(ctx, ctx->tri_emitter, static_cast<const uint32_t*>(s.triangle_to_emitter.a), size_t(s.triangle_to_emitter.count))) return rc;
  if (int rc = upload(ctx, ctx->materials, mats, size_t(s.materials.count))) return rc;
  if (int rc = upload(ctx, ctx->profiles, static_cast<const etxb_emitter_profile*>(s.emitter_profiles.a), size_t(s.emitter_profiles.count))) return rc;
  if (int rc = upload(ctx, ctx->emitters, static_cast<const etxb_emitter*>(s.emitter_instances.a), size_t(s.emitter_instances.count))) return rc;
  if (int rc = upload(ctx, ctx->spectra, dspec.data(), dspec.size())) return rc;
  if (int rc = upload(ctx, ctx->emitter_dist, static_cast<const etxb_distribution_entry*>(s.emitters_distribution.values.a), size_t(s.emitter_instances.count) + 1u))
    return rc;
  if (!keep_geometry) {
    if (int rc = copy_device(ctx, ctx->bvh_nodes, p.bvh_nodes)) return rc;
    if (int rc = copy_device(ctx, ctx->bvh_tris, p.bvh_tris)) return rc;
    d.bvh_node_count = uint32_t(p.bvh_nodes.count);
  }
  d.vertices = ctx->vertices.ptr;
  d.triangles = ctx->triangles.ptr;
  d.tri_emitter = ctx->tri_emitter.ptr;
  d.materials = ctx->materials.ptr;
  d.emitter_profiles = ctx->profiles.ptr;
  d.emitters = ctx->emitters.ptr;
  d.spectra = ctx->spectra.ptr;
  d.emitter_dist = ctx->emitter_dist.ptr;
  d.bvh_nodes = ctx->bvh_nodes.ptr;
  d.bvh_tris = ctx->bvh_tris.ptr;
  bool keep_wide = false;
#if !(defined(ETXB_PARITY) && ETXB_PARITY)
  // a geometry whose 4-wide tree the traversal stack cannot hold keeps that verdict with it: an update that keeps the geometry does not
  // collapse the tree again only to reject it
  if (!keep_geometry) ctx->wide_rejected = false;
  keep_wide = keep_geometry && ctx->has_stochastic_merge && ((d.wide_nodes != nullptr) || ctx->wide_rejected);
#endif
  if (!keep_wide) {
    d.wide_nodes = nullptr;
    d.wide_node_count = 0;
    if (reuse) ctx->wide_nodes.release();
  }
#if !(defined(ETXB_PARITY) && ETXB_PARITY)
  if (ctx->has_stochastic_merge && !keep_wide) {
    // the sampler streams of such a scene's stochastic stages are the product build's own already: its traversal kernels may meet candidates in
    // another order, so they walk the 4-wide quantised form of the tree (dwide.cuh); Lambert / delta scenes keep the oracle's candidate order
    if (!p.have_wide) {
      // collapsed on the device from the committed BVH2 (new or kept: bvh_build_device.cu, the tree of build_wide_bvh)
      auto t0 = std::chrono::steady_clock::now();
      WideNode* wide = nullptr;
      uint32_t count = 0;
      CUDA_OK(ctx, build_wide_bvh_device(ctx->bvh_nodes.ptr, d.bvh_node_count, ctx->stream, &wide, &count, &p.max_stack));
      adopt(p.wide, wide, count);
      p.have_wide = true;
      const double seconds = seconds_since(t0);
      ctx->kernel_ms[K_BVH_WIDE] += float(seconds * 1.0e3);
      ctx->kernel_count[K_BVH_WIDE] += 1;
      p.bvh_seconds += seconds;
    }
    if (p.max_stack < uint32_t(kWideStackSize)) {
      if (int rc = copy_device(ctx, ctx->wide_nodes, p.wide)) return rc;
      d.wide_nodes = ctx->wide_nodes.ptr;
      d.wide_node_count = uint32_t(p.wide.count);
    } else {
      ctx->wide_rejected = true;
    }
  }
#endif
  d.emitter_count = uint32_t(s.emitter_instances.count);
  d.triangle_count = uint32_t(s.triangles.count);
  d.emitter_total_weight = s.emitters_distribution.total_weight;
  memcpy(d.env_emitters, s.environment_emitters, sizeof(d.env_emitters));
  d.env_emitter_count = s.environment_emitter_count;
  d.bounding_sphere_center = {s.bounding_sphere_center[0], s.bounding_sphere_center[1], s.bounding_sphere_center[2]};
  d.bounding_sphere_radius = s.bounding_sphere_radius;
  d.min_path_length = s.min_path_length;
  d.max_path_length = s.max_path_length;
  d.samples = s.samples;
  d.random_path_termination = s.random_path_termination;
  d.spectral = (s.flags & ETXB_SCENE_SPECTRAL) ? 1u : 0u;
  d.spectrum_count = uint32_t(s.spectrums.count);
  d.default_dielectric_eta = s.default_dielectric_eta;
  d.default_conductor_eta = s.default_conductor_eta;
  d.default_conductor_k = s.default_conductor_k;
  d.camera = cam;
  ctx->spectral = d.spectral != 0;
  ctx->pixel_sampler_image = s.pixel_sampler_image;
  ctx->pixel_sampler_radius = s.pixel_sampler_radius;
  ctx->noise_threshold = s.noise_threshold;
  ctx->radiance_clamp = s.radiance_clamp;
  ctx->scene_samples = s.samples;

  // ---- film + queues (Film::allocate, film.cxx) ----------------------------------------------------------------------
  // an update keeps every buffer whose size is what the upload would allocate (DevBuf::ensure)
  uint32_t allocations = 0;
  auto sized = [&](auto& b, size_t count) -> cudaError_t {
    if (reuse) return b.ensure(count, allocations);
    allocations += 1;
    return b.alloc(count);
  };
  if ((ctx->width != cam.film_size[0]) || (ctx->height != cam.film_size[1])) ctx->film_denoised.release();  // Denoised starts over at a new film size
  ctx->width = cam.film_size[0];
  ctx->height = cam.film_size[1];
  ctx->path_count = ctx->width * ctx->height;
  size_t n = ctx->path_count;
  if (!reuse) {
    ctx->film_normals.release();  // sized by the film: re-allocated by the next path-tracer run
  } else if (ctx->film_normals.ptr && (ctx->film_normals.count != n)) {
    if (int rc = pt_ensure_film(ctx)) return rc;  // the path tracer's layers and per-pixel history at the new film size
    allocations += 1;
  }
  DevBuf<float4>* per_path_f4[] = {&ctx->ray_o, &ctx->ray_d, &ctx->thr, &ctx->mis, &ctx->hit, &ctx->gathered, &ctx->merged, &ctx->camera_value, &ctx->film_camera,
    &ctx->film_light, &ctx->film_light_iteration, &ctx->film_out, &ctx->bs_weight_pdf, &ctx->bs_wo_eta};
  for (auto* b : per_path_f4) CUDA_OK(ctx, sized(*b, n));
  CUDA_OK(ctx, sized(ctx->bs_props, n));
  CUDA_OK(ctx, sized(ctx->misc, n));
  CUDA_OK(ctx, sized(ctx->wavelength, n));
  DevBuf<uint32_t>* per_path_u32[] = {&ctx->lv_count, &ctx->lp_offset, &ctx->queue_a, &ctx->queue_b, &ctx->sampler_end_light, &ctx->sampler_end_camera, &ctx->merge_key};
  for (auto* b : per_path_u32) CUDA_OK(ctx, sized(*b, n));
  CUDA_OK(ctx, sized(ctx->conn_count, 1));
  CUDA_OK(ctx, sized(ctx->queue_counts, 4));
  CUDA_OK(ctx, sized(ctx->lv_tmp_count, 1));
  CUDA_OK(ctx, sized(ctx->overflow, 1));
  CUDA_OK(ctx, sized(ctx->grid_bbox, 8));
  CUDA_OK(ctx, sized(ctx->counters, 1));
  uint64_t cap = ctx->max_light_vertices_cfg ? ctx->max_light_vertices_cfg : uint64_t(n) * 16ull;
  cap = std::min<uint64_t>(cap, 0x7fffffffull);
  ctx->lv_capacity = uint32_t(cap);
  CUDA_OK(ctx, sized(ctx->lv_tmp, cap));
  CUDA_OK(ctx, sized(ctx->lv_final, cap));
  CUDA_OK(ctx, sized(ctx->conn_list, cap));
  if (ctx->has_stochastic_merge) {
    CUDA_OK(ctx, sized(ctx->conn_list_sorted, cap));
    CUDA_OK(ctx, sized(ctx->queue_sorted, n));
    CUDA_OK(ctx, sized(ctx->queue_keys, n));
    CUDA_OK(ctx, sized(ctx->queue_keys_sorted, n));
  } else {
    ctx->conn_list_sorted.release();
    ctx->queue_sorted.release();
    ctx->queue_keys.release();
    ctx->queue_keys_sorted.release();
  }
#if defined(ETXB_PARITY) && ETXB_PARITY
  ctx->conn_rec.release();
#else
  // the connection stage's per-path camera vertex records (make_params: connect_stage = has_stochastic_merge)
  if (ctx->has_stochastic_merge) {
    CUDA_OK(ctx, sized(ctx->conn_rec, n * (ctx->spectral ? kConnRecRows<true> : kConnRecRows<false>)));
  } else {
    ctx->conn_rec.release();
  }
#endif
  CUDA_OK(ctx, sized(ctx->trace_cursor, 1));
  const bool atomic_candidate = ctx->opaque_scene && ctx->plain_scene && ctx->has_stochastic_merge;
  if (ctx->dscene.deferred_shadow_rays || atomic_candidate) {
    // atomic mode: a camera bounce queues its vertex connections (<= cap, the pair list's capacity) plus one emitter segment per path
    const uint64_t shadow_cap = std::min<uint64_t>(cap + (atomic_candidate ? n : 0), 0x7fffffffull);
    CUDA_OK(ctx, sized(ctx->shadow_span, n));
    CUDA_OK(ctx, sized(ctx->shadow_p0, shadow_cap));
    CUDA_OK(ctx, sized(ctx->shadow_p1, shadow_cap));
    CUDA_OK(ctx, sized(ctx->shadow_value, shadow_cap));
    CUDA_OK(ctx, sized(ctx->shadow_result, shadow_cap));
    CUDA_OK(ctx, sized(ctx->shadow_count, 2));
  } else {
    ctx->shadow_span.release();
    ctx->shadow_p0.release();
    ctx->shadow_p1.release();
    ctx->shadow_value.release();
    ctx->shadow_result.release();
  }
  // the sort buffers also hold the gather queue and the path queues (up to one entry per path), whatever the configured pool capacity
  const uint64_t sort_cap = std::max<uint64_t>(cap, n);
  DevBuf<uint32_t>* per_vertex_u32[] = {&ctx->keys_in, &ctx->keys_out, &ctx->vals_in, &ctx->vals_out};
  for (auto* b : per_vertex_u32) CUDA_OK(ctx, sized(*b, sort_cap));
  DevBuf<float4>* per_vertex_f4[] = {&ctx->g_pos, &ctx->g_nrm, &ctx->g_win, &ctx->g_thr};
  for (auto* b : per_vertex_f4) CUDA_OK(ctx, sized(*b, cap));
  CUDA_OK(ctx, sized(ctx->cell_range, next_pow2(cap)));
  // one scratch buffer for every CUB call of an iteration: the 32-bit pair sorts (photon grid, gather queue, path queues), the pair-list
  // sort with its 64-bit (path, light vertex) values, and the scan over the per-path vertex counts
  size_t temp_sort = 0, temp_sort64 = 0, temp_scan = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, temp_sort, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, int(sort_cap));
  cub::DeviceRadixSort::SortPairs(nullptr, temp_sort64, (uint32_t*)nullptr, (uint32_t*)nullptr, (unsigned long long*)nullptr, (unsigned long long*)nullptr, int(sort_cap), 0, 16);
  cub::DeviceScan::ExclusiveSum(nullptr, temp_scan, (uint32_t*)nullptr, (uint32_t*)nullptr, int(n));
  CUDA_OK(ctx, sized(ctx->cub_temp, std::max(std::max(temp_sort, temp_sort64), temp_scan) + 256));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->overflow.ptr, 0, 4, ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->counters.ptr, 0, sizeof(DeviceCounters), ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->sampler_end_light.ptr, 0, n * 4, ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->sampler_end_camera.ptr, 0, n * 4, ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->lv_count.ptr, 0, n * 4, ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->lp_offset.ptr, 0, n * 4, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->hashes = p.hashes;
  ctx->scene_ready = true;
  if (info) {
    st.kept = (keep_geometry ? ETXB_KEPT_GEOMETRY : 0u) | ((keep_wide && (d.wide_nodes != nullptr)) ? ETXB_KEPT_WIDE_TREE : 0u) | (allocations == 0 ? ETXB_KEPT_PATH_STATE : 0u);
    st.fingerprint_seconds = p.fingerprint_seconds;
    st.bytes_hashed = p.bytes_hashed;
    st.bvh_seconds = p.bvh_seconds;
    *info = st;
  }
  return etxb_begin(ctx, 0);
}

// The three passes of a VCM iteration, each instantiated for the context's scene class.  The light pass starts the iteration's clock,
// the camera pass stops it (finish_iteration).
int light_pass(etxb_ctx* ctx) {
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  cudaSetDevice(ctx->device);
  CUDA_OK(ctx, cudaEventRecord(ctx->ev_iter_start, ctx->stream));
  if (ctx->spectral) return ctx->plain_scene ? run_light_pass<true, true>(ctx) : run_light_pass<true, false>(ctx);
  return ctx->plain_scene ? run_light_pass<false, true>(ctx) : run_light_pass<false, false>(ctx);
}

int grid_build(etxb_ctx* ctx, const LightVertexRec* records, uint32_t count) {
  return ctx->spectral ? run_grid_build<true>(ctx, records, count) : run_grid_build<false>(ctx, records, count);
}

int camera_pass(etxb_ctx* ctx) {
  int rc = ctx->spectral ? (ctx->plain_scene ? run_camera_pass<true, true>(ctx) : run_camera_pass<true, false>(ctx))
                         : (ctx->plain_scene ? run_camera_pass<false, true>(ctx) : run_camera_pass<false, false>(ctx));
  if (rc) return rc;
  return finish_iteration(ctx);
}

// one whole iteration on the calling thread; returns when it has finished (the bounce loops read queue sizes back)
int run_iteration_blocking(etxb_ctx* ctx) {
  if (ctx->integrator == ETXB_INTEGRATOR_PT) {
    cudaSetDevice(ctx->device);
    if (ctx->spectral) return ctx->plain_scene ? run_pt_iteration<true, true>(ctx) : run_pt_iteration<true, false>(ctx);
    return ctx->plain_scene ? run_pt_iteration<false, true>(ctx) : run_pt_iteration<false, false>(ctx);
  }
  if (int rc = light_pass(ctx)) return rc;
  const LightVertexRec* records = ctx->lv_final.ptr;
  uint32_t count = ctx->last_light_vertices;
  if (ctx->comm != nullptr) {  // pixel tiles over several GPUs: light image + photon records are exchanged here (comm_exchange)
    if (int rc = comm_exchange(ctx, &records, &count)) return rc;
  }
  if (int rc = grid_build(ctx, records, count)) return rc;
  return camera_pass(ctx);
}

void ctx_worker(etxb_ctx* ctx) {
  std::unique_lock<std::mutex> lock(ctx->worker_m);
  for (;;) {
    ctx->worker_cv.wait(lock, [&] { return ctx->worker_quit || (ctx->worker_queued > 0); });
    if (ctx->worker_quit) return;
    ctx->worker_queued -= 1;
    ctx->worker_busy = true;
    lock.unlock();
    int rc = run_iteration_blocking(ctx);
    lock.lock();
    ctx->worker_busy = false;
    if ((rc != ETXB_OK) && (ctx->worker_error == ETXB_OK)) {
      ctx->worker_error = rc;
      ctx->worker_queued = 0;
    }
    if (ctx->worker_queued == 0) ctx->worker_idle.notify_all();
  }
}

// blocks until every queued iteration has finished; returns (and clears) the first error one of them hit
int ctx_drain(etxb_ctx* ctx) {
  std::unique_lock<std::mutex> lock(ctx->worker_m);
  ctx->worker_idle.wait(lock, [&] { return (ctx->worker_queued == 0) && !ctx->worker_busy; });
  int rc = ctx->worker_error;
  ctx->worker_error = ETXB_OK;
  return rc;
}

// Film::layer (film.cxx:381-418): the device buffer that holds `layer` as float4 (computed into film_out where the layer is derived)
int film_layer_source(etxb_ctx* ctx, uint32_t layer, const float4** out_src) {
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  cudaSetDevice(ctx->device);
  const float4* src = nullptr;
  switch (layer) {
    case ETXB_FILM_RESULT: {
      FilmBuffers film = {ctx->film_camera.ptr, ctx->film_light.ptr, ctx->film_light_iteration.ptr, ctx->width, ctx->height};
      k_film_resolve<<<blocks_for(ctx->path_count, 256), 256, 0, ctx->stream>>>(film, ctx->film_out.ptr);
      ctx->kernel_launches += 1;
      src = ctx->film_out.ptr;
      break;
    }
    case ETXB_FILM_CAMERA:
      src = ctx->film_camera.ptr;
      break;
    case ETXB_FILM_LIGHT:
      src = ctx->film_light.ptr;
      break;
    case ETXB_FILM_LIGHT_ITERATION:
      src = ctx->film_light_iteration.ptr;
      break;
    case ETXB_FILM_CAMERA_ADAPTIVE:
      if (int rc = film_ensure_adaptive(ctx)) return rc;
      src = ctx->film_adaptive.ptr;
      break;
    case ETXB_FILM_DENOISED:
      if (ctx->film_denoised.count != ctx->path_count) {
        CUDA_OK(ctx, ctx->film_denoised.alloc(ctx->path_count));
        CUDA_OK(ctx, cudaMemsetAsync(ctx->film_denoised.ptr, 0, ctx->film_denoised.bytes(), ctx->stream));
      }
      src = ctx->film_denoised.ptr;
      break;
    case ETXB_FILM_NORMALS:
    case ETXB_FILM_ALBEDO: {
      if (int rc = pt_ensure_film(ctx)) return rc;
      if (layer == ETXB_FILM_NORMALS) {
        k_film_layer_normals<<<blocks_for(ctx->path_count, 256), 256, 0, ctx->stream>>>(ctx->film_normals.ptr, ctx->film_out.ptr, ctx->path_count);
        ctx->kernel_launches += 1;
        src = ctx->film_out.ptr;
      } else {
        src = ctx->film_albedo.ptr;
      }
      break;
    }
    default:
      return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "unknown film layer %u", layer);
  }
  *out_src = src;
  return ETXB_OK;
}

// Film::denoise (DESIGN §13): the three kernels of kernels_denoise.cuh on `in`, into `out` (and the smoothed variance into `out_variance`, when
// given).  ETXB_ERR_NOT_READY, with `out` untouched, where a pixel has fewer than two samples.  Synchronous.
int run_denoise(etxb_ctx* ctx, const DenoiseInputs& in, float4* out, float4* out_variance) {
  const uint32_t n = in.width * in.height;
  DevBuf<float4>* scratch[] = {&ctx->denoise_u, &ctx->denoise_var_raw, &ctx->denoise_var};
  for (auto* b : scratch)
    if (b->count != n) CUDA_OK(ctx, b->alloc(n));
  if (!ctx->denoise_flag.ptr) CUDA_OK(ctx, ctx->denoise_flag.alloc(1));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->denoise_flag.ptr, 0, 4, ctx->stream));
  {
    LaunchTimer t(ctx, K_DENOISE_VARIANCE);
    k_denoise_variance<<<blocks_for(n, 256), 256, 0, ctx->stream>>>(in, ctx->denoise_u.ptr, ctx->denoise_var_raw.ptr, ctx->denoise_flag.ptr);
  }
  uint32_t not_ready = 0;
  CUDA_OK(ctx, cudaMemcpyAsync(&not_ready, ctx->denoise_flag.ptr, 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  if (not_ready) {
    resolve_timers(ctx);
    return fail(ctx, ETXB_ERR_NOT_READY, "denoise: a pixel has fewer than two samples (the variance estimate needs both half buffers)");
  }
  {
    LaunchTimer t(ctx, K_DENOISE_SMOOTH);
    k_denoise_smooth<<<blocks_for(n, 256), 256, 0, ctx->stream>>>(ctx->denoise_var_raw.ptr, ctx->denoise_var.ptr, in.width, in.height);
  }
  {
    LaunchTimer t(ctx, K_DENOISE_NLM);
    const dim3 tiles((in.width + kDenoiseTile - 1) / kDenoiseTile, (in.height + kDenoiseTile - 1) / kDenoiseTile);
    k_denoise_nlm<<<tiles, kDenoiseTile * kDenoiseTile, 0, ctx->stream>>>(in, ctx->denoise_u.ptr, ctx->denoise_var.ptr, out);
  }
  if (out_variance) CUDA_OK(ctx, cudaMemcpyAsync(out_variance, ctx->denoise_var.ptr, size_t(n) * 16, cudaMemcpyDeviceToDevice, ctx->stream));
  CUDA_OK(ctx, cudaGetLastError());
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  resolve_timers(ctx);
  return ETXB_OK;
}

template <bool SP>
int debug_merge(etxb_ctx* ctx, uint32_t record_count, const etxb_merge_query* d_queries, uint32_t count, float4* d_pos_nrm) {
  if (int rc = run_grid_build<SP>(ctx, ctx->lv_final.ptr, record_count)) return rc;
  LaunchParams p = make_params(ctx);
  if (count) k_debug_merge_stage<SP><<<blocks_for(count, 128), 128, 0, ctx->stream>>>(p, d_queries, count, ctx->queue_a.ptr, d_pos_nrm);
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaMemcpyAsync(ctx->queue_counts.ptr, &count, 4, cudaMemcpyHostToDevice, ctx->stream));
  if (count == 0) return ETXB_OK;
  return launch_merge<SP>(ctx, p, ctx->queue_a.ptr, ctx->queue_counts.ptr, count);
}

// What one rank takes of `iterations` more iterations of a replica-mode job (ordinals base .. base + iterations - 1).  Whole frames are dealt
// round-robin (ordinal j on rank j % world).  What is left when the count is not a multiple of the ranks would leave some ranks a whole iteration
// behind the others (20 iterations on 8 ranks: 3, 3, 3, 3, 2, 2, 2, 2): with a split lane those R iterations are split instead, each over
// P = world / R ranks by camera tile — every part traces the whole light pass itself (same photon map, no exchange) and the camera pass of its
// tiles; the parts meet in the frame reduce.  A split lane's film is made of ONE (part, parts) geometry: a later round that would need another
// parts count is dealt as whole frames (with the count fixed, a rank's part is always rank % parts).  Returns the parts of this round's split
// (0: none).
uint32_t replica_plan(uint32_t world, uint32_t rank, uint32_t base, uint32_t iterations, bool split_lane, uint32_t have_parts, std::vector<WorkItem>& out) {
  uint32_t whole = iterations, rest = 0, parts = 1;
  if ((iterations >= world) && split_lane) {
    rest = iterations % world;
    parts = rest ? (world / rest) : 1u;
    if ((parts >= 2u) && ((have_parts == 0u) || (have_parts == parts))) {
      whole = iterations - rest;
    } else {
      rest = 0;
    }
  }
  for (uint32_t j = base; j < base + whole; ++j)
    if ((j % world) == rank) out.push_back({j, 0u, 1u});
  for (uint32_t r = 0; r < rest; ++r) {
    if ((rank / parts) == r) out.push_back({base + whole + r, rank % parts, parts});
  }
  return rest ? parts : 0u;
}

// The planner: deals the ordinals enqueued .. enqueued + iterations - 1 into the queues and routes every lane to its queue (see WorkPlan).
void plan_enqueue(WorkPlan& p, uint32_t iterations) {
  const uint32_t lanes = uint32_t(p.queues.size());
  const bool tiles = p.mode == GroupMode::tiles;
  for (uint32_t l = 0; l < lanes; ++l) p.lane_queue[l] = (tiles || (l == p.split_lane)) ? l : 0u;
  if (p.mode == GroupMode::replicas) {
    std::vector<WorkItem> items;
    uint32_t parts_used = replica_plan(p.world, p.rank, p.enqueued, iterations, p.split_lane != 0xffffffffu, p.split_parts, items);
    for (const WorkItem& it : items) {
      if (it.parts > 1u) p.split_part = it.part;
      p.queues[(it.parts > 1u) ? p.split_lane : 0u].push_back(it);
    }
    if (parts_used) p.split_parts = parts_used;  // every rank records the split geometry, also those that got no part of this round
  } else {
    for (uint32_t k = p.enqueued; k < p.enqueued + iterations; ++k) p.queues[tiles ? (k % lanes) : 0u].push_back({k, 0u, 1u});
  }
  p.enqueued += iterations;
}
void plan_clear(WorkPlan& p) {
  for (auto& q : p.queues) q.clear();
  p.enqueued = 0;
}

bool group_has_work(const etxb_group* grp, uint32_t lane) { return !grp->plan.queues[grp->plan.lane_queue[lane]].empty(); }
bool group_idle(const etxb_group* grp) {
  if (grp->in_flight > 0) return false;
  for (const auto& q : grp->plan.queues)
    if (!q.empty()) return false;
  return true;
}

void group_worker(etxb_group* grp, uint32_t lane) {
  cudaSetDevice(grp->device);
  etxb_ctx* ctx = grp->lanes[lane];
  std::unique_lock<std::mutex> lock(grp->m);
  for (;;) {
    grp->cv_work.wait(lock, [&] { return grp->quit || group_has_work(grp, lane); });
    if (grp->quit) return;
    auto& queue = grp->plan.queues[grp->plan.lane_queue[lane]];
    const WorkItem item = queue.front();
    queue.pop_front();
    grp->taken = std::max(grp->taken, item.ordinal + 1u);
    uint32_t iteration = grp->first_iteration + item.ordinal;
    grp->in_flight += 1;
    lock.unlock();
    if (item.parts > 1u) {
      // this lane renders the camera pass of its part only; the light pass (and so the photon map) in full
      ctx->rank = item.part;
      ctx->world = item.parts;
      ctx->light_full = true;
    }
    int rc = etxb_set_next_iteration(ctx, iteration);
    if (rc == ETXB_OK) rc = run_iteration_blocking(ctx);  // returns when the iteration has finished (the bounce loops read queue sizes back)
    lock.lock();
    grp->in_flight -= 1;
    grp->last_iteration_seconds = ctx->last_iteration_time;
    if ((rc != ETXB_OK) && (grp->error == ETXB_OK)) {
      grp->error = rc;
      grp->error_text = etxb_last_error(ctx);
      plan_clear(grp->plan);
    }
    if (group_idle(grp)) {
      grp->busy_seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - grp->busy_since).count();
      grp->cv_idle.notify_all();
    }
  }
}

// A call the group refuses in its present state: the reason goes to etxb_group_last_error and to lane 0's etxb_last_error
int group_refuse(etxb_group* grp, const char* why, int code = ETXB_ERR_INVALID_ARGUMENT) {
  fail(grp->lanes[0], code, "%s", why);
  std::lock_guard<std::mutex> lock(grp->m);
  grp->error_text = why;
  return code;
}

int group_combine_into(etxb_group* grp, uint32_t layer, DevBuf<float4>& target, uint32_t* completed, bool raw = false) {
  etxb_ctx* first = grp->lanes[0];
  if (!first->scene_ready) return fail(first, ETXB_ERR_NOT_READY, "no scene uploaded");
  size_t n = first->path_count;
  cudaSetDevice(grp->device);
  if (target.count < n) CUDA_OK(first, target.alloc(n));
  FilmLanes f = {};
  f.lanes = uint32_t(grp->lanes.size());
  f.layer = layer;
  f.pixels = uint32_t(n);
  uint32_t total = 0;
  for (auto* c : grp->lanes) total += c->completed;
  for (uint32_t l = 0; l < f.lanes; ++l) {
    f.camera[l] = grp->lanes[l]->film_camera.ptr;
    f.light[l] = grp->lanes[l]->film_light.ptr;
    f.weight[l] = raw ? float(grp->lanes[l]->completed) : (total ? float(double(grp->lanes[l]->completed) / double(total)) : 0.0f);
    f.weight_light[l] = f.weight[l];
    f.weight_count[l] = f.weight[l];
    if (raw && (l == grp->plan.split_lane) && (grp->plan.split_part != 0u)) {
      // a camera-split lane that is not part 0: its camera tiles count, its (complete, redundant) light image and its iteration count do not
      f.weight_light[l] = 0.0f;
      f.weight_count[l] = 0.0f;
    }
  }
  f.raw = raw ? 1u : 0u;
  // lanes that are still rendering keep updating their films (a preview, like reading the reference's film while it runs); after
  // etxb_group_wait every lane has synchronised its stream and the result is exact
  k_film_combine<<<blocks_for(f.pixels, 256), 256, 0, grp->stream>>>(f, target.ptr);
  CUDA_OK(first, cudaStreamSynchronize(grp->stream));
  if (completed) *completed = total;
  return ETXB_OK;
}

}  // namespace

const char* etxb_build_flavor(void) { return kFlavor; }

int etxb_device_count(void) {
  int n = 0;
  cudaError_t err = cudaGetDeviceCount(&n);
  if (err != cudaSuccess) return ETXB_ERR_NO_DEVICE;
  return n;
}

int etxb_create(etxb_ctx** out_ctx, const etxb_device_config* cfg) {
  if (!out_ctx) return ETXB_ERR_INVALID_ARGUMENT;
  *out_ctx = nullptr;
  int n = etxb_device_count();
  if (n <= 0) return ETXB_ERR_NO_DEVICE;
  int device = cfg ? cfg->device_index : 0;
  if (device < 0 || device >= n) return ETXB_ERR_INVALID_ARGUMENT;
  if (cudaSetDevice(device) != cudaSuccess) return ETXB_ERR_CUDA;
  auto* ctx = new etxb_ctx();
  ctx->device = device;
  int sms = 0;
  if ((cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess) && (sms > 0)) ctx->sm_count = uint32_t(sms);
  ctx->max_light_vertices_cfg = cfg ? cfg->max_light_vertices : 0;
  ctx->profile = cfg ? (cfg->flags & 1u) != 0 : false;
  if (ctx->profile) {
    // the per-launch timing events of an iteration (two per launch, a few thousand per iteration) exist from the start: a lane that renders its first
    // iteration inside a timed region (the camera-split lane of the replica mode) must not pay for creating them there
    ctx->event_pool.reserve(8192);
    for (uint32_t k = 0; k < 6144u; ++k) {
      cudaEvent_t e = nullptr;
      if (cudaEventCreate(&e) != cudaSuccess) break;
      ctx->event_pool.push_back(e);
    }
  }
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
    delete ctx;
    return ETXB_ERR_CUDA;
  }
  cudaEventCreate(&ctx->ev_iter_start);
  cudaEventCreate(&ctx->ev_iter_stop);
  etxb_options_default(&ctx->options);
  *out_ctx = ctx;
  return ETXB_OK;
}

void etxb_destroy(etxb_ctx* ctx) {
  if (!ctx) return;
  if (ctx->worker.joinable()) {
    {
      std::lock_guard<std::mutex> lock(ctx->worker_m);
      ctx->worker_queued = 0;
      ctx->worker_quit = true;
    }
    ctx->worker_cv.notify_all();
    ctx->worker.join();
  }
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  if (ctx->comm != nullptr) {
    if (NcclApi* n = nccl_api()) n->CommDestroy(ctx->comm);
    ctx->comm = nullptr;
  }
  if (ctx->comm_stream) cudaStreamDestroy(ctx->comm_stream);
  if (ctx->comm_ev_in) cudaEventDestroy(ctx->comm_ev_in);
  if (ctx->comm_ev_out) cudaEventDestroy(ctx->comm_ev_out);
  for (auto e : ctx->event_pool) cudaEventDestroy(e);
  cudaEventDestroy(ctx->ev_iter_start);
  cudaEventDestroy(ctx->ev_iter_stop);
  cudaStreamDestroy(ctx->stream);
  delete ctx;  // the device buffers free themselves, on ctx->device
}

const char* etxb_last_error(const etxb_ctx* ctx) { return ctx ? ctx->error.c_str() : "null context"; }

int etxb_upload_color_tables(etxb_ctx* ctx, const float* xyz_441x3, const float* rgb_response_391x3) {
  if (!ctx || !xyz_441x3 || !rgb_response_391x3) return ETXB_ERR_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  if (int rc = upload(ctx, ctx->xyz_table, xyz_441x3, 441 * 3)) return rc;
  if (int rc = upload(ctx, ctx->rgb_response_table, rgb_response_391x3, 391 * 3)) return rc;
  float sum = 0.0f;  // spectrum::kYIntegral (spectrum.hxx:187-193): float sum in table order
  for (int i = 0; i < 441; ++i) sum += xyz_441x3[i * 3 + 1];
  ctx->y_integral = sum;
  ctx->dscene.xyz_table = ctx->xyz_table.ptr;
  ctx->dscene.rgb_response_table = ctx->rgb_response_table.ptr;
  ctx->dscene.y_scale = 1.0f / sum;
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  return ETXB_OK;
}

int etxb_upload_blue_noise(etxb_ctx* ctx, const uint8_t* sobol_256x256, const uint8_t* scrambling, const uint8_t* ranking) {
  if (!ctx || !sobol_256x256 || !scrambling || !ranking) return ETXB_ERR_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  if (int rc = upload(ctx, ctx->bn_sobol, sobol_256x256, 256 * 256)) return rc;
  if (int rc = upload(ctx, ctx->bn_scrambling, scrambling, 128 * 128 * 8)) return rc;
  if (int rc = upload(ctx, ctx->bn_ranking, ranking, 128 * 128 * 8)) return rc;
  ctx->dscene.bn_sobol = ctx->bn_sobol.ptr;
  ctx->dscene.bn_scrambling = ctx->bn_scrambling.ptr;
  ctx->dscene.bn_ranking = ctx->bn_ranking.ptr;
  ctx->dscene.has_blue_noise = 1;
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  return ETXB_OK;
}

int etxb_upload_scene(etxb_ctx* ctx, const void* scene_blob, uint64_t scene_bytes, const void* camera_blob, uint64_t camera_bytes) {
  if (!ctx || !scene_blob || !camera_blob) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = check_scene_args(ctx, scene_bytes, camera_bytes)) return rc;
  ctx_drain(ctx);
  cudaSetDevice(ctx->device);
  ctx->scene_ready = false;
  const etxb_scene& s = *static_cast<const etxb_scene*>(scene_blob);
  const etxb_camera& cam = *static_cast<const etxb_camera*>(camera_blob);
  ScenePrep p;
  if (int rc = prepare_scene(ctx, s, cam, p)) return rc;
  return commit_scene(ctx, s, cam, p, false, nullptr);
}

int etxb_update_scene(etxb_ctx* ctx, const void* scene_blob, uint64_t scene_bytes, const void* camera_blob, uint64_t camera_bytes, etxb_update_info* info) {
  const auto t0 = std::chrono::steady_clock::now();
  if (info) memset(info, 0, sizeof(*info));
  if (!ctx || !scene_blob || !camera_blob) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = check_scene_args(ctx, scene_bytes, camera_bytes)) return rc;
  if (ctx->comm != nullptr) return fail(ctx, ETXB_ERR_UNSUPPORTED, "etxb_update_scene: a context with a communicator takes a new scene through etxb_upload_scene");
  ctx_drain(ctx);
  cudaSetDevice(ctx->device);
  const etxb_scene& s = *static_cast<const etxb_scene*>(scene_blob);
  const etxb_camera& cam = *static_cast<const etxb_camera*>(camera_blob);
  ScenePrep p;
  if (int rc = prepare_scene(ctx, s, cam, p)) return rc;
  int rc = commit_scene(ctx, s, cam, p, ctx->scene_ready, info);
  if (info) info->total_seconds = seconds_since(t0);
  return rc;
}

void etxb_options_default(etxb_vcm_options* opt) {
  if (!opt) return;
  opt->options = ETXB_VCM_FULL;
  opt->radius_decay = 256u;
  opt->kernel = 1u;
  opt->initial_radius = 0.0f;
  opt->blue_noise = 1u;
}

int etxb_options_set_key(etxb_vcm_options* opt, const char* key, double value) {
  if (!opt || !key) return ETXB_ERR_INVALID_ARGUMENT;
  auto set_bit = [&](uint32_t bit) { opt->options = (value != 0.0) ? (opt->options | bit) : (opt->options & ~bit); };
  std::string k = key;
  if (k == "vcm-initial_radius") opt->initial_radius = float(value);
  else if (k == "vcm-radius_decay") opt->radius_decay = uint32_t(value);
  else if (k == "vcm-blue_noise") opt->blue_noise = value != 0.0;
  else if (k == "vcm-kernel") opt->kernel = uint32_t(value);
  else if (k == "vcm-direct_hit") set_bit(ETXB_VCM_DIRECT_HIT);
  else if (k == "vcm-connect_to_light") set_bit(ETXB_VCM_CONNECT_TO_LIGHT);
  else if (k == "vcm-connect_to_camera") set_bit(ETXB_VCM_CONNECT_TO_CAMERA);
  else if (k == "vcm-connect_vertices") set_bit(ETXB_VCM_CONNECT_VERTICES);
  else if (k == "vcm-merge_vertices") set_bit(ETXB_VCM_MERGE_VERTICES);
  else if (k == "vcm-mis") set_bit(ETXB_VCM_ENABLE_MIS);
  else if (k == "vcm-merging") set_bit(ETXB_VCM_ENABLE_MERGING);
  else return ETXB_ERR_INVALID_ARGUMENT;
  return ETXB_OK;
}

int etxb_set_options(etxb_ctx* ctx, const etxb_vcm_options* opt) {
  if (!ctx || !opt) return ETXB_ERR_INVALID_ARGUMENT;
  if (opt->radius_decay == 0) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "radius_decay must be >= 1");
  ctx->options = *opt;
  return ETXB_OK;
}

int etxb_set_partition(etxb_ctx* ctx, uint32_t rank, uint32_t world) {
  if (!ctx || world == 0 || rank >= world) return ETXB_ERR_INVALID_ARGUMENT;
  if ((world > 1u) && (ctx->target_pixel_size > 1u)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "etxb_set_partition: pixel tiles and a film pixel size above 1 exclude each other");
  ctx->rank = rank;
  ctx->world = world;
  return ETXB_OK;
}

int etxb_set_next_iteration(etxb_ctx* ctx, uint32_t iteration) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  ctx->iteration = iteration;
  ctx->external_iteration = true;  // no auto-advance; the film mean counts this context's own iterations
  return ETXB_OK;
}

int etxb_set_film_pixel_size(etxb_ctx* ctx, uint32_t size) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  size = std::min(std::max(size, 1u), 1024u);  // Film::set_pixel_size (film.cxx:483-485)
  if ((size > 1u) && ((ctx->comm != nullptr) || (ctx->world > 1u)))
    return fail(ctx, ETXB_ERR_UNSUPPORTED, "etxb_set_film_pixel_size: pixel tiles index film pixels; the coarse preview renders on one GPU");
  ctx->target_pixel_size = size;
  return ETXB_OK;
}

int etxb_begin(etxb_ctx* ctx, uint32_t first_iteration) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  ctx_drain(ctx);  // Integrator::run first stops what is running (vcm_cpu.cxx:255-262)
  cudaSetDevice(ctx->device);
  size_t n = ctx->path_count;
  CUDA_OK(ctx, cudaMemsetAsync(ctx->film_camera.ptr, 0, n * 16, ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->film_light.ptr, 0, n * 16, ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->film_light_iteration.ptr, 0, n * 16, ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->counters.ptr, 0, sizeof(DeviceCounters), ctx->stream));
  CUDA_OK(ctx, cudaMemsetAsync(ctx->overflow.ptr, 0, 4, ctx->stream));
  if (ctx->pt_info.count == n) {
    // Film::clear(ClearCameraData) (film.cxx:345-368): the per-pixel history starts over
    CUDA_OK(ctx, cudaMemsetAsync(ctx->pt_info.ptr, 0, n * 4, ctx->stream));
    CUDA_OK(ctx, cudaMemsetAsync(ctx->pt_error.ptr, 0, n * 4, ctx->stream));
    DevBuf<float4>* layers[] = {&ctx->film_normals, &ctx->film_albedo};
    for (auto* b : layers) CUDA_OK(ctx, cudaMemsetAsync(b->ptr, 0, n * 16, ctx->stream));
  }
  if (ctx->film_adaptive.count == n) CUDA_OK(ctx, cudaMemsetAsync(ctx->film_adaptive.ptr, 0, n * 16, ctx->stream));
  // Film::clear applies the stored pixel size (film.cxx:365)
  ctx->pixel_size = ctx->target_pixel_size;
  ctx->launch_count = film_dims_x(ctx) * film_dims_y(ctx);
  ctx->pt_pixels_processed = 0;
  ctx->pt_active_pixels = ctx->launch_count;
  ctx->pt_noise_level = 0.0f;
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->iteration = first_iteration;
  ctx->completed = 0;
  ctx->total_time = 0.0;
  ctx->last_iteration_time = 0.0;
  ctx->overflow_flag = 0;
  ctx->kernel_launches = 0;
  ctx->branch_counts = {};
  memset(ctx->kernel_ms, 0, sizeof(ctx->kernel_ms));
  memset(ctx->kernel_count, 0, sizeof(ctx->kernel_count));
  return ETXB_OK;
}

int etxb_enqueue_iteration(etxb_ctx* ctx) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  std::lock_guard<std::mutex> lock(ctx->worker_m);
  if (ctx->worker_error != ETXB_OK) {
    int rc = ctx->worker_error;
    ctx->worker_error = ETXB_OK;
    return rc;
  }
  if (!ctx->worker.joinable()) ctx->worker = std::thread(ctx_worker, ctx);
  ctx->worker_queued += 1;
  ctx->worker_cv.notify_one();
  return ETXB_OK;
}


// ---- unidirectional path tracer (CPUPathTracing, rt/integrators/path_tracing.cxx) ---------------------------------------------------------
void etxb_pt_options_default(etxb_pt_options* opt) {
  if (!opt) return;
  opt->nee = opt->direct = opt->mis = opt->blue_noise = 1u;  // PTOptions (path_tracing_shared.hxx:8-14)
}

// the reference's option ids (path_tracing.cxx:36-39, 112-119)
int etxb_pt_options_set_key(etxb_pt_options* opt, const char* key, double value) {
  if (!opt || !key) return ETXB_ERR_INVALID_ARGUMENT;
  const uint32_t v = (value != 0.0) ? 1u : 0u;
  if (!strcmp(key, "direct")) opt->direct = v;
  else if (!strcmp(key, "nee")) opt->nee = v;
  else if (!strcmp(key, "mis")) opt->mis = v;
  else if (!strcmp(key, "bn")) opt->blue_noise = v;
  else return ETXB_ERR_INVALID_ARGUMENT;
  return ETXB_OK;
}

int etxb_pt_set_options(etxb_ctx* ctx, const etxb_pt_options* opt) {
  if (!ctx || !opt) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = ctx_drain(ctx)) return rc;
  ctx->pt_options = *opt;
  return ETXB_OK;
}

int etxb_set_integrator(etxb_ctx* ctx, uint32_t integrator) {
  if (!ctx || (integrator > ETXB_INTEGRATOR_PT)) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = ctx_drain(ctx)) return rc;
  // pixel tiles need the ranks' noise estimates combined (a communicator), and a group's lanes would each keep their own history
  if ((integrator == ETXB_INTEGRATOR_PT) && (ctx->world > 1u) && ((ctx->comm == nullptr) || ctx->group_lane))
    return fail(ctx, ETXB_ERR_UNSUPPORTED, ctx->group_lane ? "the path tracer does not run on a group in pixel-tile mode: each lane would keep its own per-pixel history"
                                                          : "the path tracer renders pixel tiles only with a communicator (etxb_comm_init)");
  ctx->integrator = integrator;
  return ETXB_OK;
}

int etxb_pt_get_status(etxb_ctx* ctx, etxb_pt_status* out) {
  if (!ctx || !out) return ETXB_ERR_INVALID_ARGUMENT;
  memset(out, 0, sizeof(*out));
  out->pixels_processed = ctx->pt_pixels_processed;
  out->active_pixels = ctx->pt_active_pixels;
  out->noise_level = ctx->pt_noise_level;
  out->max_sample_count = ctx->scene_samples;
  return ETXB_OK;
}

// Scene::noise_threshold / radiance_clamp / samples are scene settings the application edits between runs (ui.cxx) without a new upload
int etxb_set_scene_settings(etxb_ctx* ctx, float noise_threshold, float radiance_clamp) {
  if (!ctx || !(noise_threshold >= 0.0f) || !(radiance_clamp >= 0.0f)) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = ctx_drain(ctx)) return rc;
  ctx->noise_threshold = noise_threshold;
  ctx->radiance_clamp = radiance_clamp;
  return ETXB_OK;
}

// ---- pixel-tile sharding over NCCL -------------------------------------------------------------------------------------------------------
int etxb_comm_unique_id(void* out_id, uint64_t bytes) {
  if (!out_id || (bytes < sizeof(ncclUniqueId))) return ETXB_ERR_INVALID_ARGUMENT;
  NcclApi* n = nccl_api();
  if (!n) return ETXB_ERR_NOT_READY;
  ncclUniqueId id;
  if (n->GetUniqueId(&id) != ncclSuccess) return ETXB_ERR_CUDA;
  memcpy(out_id, &id, sizeof(id));
  return ETXB_OK;
}

int etxb_comm_init(etxb_ctx* ctx, uint32_t world, uint32_t rank, const void* id, uint64_t bytes) {
  if (!ctx || !id || (bytes < sizeof(ncclUniqueId)) || (world == 0u) || (rank >= world)) return ETXB_ERR_INVALID_ARGUMENT;
  if (ctx->comm != nullptr) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "the context already has a communicator");
  if (ctx->target_pixel_size > 1u) return fail(ctx, ETXB_ERR_UNSUPPORTED, "etxb_comm_init: the coarse preview (film pixel size above 1) renders on one GPU");
  cudaSetDevice(ctx->device);
  if (int rc = comm_init_rank(ctx, &ctx->comm, world, rank, id)) return rc;
  ctx->rank = rank;
  ctx->world = world;
  CUDA_OK(ctx, ctx->comm_counts.alloc(world));
  CUDA_OK(ctx, create_priority_stream(&ctx->comm_stream));
  CUDA_OK(ctx, cudaEventCreateWithFlags(&ctx->comm_ev_in, cudaEventDisableTiming));
  CUDA_OK(ctx, cudaEventCreateWithFlags(&ctx->comm_ev_out, cudaEventDisableTiming));
  return ETXB_OK;
}

int etxb_comm_world(const etxb_ctx* ctx, uint32_t* world, uint32_t* rank) {
  if (!ctx || !world || !rank) return ETXB_ERR_INVALID_ARGUMENT;
  *world = (ctx->comm != nullptr) ? ctx->world : 1u;
  *rank = (ctx->comm != nullptr) ? ctx->rank : 0u;
  return ETXB_OK;
}

// Collective: every rank calls it.  The disjoint camera tiles are summed on rank 0 (ncclReduce of the float4 film); the light layer is already
// complete on every rank.  On rank 0 `dst_rgba` (may be null elsewhere) receives the layer like etxb_read_film.
int etxb_comm_reduce_film(etxb_ctx* ctx, uint32_t layer, float* dst_rgba, uint64_t dst_bytes) {
  if (!ctx || (layer == ETXB_FILM_LIGHT_ITERATION) || (layer > ETXB_FILM_CAMERA_ADAPTIVE)) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (ctx->comm == nullptr) return etxb_read_film(ctx, layer, dst_rgba, dst_bytes);
  if (int rc = ctx_drain(ctx)) return rc;
  NcclApi* n = nccl_api();
  cudaSetDevice(ctx->device);
  const size_t px = ctx->path_count;
  if (ctx->film_reduced.count < px) CUDA_OK(ctx, ctx->film_reduced.alloc(px));
  // the tiled layers: each rank holds its own tiles and zeros elsewhere (k_pt_accumulate and k_film_adaptive_vcm write owned pixels only)
  const float4* tiles = ctx->film_camera.ptr;
  if ((layer == ETXB_FILM_NORMALS) || (layer == ETXB_FILM_ALBEDO)) {
    if (int rc = pt_ensure_film(ctx)) return rc;
    tiles = (layer == ETXB_FILM_NORMALS) ? ctx->film_normals.ptr : ctx->film_albedo.ptr;
  } else if (layer == ETXB_FILM_CAMERA_ADAPTIVE) {
    if (int rc = film_ensure_adaptive(ctx)) return rc;
    tiles = ctx->film_adaptive.ptr;
  }
  if (layer != ETXB_FILM_LIGHT)
    NCCL_OK(ctx, n->Reduce(tiles, ctx->film_reduced.ptr, px * 4u, ncclFloat, ncclSum, 0, ctx->comm, ctx->stream));
  if (ctx->rank != 0u) {
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return ETXB_OK;
  }
  if (!dst_rgba || (dst_bytes < px * 16u)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "film buffer too small");
  const float4* src = (layer == ETXB_FILM_LIGHT) ? ctx->film_light.ptr : ctx->film_reduced.ptr;
  if (layer == ETXB_FILM_NORMALS) {  // etxb_read_film's read-out (Film::layer: n * 0.5 + 0.5)
    k_film_layer_normals<<<blocks_for(ctx->path_count, 256), 256, 0, ctx->stream>>>(ctx->film_reduced.ptr, ctx->film_out.ptr, ctx->path_count);
    ctx->kernel_launches += 1;
    src = ctx->film_out.ptr;
  }
  if (layer == ETXB_FILM_RESULT) {
    FilmBuffers film = {ctx->film_reduced.ptr, ctx->film_light.ptr, ctx->film_light_iteration.ptr, ctx->width, ctx->height};
    k_film_resolve<<<blocks_for(ctx->path_count, 256), 256, 0, ctx->stream>>>(film, ctx->film_out.ptr);
    ctx->kernel_launches += 1;
    src = ctx->film_out.ptr;
  }
  CUDA_OK(ctx, cudaMemcpyAsync(dst_rgba, src, px * 16u, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  return ETXB_OK;
}

int etxb_poll(etxb_ctx* ctx, etxb_status* status) {
  if (!ctx || !status) return ETXB_ERR_INVALID_ARGUMENT;
  memset(status, 0, sizeof(*status));
  status->last_iteration_time = ctx->last_iteration_time;
  status->total_time = ctx->total_time;
  status->completed_iterations = ctx->completed;
  status->current_iteration = ctx->iteration;
  {
    std::lock_guard<std::mutex> lock(ctx->worker_m);
    status->iteration_in_flight = ((ctx->worker_queued > 0) || ctx->worker_busy) ? 1u : 0u;
  }
  status->light_vertices = ctx->last_light_vertices;
  status->overflow = ctx->overflow_flag;
  return ETXB_OK;
}

int etxb_wait(etxb_ctx* ctx) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = ctx_drain(ctx)) return rc;
  cudaSetDevice(ctx->device);
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  return ETXB_OK;
}

// CPUVCM::stop (vcm_cpu.cxx:278-288): Immediate drops the queued iterations (the one in flight still completes: its film update is atomic per
// iteration), WaitForCompletion lets everything queued finish
int etxb_stop(etxb_ctx* ctx, int wait_for_iteration) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  if (!wait_for_iteration) {
    std::lock_guard<std::mutex> lock(ctx->worker_m);
    ctx->worker_queued = 0;
  }
  return etxb_wait(ctx);
}

int etxb_film_size(const etxb_ctx* ctx, uint32_t* width, uint32_t* height) {
  if (!ctx || !width || !height) return ETXB_ERR_INVALID_ARGUMENT;
  *width = ctx->width;
  *height = ctx->height;
  return ETXB_OK;
}

int etxb_read_film(etxb_ctx* ctx, uint32_t layer, float* dst_rgba, uint64_t dst_bytes) {
  if (!ctx || !dst_rgba) return ETXB_ERR_INVALID_ARGUMENT;
  size_t n = ctx->path_count;
  if (ctx->scene_ready && (dst_bytes < n * 16)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "film buffer too small");
  const float4* src = nullptr;
  if (int rc = film_layer_source(ctx, layer, &src)) return rc;
  CUDA_OK(ctx, cudaMemcpyAsync(dst_rgba, src, n * 16, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  return ETXB_OK;
}

// Film::denoise (film.cxx:420-423) with the filter of DESIGN §13 in place of OpenImageDenoise: Result or Camera into the Denoised layer
int etxb_denoise(etxb_ctx* ctx, uint32_t layer) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  if ((layer != ETXB_FILM_RESULT) && (layer != ETXB_FILM_CAMERA)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "etxb_denoise: layer %u is neither Result nor Camera", layer);
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if ((ctx->comm != nullptr) || (ctx->world > 1u)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "etxb_denoise: the film of a context with pixel tiles holds only its own tiles");
  if (int rc = ctx_drain(ctx)) return rc;
  cudaSetDevice(ctx->device);
  const size_t n = ctx->path_count;
  const bool pt = ctx->integrator == ETXB_INTEGRATOR_PT;
  if ((ctx->film_adaptive.count != n) || (pt && (ctx->pt_info.count != n)) || (!pt && (ctx->completed < 2u)))
    return fail(ctx, ETXB_ERR_NOT_READY, "etxb_denoise: fewer than two iterations on this film");
  const float4* color = nullptr;
  if (int rc = film_layer_source(ctx, layer, &color)) return rc;
  if (ctx->film_denoised.count != n) {
    CUDA_OK(ctx, ctx->film_denoised.alloc(n));
    CUDA_OK(ctx, cudaMemsetAsync(ctx->film_denoised.ptr, 0, n * 16, ctx->stream));  // zeros if the variance estimate refuses
  }
  // the path tracer's per-pixel sample counts and its guides; the VCM: every pixel has `completed` samples and, as in the reference (whose VCM
  // writes zero normals and albedo), no guides
  DenoiseInputs in = {color, ctx->film_camera.ptr, ctx->film_adaptive.ptr, pt ? ctx->pt_info.ptr : nullptr, ctx->completed,
    pt ? ctx->film_normals.ptr : nullptr, pt ? ctx->film_albedo.ptr : nullptr, ctx->width, ctx->height};
  return run_denoise(ctx, in, ctx->film_denoised.ptr, nullptr);
}

// The tone-mapped 8-bit frame the application shows and exports (app.cxx:268-282): computed on the device, 4 bytes per pixel cross the bus.
int etxb_read_film_ldr(etxb_ctx* ctx, uint32_t layer, float exposure, uint8_t* dst_rgba8, uint64_t dst_bytes) {
  if (!ctx || !dst_rgba8) return ETXB_ERR_INVALID_ARGUMENT;
  size_t n = ctx->path_count;
  if (ctx->scene_ready && (dst_bytes < n * 4)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "film buffer too small");
  const float4* src = nullptr;
  if (int rc = film_layer_source(ctx, layer, &src)) return rc;
  // a buffer of its own: a preview may be taken while an iteration is in flight on this stream, whose scratch buffers must stay untouched
  if (ctx->film_ldr.count != n) CUDA_OK(ctx, ctx->film_ldr.alloc(n));
  uint32_t* packed = ctx->film_ldr.ptr;
  k_film_tonemap<<<blocks_for(ctx->path_count, 256), 256, 0, ctx->stream>>>(src, packed, ctx->path_count, exposure);
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaMemcpyAsync(dst_rgba8, packed, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  return ETXB_OK;
}

// RTApplication::on_save_image_selected (app.cxx:261-295): mode 0 = the float layer as OpenEXR, mode 1 = the tone-mapped layer as PNG
int etxb_save_film(etxb_ctx* ctx, uint32_t layer, const char* file_name, uint32_t mode, float exposure) {
  if (!ctx || !file_name || (mode > ETXB_SAVE_PNG_TONEMAPPED)) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (int rc = ctx_drain(ctx)) return rc;
  const size_t n = ctx->path_count;
  int rc = ETXB_OK;
  if (mode == ETXB_SAVE_EXR) {
    std::vector<float> pixels(n * 4u);
    if ((rc = etxb_read_film(ctx, layer, pixels.data(), pixels.size() * 4u)) != ETXB_OK) return rc;
    rc = etxb_write_exr(file_name, pixels.data(), ctx->width, ctx->height);
  } else {
    std::vector<uint8_t> pixels(n * 4u);
    if ((rc = etxb_read_film_ldr(ctx, layer, exposure, pixels.data(), pixels.size())) != ETXB_OK) return rc;
    rc = etxb_write_png(file_name, pixels.data(), ctx->width, ctx->height);
  }
  return (rc == ETXB_OK) ? ETXB_OK : fail(ctx, rc, "could not write %s", file_name);
}

int etxb_get_counters(etxb_ctx* ctx, etxb_counters* out) {
  if (!ctx || !out) return ETXB_ERR_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  DeviceCounters c;
  CUDA_OK(ctx, cudaMemcpyAsync(&c, ctx->counters.ptr, sizeof(c), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  out->rays_closest = c.rays_closest;
  out->rays_shadow = c.rays_shadow;
  out->nodes_visited = c.nodes;
  out->tris_tested = c.tris;
  out->bounces_light = c.bounces_light;
  out->bounces_camera = c.bounces_camera;
  out->light_vertices = c.light_vertices;
  out->connections = c.connections;
  out->merge_queries = c.merge_queries;
  out->merge_candidates = c.merge_candidates;
  out->merge_accepts = c.merge_accepts;
  out->splats = c.splats;
  out->kernel_launches = ctx->kernel_launches;
  out->nodes_closest = c.nodes_closest;
  out->tris_closest = c.tris_closest;
  return ETXB_OK;
}

int etxb_get_kernel_times(etxb_ctx* ctx, const char** names, float* ms, uint32_t* launches, uint32_t capacity) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  uint32_t n = std::min<uint32_t>(capacity, K_COUNT);
  for (uint32_t i = 0; i < n; ++i) {
    if (names) names[i] = kKernelNames[i];
    if (ms) ms[i] = ctx->kernel_ms[i];
    if (launches) launches[i] = ctx->kernel_count[i];
  }
  return int(K_COUNT);
}

namespace {
// the device buffer behind an ETXB_BUF_* id that etxb_read_buffer copies as it is
int buffer_pointer(etxb_ctx* ctx, uint32_t buffer_id, void** out_ptr, uint64_t* out_bytes) {
  size_t n = ctx->path_count;
  switch (buffer_id) {
    case ETXB_BUF_LIGHT_PATH_COUNT: *out_ptr = ctx->lv_count.ptr; *out_bytes = n * 4; break;
    case ETXB_BUF_LIGHT_PATH_OFFSET: *out_ptr = ctx->lp_offset.ptr; *out_bytes = n * 4; break;
    case ETXB_BUF_LIGHT_PATH_WAVELENGTH: *out_ptr = ctx->wavelength.ptr; *out_bytes = n * 4; break;
    case ETXB_BUF_LIGHT_SAMPLER: *out_ptr = ctx->sampler_end_light.ptr; *out_bytes = n * 4; break;
    case ETXB_BUF_CAMERA_SAMPLER: *out_ptr = ctx->sampler_end_camera.ptr; *out_bytes = n * 4; break;
    case ETXB_BUF_FILM_LIGHT_ITERATION: *out_ptr = ctx->film_light_iteration.ptr; *out_bytes = n * 16; break;
    case ETXB_BUF_FILM_CAMERA: *out_ptr = ctx->film_camera.ptr; *out_bytes = n * 16; break;
    case ETXB_BUF_FILM_LIGHT: *out_ptr = ctx->film_light.ptr; *out_bytes = n * 16; break;
    case ETXB_BUF_PHOTON_RECORDS: *out_ptr = ctx->lv_final.ptr; *out_bytes = size_t(ctx->last_light_vertices) * sizeof(LightVertexRec); break;
    case ETXB_BUF_CAMERA_GATHERED: *out_ptr = ctx->camera_value.ptr; *out_bytes = n * 16; break;
    case ETXB_BUF_PIXEL_INFO:
      if (ctx->pt_info.count != n) return fail(ctx, ETXB_ERR_NOT_READY, "the path tracer has not run on this film");
      *out_ptr = ctx->pt_info.ptr; *out_bytes = n * 4; break;
    case ETXB_BUF_PIXEL_ERROR:
      if (ctx->pt_error.count != n) return fail(ctx, ETXB_ERR_NOT_READY, "the path tracer has not run on this film");
      *out_ptr = ctx->pt_error.ptr; *out_bytes = n * 4; break;
    case ETXB_BUF_BVH_NODES:
    case ETXB_BUF_BVH_TRIS:
    case ETXB_BUF_WIDE_NODES:
      if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
      if (buffer_id == ETXB_BUF_BVH_NODES) {
        *out_ptr = ctx->bvh_nodes.ptr; *out_bytes = size_t(ctx->dscene.bvh_node_count) * sizeof(BvhNode);
      } else if (buffer_id == ETXB_BUF_BVH_TRIS) {
        *out_ptr = ctx->bvh_tris.ptr; *out_bytes = ctx->bvh_tris.bytes();
      } else {
        *out_ptr = const_cast<WideNode*>(ctx->dscene.wide_nodes); *out_bytes = size_t(ctx->dscene.wide_node_count) * sizeof(WideNode);
      }
      break;
    default: return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "buffer %u has no direct device pointer", buffer_id);
  }
  return ETXB_OK;
}
}  // namespace

int etxb_read_buffer(etxb_ctx* ctx, uint32_t buffer_id, void* dst, uint64_t dst_bytes, uint64_t* out_bytes) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = ctx_drain(ctx)) return rc;
  cudaSetDevice(ctx->device);
  size_t lv = ctx->last_light_vertices;
  if (buffer_id == ETXB_BUF_LV_POS || buffer_id == ETXB_BUF_LV_THROUGHPUT || buffer_id == ETXB_BUF_LV_MIS) {
    uint64_t need = lv * 12;
    if (out_bytes) *out_bytes = need;
    if (!dst) return ETXB_OK;
    if (dst_bytes < need) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "buffer too small");
    std::vector<LightVertexRec> host(lv);
    if (lv) CUDA_OK(ctx, cudaMemcpy(host.data(), ctx->lv_final.ptr, lv * sizeof(LightVertexRec), cudaMemcpyDeviceToHost));
    float* out = static_cast<float*>(dst);
    for (size_t i = 0; i < lv; ++i) {
      const LightVertexRec& r = host[i];
      if (buffer_id == ETXB_BUF_LV_POS) {
        out[i * 3 + 0] = r.pos_tri.x; out[i * 3 + 1] = r.pos_tri.y; out[i * 3 + 2] = r.pos_tri.z;
      } else if (buffer_id == ETXB_BUF_LV_THROUGHPUT) {
        out[i * 3 + 0] = r.thr_dvcm.x; out[i * 3 + 1] = r.thr_dvcm.y; out[i * 3 + 2] = r.thr_dvcm.z;
      } else {
        out[i * 3 + 0] = r.thr_dvcm.w; out[i * 3 + 1] = r.wi_dvc.w; out[i * 3 + 2] = r.bc_dvm.w;
      }
    }
    return ETXB_OK;
  }
  void* ptr = nullptr;
  uint64_t bytes = 0;
  if (int rc = buffer_pointer(ctx, buffer_id, &ptr, &bytes)) return rc;
  if (buffer_id == ETXB_BUF_CAMERA_GATHERED) {
    uint64_t need = uint64_t(ctx->path_count) * 12;
    if (out_bytes) *out_bytes = need;
    if (!dst) return ETXB_OK;
    if (dst_bytes < need) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "buffer too small");
    std::vector<float4> host(ctx->path_count);
    CUDA_OK(ctx, cudaMemcpy(host.data(), ptr, bytes, cudaMemcpyDeviceToHost));
    float* out = static_cast<float*>(dst);
    for (size_t i = 0; i < host.size(); ++i) {
      out[i * 3 + 0] = host[i].x; out[i * 3 + 1] = host[i].y; out[i * 3 + 2] = host[i].z;
    }
    return ETXB_OK;
  }
  if (out_bytes) *out_bytes = bytes;
  if (!dst) return ETXB_OK;
  if (dst_bytes < bytes) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "buffer too small");
  if (bytes) CUDA_OK(ctx, cudaMemcpy(dst, ptr, bytes, cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

void* etxb_stream(etxb_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

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

// Test hook: etxb_denoise's kernels on host arrays (RGBA float per pixel, storage order; `counts` per pixel; guides may be null)
int etxb_debug_denoise(etxb_ctx* ctx, const float* color, const float* camera, const float* half, const uint32_t* counts, const float* normals, const float* albedo,
                       uint32_t width, uint32_t height, float* out, float* out_variance) {
  if (!ctx || !color || !camera || !half || !counts || !out || !width || !height) return ETXB_ERR_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  const size_t n = size_t(width) * height;
  DevBuf<float4> dc, df, dh, dn, da, dout, dvar;
  DevBuf<uint32_t> dcount;
  if (int rc = upload(ctx, dc, reinterpret_cast<const float4*>(color), n)) return rc;
  if (int rc = upload(ctx, df, reinterpret_cast<const float4*>(camera), n)) return rc;
  if (int rc = upload(ctx, dh, reinterpret_cast<const float4*>(half), n)) return rc;
  if (int rc = upload(ctx, dcount, counts, n)) return rc;
  if (normals)
    if (int rc = upload(ctx, dn, reinterpret_cast<const float4*>(normals), n)) return rc;
  if (albedo)
    if (int rc = upload(ctx, da, reinterpret_cast<const float4*>(albedo), n)) return rc;
  CUDA_OK(ctx, dout.alloc(n));
  CUDA_OK(ctx, dvar.alloc(n));
  DenoiseInputs in = {dc.ptr, df.ptr, dh.ptr, dcount.ptr, 0u, normals ? dn.ptr : nullptr, albedo ? da.ptr : nullptr, width, height};
  if (int rc = run_denoise(ctx, in, dout.ptr, dvar.ptr)) return rc;
  CUDA_OK(ctx, cudaMemcpy(out, dout.ptr, n * 16, cudaMemcpyDeviceToHost));
  if (out_variance) CUDA_OK(ctx, cudaMemcpy(out_variance, dvar.ptr, n * 16, cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

// Test hook: the noise estimate of `world` pixel-tile ranks on one device (layout in include/etx_b200.h).  Each rank's view holds its own pixels
// and zeros elsewhere, as a rank's buffers do; the all-reduce of pt_estimate_noise_levels is replaced by the same sum on the host.
int etxb_debug_noise_estimate(etxb_ctx* ctx, uint32_t width, uint32_t height, uint32_t world, float threshold, const float* camera, const float* adaptive,
                              const uint32_t* info_in, uint32_t* info_out, float* error_out, uint32_t* stats_out) {
  if (!ctx || !camera || !adaptive || !info_in || !info_out || !error_out || !stats_out || !width || !height || !world) return ETXB_ERR_INVALID_ARGUMENT;
  if (!(threshold >= 0.0f) || (uint64_t(width) * height > (1ull << 26)) || (world > 1024u)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "etxb_debug_noise_estimate: bad threshold, film size or world");
  if (int rc = ctx_drain(ctx)) return rc;
  cudaSetDevice(ctx->device);
  const size_t n = size_t(width) * height;
  const uint32_t words = noise_mask_words(width, height);
  struct RankBuffers {
    DevBuf<float4> camera, adaptive;
    DevBuf<uint32_t> info, mask;
    DevBuf<float> error;
  };
  std::vector<RankBuffers> ranks(world);
  std::vector<NoiseView> views(world);
  std::vector<float4> cam(n), ada(n);
  std::vector<uint32_t> inf(n);
  auto owner = [&](size_t i) { return tile_rank(width, uint32_t(i % width), height - 1u - uint32_t(i / width), world); };
  const float4* camera4 = reinterpret_cast<const float4*>(camera);
  const float4* adaptive4 = reinterpret_cast<const float4*>(adaptive);
  for (uint32_t r = 0; r < world; ++r) {
    for (size_t i = 0; i < n; ++i) {
      const bool mine = owner(i) == r;
      cam[i] = mine ? camera4[i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      ada[i] = mine ? adaptive4[i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
      inf[i] = mine ? info_in[i] : 0u;
    }
    RankBuffers& b = ranks[r];
    if (int rc = upload(ctx, b.camera, cam.data(), n)) return rc;
    if (int rc = upload(ctx, b.adaptive, ada.data(), n)) return rc;
    if (int rc = upload(ctx, b.info, inf.data(), n)) return rc;
    CUDA_OK(ctx, b.error.alloc(n));
    CUDA_OK(ctx, cudaMemsetAsync(b.error.ptr, 0, n * 4, ctx->stream));
    CUDA_OK(ctx, b.mask.alloc(size_t(words) + kNoiseStats));
    views[r] = {{b.camera.ptr, nullptr, nullptr, width, height}, {nullptr, nullptr, b.adaptive.ptr, b.info.ptr, b.error.ptr}, b.mask.ptr, r, world};
    if (int rc = noise_level_pass(ctx, views[r], threshold)) return rc;
  }
  std::vector<uint32_t> sum(size_t(words) + kNoiseStats, 0u), part(size_t(words) + kNoiseStats);
  float error_sum = 0.0f;
  for (uint32_t r = 0; r < world; ++r) {
    CUDA_OK(ctx, cudaMemcpyAsync(part.data(), ranks[r].mask.ptr, part.size() * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    for (size_t j = 0; j < size_t(words) + kNoiseStatProcessed + 1u; ++j) sum[j] += part[j];
    float e = 0.0f;
    memcpy(&e, &part[words + kNoiseStatError], 4);
    error_sum += e;
  }
  memcpy(&sum[words + kNoiseStatError], &error_sum, 4);
  for (uint32_t r = 0; r < world; ++r) {
    CUDA_OK(ctx, cudaMemcpyAsync(ranks[r].mask.ptr, sum.data(), sum.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    if (int rc = noise_dilate_pass(ctx, views[r])) return rc;
  }
  CUDA_OK(ctx, cudaGetLastError());
  std::vector<float> err(n);
  for (uint32_t r = 0; r < world; ++r) {
    CUDA_OK(ctx, cudaMemcpyAsync(inf.data(), ranks[r].info.ptr, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(err.data(), ranks[r].error.ptr, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < n; ++i) {
      if (owner(i) != r) continue;
      info_out[i] = inf[i];
      error_out[i] = err[i];
    }
  }
  stats_out[0] = sum[words + kNoiseStatConverged];
  stats_out[1] = sum[words + kNoiseStatError];
  return ETXB_OK;
}

// Test hook: the vertex closures of dclosure.cuh, query by query (layout and outputs in include/etx_b200.h)
int etxb_debug_closure_eval(etxb_ctx* ctx, const etxb_closure_query* queries, uint32_t count, uint32_t repetitions, double* out) {
  if (!ctx || !queries || !out || (repetitions == 0)) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (count == 0) return ETXB_OK;
  for (uint32_t i = 0; i < count; ++i) {
    if (queries[i].material >= ctx->materials.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "closure query material index out of range");
  }
  cudaSetDevice(ctx->device);
  DevBuf<etxb_closure_query> d_queries;
  DevBuf<double> d_out;
  if (int rc = upload(ctx, d_queries, queries, count)) return rc;
  CUDA_OK(ctx, d_out.alloc(size_t(count) * ETXB_CLOSURE_STATS));
  if (ctx->spectral) {
    k_debug_closure<true><<<blocks_for(count, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  } else {
    k_debug_closure<false><<<blocks_for(count, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  }
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaGetLastError());
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(out, d_out.ptr, d_out.bytes(), cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

// Test hook: bsdf_sample of dbsdf.cuh, query by query and repetition by repetition (layout and modes in include/etx_b200.h)
int etxb_debug_bsdf_sample(etxb_ctx* ctx, const etxb_sample_query* queries, uint32_t count, uint32_t repetitions, etxb_sample_result* out) {
  if (!ctx || !queries || !out || (repetitions == 0)) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (count == 0) return ETXB_OK;
  if (uint64_t(count) * repetitions > 0x7fffffffull) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "%u queries x %u repetitions exceed 2^31 samples", count, repetitions);
  for (uint32_t i = 0; i < count; ++i) {
    if (queries[i].material >= ctx->materials.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "sample query %u: material index out of range", i);
    if (queries[i].mode > 1u) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "sample query %u: mode must be 0 or 1", i);
  }
  cudaSetDevice(ctx->device);
  const uint32_t total = count * repetitions;
  DevBuf<etxb_sample_query> d_queries;
  DevBuf<etxb_sample_result> d_out;
  if (int rc = upload(ctx, d_queries, queries, count)) return rc;
  CUDA_OK(ctx, d_out.alloc(total));
  if (ctx->spectral) {
    k_debug_bsdf_sample<true><<<blocks_for(total, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  } else {
    k_debug_bsdf_sample<false><<<blocks_for(total, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  }
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaGetLastError());
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(out, d_out.ptr, d_out.bytes(), cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

// Test hook: the emitter routines of dvcm.cuh, query by query and repetition by repetition (layout and ops in include/etx_b200.h)
int etxb_debug_emitter(etxb_ctx* ctx, const etxb_emitter_query* queries, uint32_t count, uint32_t repetitions, etxb_emitter_result* out) {
  if (!ctx || !queries || !out || (repetitions == 0)) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (count == 0) return ETXB_OK;
  if (uint64_t(count) * repetitions > 0x7fffffffull) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "%u queries x %u repetitions exceed 2^31 samples", count, repetitions);
  if (ctx->emitters.count == 0) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "the scene has no emitter");
  for (uint32_t i = 0; i < count; ++i) {
    if (queries[i].op > ETXB_EMITTER_RADIANCE) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter query %u: op must be 0 to 3", i);
    const bool indexed = (queries[i].op == ETXB_EMITTER_SAMPLE_IN) || (queries[i].op == ETXB_EMITTER_RADIANCE);
    if (indexed && (queries[i].emitter >= ctx->emitters.count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "emitter query %u: emitter index out of range", i);
  }
  cudaSetDevice(ctx->device);
  const uint32_t total = count * repetitions;
  DevBuf<etxb_emitter_query> d_queries;
  DevBuf<etxb_emitter_result> d_out;
  if (int rc = upload(ctx, d_queries, queries, count)) return rc;
  CUDA_OK(ctx, d_out.alloc(total));
  if (ctx->spectral) {
    k_debug_emitter<true><<<blocks_for(total, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  } else {
    k_debug_emitter<false><<<blocks_for(total, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  }
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaGetLastError());
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(out, d_out.ptr, d_out.bytes(), cudaMemcpyDeviceToHost));
  return ETXB_OK;
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
  if (!ctx || !queries || !out || (repetitions == 0)) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (count == 0) return ETXB_OK;
  if (uint64_t(count) * repetitions > 0x7fffffffull) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "%u queries x %u repetitions exceed 2^31 samples", count, repetitions);
  cudaSetDevice(ctx->device);
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
  const uint32_t total = count * repetitions;
  DevBuf<etxb_medium_query> d_queries;
  DevBuf<etxb_medium_result> d_out;
  if (int rc = upload(ctx, d_queries, queries, count)) return rc;
  CUDA_OK(ctx, d_out.alloc(total));
  if (ctx->spectral) {
    k_debug_medium<true><<<blocks_for(total, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  } else {
    k_debug_medium<false><<<blocks_for(total, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  }
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaGetLastError());
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(out, d_out.ptr, d_out.bytes(), cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

// Test hook: the subsurface routines of dsss.cuh, query by query and repetition by repetition (layout and ops in include/etx_b200.h).
// Every loop they run is bounded (a traversal of the tree, at most 1024 random-walk steps), so the checks are on indices and finite inputs.
int etxb_debug_subsurface(etxb_ctx* ctx, const etxb_subsurface_query* queries, uint32_t count, uint32_t repetitions, etxb_subsurface_result* out) {
  if (!ctx || !queries || !out || (repetitions == 0)) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (count == 0) return ETXB_OK;
  if (uint64_t(count) * repetitions > 0x7fffffffull) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "%u queries x %u repetitions exceed 2^31 samples", count, repetitions);
  cudaSetDevice(ctx->device);
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
  const uint32_t total = count * repetitions;
  DevBuf<etxb_subsurface_query> d_queries;
  DevBuf<etxb_subsurface_result> d_out;
  if (int rc = upload(ctx, d_queries, queries, count)) return rc;
  CUDA_OK(ctx, d_out.alloc(total));
  CUDA_OK(ctx, cudaMemsetAsync(d_out.ptr, 0, d_out.bytes(), ctx->stream));  // the kernel writes only the fields its op names
  if (ctx->spectral) {
    k_debug_subsurface<true><<<blocks_for(total, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  } else {
    k_debug_subsurface<false><<<blocks_for(total, 128), 128, 0, ctx->stream>>>(ctx->dscene, d_queries.ptr, count, repetitions, d_out.ptr);
  }
  ctx->kernel_launches += 1;
  CUDA_OK(ctx, cudaGetLastError());
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  CUDA_OK(ctx, cudaMemcpy(out, d_out.ptr, d_out.bytes(), cudaMemcpyDeviceToHost));
  return ETXB_OK;
}

// Test hook: the queue sizes from which the passes take their large-queue branches (NULL = the defaults), and what ran since etxb_begin
int etxb_debug_set_thresholds(etxb_ctx* ctx, const etxb_debug_thresholds* thresholds) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  const etxb_debug_thresholds t = thresholds ? *thresholds : kDefaultThresholds;
  if ((t.merge_qpw > 32u) || (t.merge_qpw & (t.merge_qpw - 1u))) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "merge_qpw must be 0, 1, 2, 4, 8, 16 or 32");
  if (t.merge_sort_min_queries < t.tail_queue) {
    // below tail_queue the host enqueues bounces on a stale queue size, and the gather's sort would take in slots past the count
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "merge_sort_min_queries (%u) must not be below tail_queue (%u)", t.merge_sort_min_queries, t.tail_queue);
  }
  ctx_drain(ctx);
  ctx->thresholds = t;
  return ETXB_OK;
}

int etxb_debug_get_branch_counts(etxb_ctx* ctx, etxb_debug_branch_counts* out) {
  if (!ctx || !out) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = ctx_drain(ctx)) return rc;
  *out = ctx->branch_counts;
  return ETXB_OK;
}

// Test hook: the photon gather query by query (layout and outputs in include/etx_b200.h)
int etxb_debug_merge(etxb_ctx* ctx, const void* records, uint32_t record_count, const float* light_wavelengths, const etxb_merge_query* queries, uint32_t count,
                     etxb_merge_result* out, etxb_merge_grid* grid) {
  if (!ctx || (record_count && !records) || !light_wavelengths || (count && (!queries || !out)) || !grid) return ETXB_ERR_INVALID_ARGUMENT;
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if (count > ctx->path_count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "%u merge queries exceed the %u paths of the context", count, ctx->path_count);
  if (record_count > ctx->lv_capacity) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "%u light vertices exceed the pool capacity %u", record_count, ctx->lv_capacity);
  const LightVertexRec* recs = static_cast<const LightVertexRec*>(records);
  for (uint32_t k = 0; k < record_count; ++k) {
    if (recs[k].ids.z >= ctx->path_count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "light vertex %u: path index out of range", k);
  }
  for (uint32_t k = 0; k < count; ++k) {
    if (queries[k].tri >= ctx->triangles.count) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "merge query %u: triangle index out of range", k);
    if ((queries[k].medium != ETXB_INVALID_INDEX) && (queries[k].medium >= ctx->dscene.medium_count)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "merge query %u: medium index out of range", k);
  }
  if (int rc = ctx_drain(ctx)) return rc;
  cudaSetDevice(ctx->device);
  if (record_count) CUDA_OK(ctx, cudaMemcpyAsync(ctx->lv_final.ptr, records, size_t(record_count) * sizeof(LightVertexRec), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_OK(ctx, cudaMemcpyAsync(ctx->wavelength.ptr, light_wavelengths, size_t(ctx->path_count) * 4u, cudaMemcpyHostToDevice, ctx->stream));
  DeviceCounters before = {}, after = {};
  CUDA_OK(ctx, cudaMemcpyAsync(&before, ctx->counters.ptr, sizeof(before), cudaMemcpyDeviceToHost, ctx->stream));
  DevBuf<etxb_merge_query> d_queries;
  DevBuf<float4> d_pos_nrm;
  if (int rc = upload(ctx, d_queries, queries, count)) return rc;
  CUDA_OK(ctx, d_pos_nrm.alloc(2u * std::max<uint32_t>(count, 1u)));
  int rc = ctx->spectral ? debug_merge<true>(ctx, record_count, d_queries.ptr, count, d_pos_nrm.ptr) : debug_merge<false>(ctx, record_count, d_queries.ptr, count, d_pos_nrm.ptr);
  if (rc) return rc;
  CUDA_OK(ctx, cudaGetLastError());
  std::vector<float4> merged(count), pos_nrm(2u * size_t(count));
  std::vector<uint4> misc(count);
  if (count) {
    CUDA_OK(ctx, cudaMemcpyAsync(merged.data(), ctx->merged.ptr, size_t(count) * 16u, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(misc.data(), ctx->misc.ptr, size_t(count) * 16u, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(pos_nrm.data(), d_pos_nrm.ptr, size_t(count) * 32u, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CUDA_OK(ctx, cudaMemcpyAsync(&after, ctx->counters.ptr, sizeof(after), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  for (uint32_t k = 0; k < count; ++k) {
    etxb_merge_result& r = out[k];
    r = {};
    r.merged[0] = merged[k].x, r.merged[1] = merged[k].y, r.merged[2] = merged[k].z;
    r.seed = misc[k].x;
    r.pos[0] = pos_nrm[2 * k].x, r.pos[1] = pos_nrm[2 * k].y, r.pos[2] = pos_nrm[2 * k].z;
    r.nrm[0] = pos_nrm[2 * k + 1].x, r.nrm[1] = pos_nrm[2 * k + 1].y, r.nrm[2] = pos_nrm[2 * k + 1].z;
  }
  const GridData& g = ctx->grid;
  *grid = {};
  grid->bbox_min[0] = g.bbox_min.x, grid->bbox_min[1] = g.bbox_min.y, grid->bbox_min[2] = g.bbox_min.z;
  grid->bbox_max[0] = g.bbox_max.x, grid->bbox_max[1] = g.bbox_max.y, grid->bbox_max[2] = g.bbox_max.z;
  grid->cell_size = g.cell_size;
  grid->radius_squared = g.radius_squared;
  grid->hash_table_mask = g.hash_table_mask;
  grid->photon_count = g.photon_count;
  grid->merge_queries = after.merge_queries - before.merge_queries;
  grid->merge_candidates = after.merge_candidates - before.merge_candidates;
  grid->merge_accepts = after.merge_accepts - before.merge_accepts;
  return ETXB_OK;
}

// ---- iterations in flight (etxb_group) ----------------------------------------------------------------------------------------------------
int etxb_group_create(etxb_group** out, const etxb_device_config* cfg, uint32_t lanes) {
  if (!out || (lanes == 0) || (lanes > kMaxLanes)) return ETXB_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  auto* grp = new etxb_group();
  grp->device = cfg ? cfg->device_index : 0;
  for (uint32_t l = 0; l < lanes; ++l) {
    etxb_ctx* ctx = nullptr;
    int rc = etxb_create(&ctx, cfg);
    if (rc != ETXB_OK) {
      for (auto* c : grp->lanes) etxb_destroy(c);
      delete grp;
      return rc;
    }
    ctx->group_lane = true;
    grp->lanes.push_back(ctx);
  }
  grp->plan.queues.resize(lanes);
  grp->plan.lane_queue.assign(lanes, 0u);
  cudaSetDevice(grp->device);
  create_priority_stream(&grp->stream);  // the frame combine / reduce
  for (uint32_t l = 0; l < lanes; ++l) grp->workers.emplace_back(group_worker, grp, l);
  *out = grp;
  return ETXB_OK;
}

void etxb_group_destroy(etxb_group* grp) {
  if (!grp) return;
  {
    std::lock_guard<std::mutex> lock(grp->m);
    grp->quit = true;
  }
  grp->cv_work.notify_all();
  for (auto& w : grp->workers) w.join();
  cudaSetDevice(grp->device);
  if (grp->reduce_comm != nullptr) {
    if (NcclApi* n = nccl_api()) n->CommDestroy(grp->reduce_comm);
  }
  if (grp->stream) cudaStreamDestroy(grp->stream);
  for (auto* c : grp->lanes) etxb_destroy(c);
  delete grp;
}

uint32_t etxb_group_lanes(const etxb_group* grp) { return grp ? uint32_t(grp->lanes.size()) : 0u; }
etxb_ctx* etxb_group_lane(etxb_group* grp, uint32_t lane) { return (grp && (lane < grp->lanes.size())) ? grp->lanes[lane] : nullptr; }
const char* etxb_group_last_error(const etxb_group* grp) { return grp ? grp->error_text.c_str() : "null group"; }

int etxb_group_wait(etxb_group* grp) {
  if (!grp) return ETXB_ERR_INVALID_ARGUMENT;
  std::unique_lock<std::mutex> lock(grp->m);
  grp->cv_idle.wait(lock, [&] { return group_idle(grp); });
  return grp->error;
}

int etxb_group_begin(etxb_group* grp, uint32_t first_iteration) {
  if (!grp) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = etxb_group_wait(grp)) return rc;
  for (auto* c : grp->lanes)
    if (int rc = etxb_begin(c, first_iteration)) return rc;
  std::lock_guard<std::mutex> lock(grp->m);
  grp->first_iteration = first_iteration;
  grp->taken = 0;
  plan_clear(grp->plan);
  grp->plan.split_part = grp->plan.split_parts = 0;
  grp->busy_seconds = 0.0;
  grp->error = ETXB_OK;
  grp->error_text.clear();
  return ETXB_OK;
}

int etxb_group_set_film_pixel_size(etxb_group* grp, uint32_t size) {
  if (!grp) return ETXB_ERR_INVALID_ARGUMENT;
  if ((size > 1u) && ((grp->plan.mode != GroupMode::local) || (grp->reduce_comm != nullptr)))
    return group_refuse(grp, "etxb_group_set_film_pixel_size: a group with communicators renders film pixels in tiles or parts; the coarse preview renders on one GPU", ETXB_ERR_UNSUPPORTED);
  if (int rc = etxb_group_wait(grp)) return rc;
  for (auto* c : grp->lanes) {
    if (int rc = etxb_set_film_pixel_size(c, size)) {
      std::lock_guard<std::mutex> lock(grp->m);
      grp->error_text = etxb_last_error(c);
      return rc;
    }
  }
  return ETXB_OK;
}

int etxb_group_update_scene(etxb_group* grp, const void* scene_blob, uint64_t scene_bytes, const void* camera_blob, uint64_t camera_bytes, etxb_update_info* info) {
  const auto t0 = std::chrono::steady_clock::now();
  if (info) memset(info, 0, sizeof(*info));
  if (!grp || !scene_blob || !camera_blob) return ETXB_ERR_INVALID_ARGUMENT;
  etxb_ctx* first = grp->lanes[0];
  auto refuse = [&](int rc) {
    std::lock_guard<std::mutex> lock(grp->m);
    grp->error_text = etxb_last_error(first);
    return rc;
  };
  bool comm = grp->plan.mode != GroupMode::local;
  for (auto* c : grp->lanes) comm = comm || (c->comm != nullptr);
  if (comm) return refuse(fail(first, ETXB_ERR_UNSUPPORTED, "etxb_group_update_scene: a group with communicators takes a new scene through etxb_upload_scene on each lane"));
  if (int rc = check_scene_args(first, scene_bytes, camera_bytes)) return refuse(rc);
  if (int rc = etxb_group_wait(grp)) return rc;
  const etxb_scene& s = *static_cast<const etxb_scene*>(scene_blob);
  const etxb_camera& cam = *static_cast<const etxb_camera*>(camera_blob);
  cudaSetDevice(grp->device);
  // hashed and validated once; a new geometry's BVH is built once, and its depth checked, before any lane changes
  ScenePrep p;
  if (int rc = prepare_scene(first, s, cam, p)) return refuse(rc);
  for (auto* c : grp->lanes)
    if (!geometry_kept(c, p, c->scene_ready))
      if (int rc = prepare_bvh(first, s, p)) return refuse(rc);
  uint32_t kept = ~0u;
  for (size_t l = 0; l < grp->lanes.size(); ++l) {
    etxb_ctx* c = grp->lanes[l];
    etxb_update_info lane = {};
    ctx_drain(c);
    if (int rc = commit_scene(c, s, cam, p, c->scene_ready, &lane)) {
      std::lock_guard<std::mutex> lock(grp->m);
      grp->error_text = etxb_last_error(c);
      return rc;
    }
    kept &= lane.kept;
    if (info && (l == 0)) *info = lane;
  }
  if (info) {
    info->kept = kept;  // what every lane kept; the image and grid counts are lane 0's
    info->total_seconds = seconds_since(t0);
  }
  return etxb_group_begin(grp, 0);
}

int etxb_group_enqueue(etxb_group* grp, uint32_t iterations) {
  if (!grp) return ETXB_ERR_INVALID_ARGUMENT;
  {
    std::lock_guard<std::mutex> lock(grp->m);
    if (grp->error != ETXB_OK) return grp->error;
    if (iterations == 0) return ETXB_OK;
    if (group_idle(grp)) grp->busy_since = std::chrono::steady_clock::now();
    plan_enqueue(grp->plan, iterations);
  }
  grp->cv_work.notify_all();
  return ETXB_OK;
}

int etxb_group_poll(etxb_group* grp, etxb_status* status) {
  if (!grp || !status) return ETXB_ERR_INVALID_ARGUMENT;
  memset(status, 0, sizeof(*status));
  std::lock_guard<std::mutex> lock(grp->m);
  for (size_t l = 0; l < grp->lanes.size(); ++l) {
    etxb_ctx* c = grp->lanes[l];
    // a camera-split iteration is finished by several ranks: it counts where part 0 ran
    if (!((l == grp->plan.split_lane) && (grp->plan.split_part != 0u))) status->completed_iterations += c->completed;
    status->light_vertices = std::max(status->light_vertices, c->last_light_vertices);
    status->overflow |= c->overflow_flag;
  }
  status->current_iteration = grp->first_iteration + grp->taken;
  status->iteration_in_flight = group_idle(grp) ? 0u : 1u;
  status->last_iteration_time = grp->last_iteration_seconds;
  status->total_time = grp->busy_seconds;
  if (status->iteration_in_flight) status->total_time += std::chrono::duration<double>(std::chrono::steady_clock::now() - grp->busy_since).count();
  return ETXB_OK;
}

// Pixel tiles over several processes, `lanes` iterations in flight on each: ids = (lanes + 1) NCCL unique ids of 128 bytes, the same on every
// rank (lane l of every rank forms communicator l; the last one carries the frame reduce).  Collective.  Refused, before any NCCL call and so
// alike on every rank, on a group that already has a communicator or, for world >= 2, a split lane.
int etxb_group_comm_init(etxb_group* grp, uint32_t world, uint32_t rank, const void* ids, uint32_t id_count) {
  if (!grp || !ids || (world == 0u) || (rank >= world) || (id_count != grp->lanes.size() + 1u)) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = etxb_group_wait(grp)) return rc;
  if (grp->reduce_comm != nullptr) return group_refuse(grp, "etxb_group_comm_init: the group already has a communicator");
  if ((world > 1u) && (grp->plan.split_lane != 0xffffffffu)) return group_refuse(grp, "etxb_group_comm_init: pixel tiles and a split lane exclude each other");
  for (auto* c : grp->lanes) {
    if (c->target_pixel_size > 1u) return group_refuse(grp, "etxb_group_comm_init: the coarse preview (film pixel size above 1) renders on one GPU", ETXB_ERR_UNSUPPORTED);
    if ((world > 1u) && (c->integrator == ETXB_INTEGRATOR_PT))
      return group_refuse(grp, "etxb_group_comm_init: the path tracer does not run on a group in pixel-tile mode: each lane would keep its own per-pixel history", ETXB_ERR_UNSUPPORTED);
  }
  const uint8_t* bytes = static_cast<const uint8_t*>(ids);
  for (size_t l = 0; l < grp->lanes.size(); ++l) {
    if (int rc = etxb_comm_init(grp->lanes[l], world, rank, bytes + l * sizeof(ncclUniqueId), sizeof(ncclUniqueId))) {
      grp->error_text = etxb_last_error(grp->lanes[l]);
      return rc;
    }
  }
  cudaSetDevice(grp->device);
  if (int rc = comm_init_rank(grp->lanes[0], &grp->reduce_comm, world, rank, bytes + grp->lanes.size() * sizeof(ncclUniqueId))) return rc;
  std::lock_guard<std::mutex> lock(grp->m);
  grp->plan.mode = (world > 1u) ? GroupMode::tiles : GroupMode::local;
  grp->plan.world = world;
  grp->plan.rank = rank;
  grp->plan.enqueued = 0;
  return ETXB_OK;
}

// Test hook (no device needed): the queues of a `lanes`-lane group in `mode` (0 local, 1 tiles, 2 replicas) on rank `rank` of `world`, with its
// last lane reserved for camera-split iterations if `split_lane`, after etxb_group_enqueue(enqueues[0]), ..., (enqueues[count - 1]) — quads
// (queue, ordinal, part, parts) into out, queue by queue in the order the lanes pop them; returns their number.
int etxb_debug_group_plan(uint32_t mode, uint32_t lanes, uint32_t world, uint32_t rank, int split_lane, const uint32_t* enqueues, uint32_t count,
                          uint32_t* out_quads, uint32_t capacity) {
  if ((mode > uint32_t(GroupMode::replicas)) || (lanes == 0u) || (lanes > kMaxLanes) || (world == 0u) || (rank >= world) || (!enqueues && count) || !out_quads)
    return ETXB_ERR_INVALID_ARGUMENT;
  if (split_lane && ((lanes < 2u) || (GroupMode(mode) == GroupMode::tiles))) return ETXB_ERR_INVALID_ARGUMENT;
  WorkPlan p;
  p.mode = GroupMode(mode);
  p.world = world;
  p.rank = rank;
  p.queues.resize(lanes);
  p.lane_queue.assign(lanes, 0u);
  if (split_lane) p.split_lane = lanes - 1u;
  for (uint32_t i = 0; i < count; ++i) plan_enqueue(p, enqueues[i]);
  uint32_t n = 0;
  for (uint32_t q = 0; q < lanes; ++q)
    for (const WorkItem& it : p.queues[q]) {
      if (n >= capacity) return int(n);
      uint32_t* o = out_quads + 4u * n++;
      o[0] = q, o[1] = it.ordinal, o[2] = it.part, o[3] = it.parts;
    }
  return int(n);
}

// Replica mode: reserves the group's LAST lane for camera-split iterations (see replica_plan); it takes no whole-frame iterations.  Call before
// etxb_group_comm_init_replicas; needs at least two lanes, and is refused on a group in tile mode.
int etxb_group_reserve_split_lane(etxb_group* grp) {
  if (!grp || (grp->lanes.size() < 2u)) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = etxb_group_wait(grp)) return rc;
  if (grp->plan.mode == GroupMode::tiles) return group_refuse(grp, "etxb_group_reserve_split_lane: pixel tiles and a split lane exclude each other");
  std::lock_guard<std::mutex> lock(grp->m);
  grp->plan.split_lane = uint32_t(grp->lanes.size()) - 1u;
  return ETXB_OK;
}

// The other way to split a K-iteration render over the ranks: whole-frame iterations, the job's j-th iteration on rank j % world (each rank's
// lanes take that rank's share in order).  No collective inside an iteration; one ncclReduce of the (count-weighted) films per frame.  id = one
// NCCL unique id.  Collective.  Refused, before any NCCL call, on a group that already has a communicator.
int etxb_group_comm_init_replicas(etxb_group* grp, uint32_t world, uint32_t rank, const void* id, uint64_t bytes) {
  if (!grp || !id || (bytes < sizeof(ncclUniqueId)) || (world == 0u) || (rank >= world)) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = etxb_group_wait(grp)) return rc;
  if (grp->reduce_comm != nullptr) return group_refuse(grp, "etxb_group_comm_init_replicas: the group already has a communicator");
  for (auto* c : grp->lanes)
    if (c->target_pixel_size > 1u) return group_refuse(grp, "etxb_group_comm_init_replicas: the coarse preview (film pixel size above 1) renders on one GPU", ETXB_ERR_UNSUPPORTED);
  cudaSetDevice(grp->device);
  if (int rc = comm_init_rank(grp->lanes[0], &grp->reduce_comm, world, rank, id)) return rc;
  std::lock_guard<std::mutex> lock(grp->m);
  grp->plan.mode = (world > 1u) ? GroupMode::replicas : GroupMode::local;
  grp->plan.world = world;
  grp->plan.rank = rank;
  grp->plan.enqueued = 0;
  return ETXB_OK;
}

// Collective over the ranks of a sharded group: the lanes' films are combined locally (mean weighted by the iterations each lane finished —
// the same weights on every rank, the lane -> iteration map is fixed), the camera tiles are summed on rank 0, Result = max(0, camera + light).
int etxb_group_comm_reduce_film(etxb_group* grp, uint32_t layer, float* dst_rgba, uint64_t dst_bytes) {
  if (!grp || (layer > ETXB_FILM_LIGHT)) return ETXB_ERR_INVALID_ARGUMENT;
  if (grp->plan.mode == GroupMode::local) return etxb_group_read_film(grp, layer, dst_rgba, dst_bytes);
  NcclApi* n = nccl_api();
  etxb_ctx* first = grp->lanes[0];
  const size_t px = first->path_count;
  cudaSetDevice(grp->device);
  if (grp->plan.mode == GroupMode::replicas) {
    // every rank: sum over its lanes of (iterations finished x mean film), .w = iterations; rank 0 divides the reduced sum by the reduced count
    if (int rc = group_combine_into(grp, layer, grp->combined, nullptr, true)) return rc;
    if (grp->reduced.count < px) CUDA_OK(first, grp->reduced.alloc(px));
    NCCL_OK(first, n->Reduce(grp->combined.ptr, grp->reduced.ptr, px * 4u, ncclFloat, ncclSum, 0, grp->reduce_comm, grp->stream));
    if (grp->plan.rank != 0u) {
      CUDA_OK(first, cudaStreamSynchronize(grp->stream));
      return ETXB_OK;
    }
    if (!dst_rgba || (dst_bytes < px * 16u)) return fail(first, ETXB_ERR_INVALID_ARGUMENT, "film buffer too small");
    k_film_finish_mean<<<blocks_for(uint32_t(px), 256), 256, 0, grp->stream>>>(grp->reduced.ptr, grp->combined.ptr, uint32_t(px), (layer == ETXB_FILM_RESULT) ? 1u : 0u);
    CUDA_OK(first, cudaMemcpyAsync(dst_rgba, grp->combined.ptr, px * 16u, cudaMemcpyDeviceToHost, grp->stream));
    CUDA_OK(first, cudaStreamSynchronize(grp->stream));
    return ETXB_OK;
  }
  if (layer != ETXB_FILM_LIGHT) {
    if (int rc = group_combine_into(grp, ETXB_FILM_CAMERA, grp->combined, nullptr)) return rc;
    if (grp->reduced.count < px) CUDA_OK(first, grp->reduced.alloc(px));
    NCCL_OK(first, n->Reduce(grp->combined.ptr, grp->reduced.ptr, px * 4u, ncclFloat, ncclSum, 0, grp->reduce_comm, grp->stream));
  }
  if (grp->plan.rank != 0u) {
    CUDA_OK(first, cudaStreamSynchronize(grp->stream));
    return ETXB_OK;
  }
  if (!dst_rgba || (dst_bytes < px * 16u)) return fail(first, ETXB_ERR_INVALID_ARGUMENT, "film buffer too small");
  const float4* src = grp->reduced.ptr;
  if (layer != ETXB_FILM_CAMERA) {
    if (int rc = group_combine_into(grp, ETXB_FILM_LIGHT, grp->combined_light, nullptr)) return rc;
    src = grp->combined_light.ptr;
  }
  if (layer == ETXB_FILM_RESULT) {
    FilmBuffers film = {grp->reduced.ptr, grp->combined_light.ptr, nullptr, first->width, first->height};
    k_film_resolve<<<blocks_for(uint32_t(px), 256), 256, 0, grp->stream>>>(film, grp->combined.ptr);
    src = grp->combined.ptr;
  }
  CUDA_OK(first, cudaMemcpyAsync(dst_rgba, src, px * 16u, cudaMemcpyDeviceToHost, grp->stream));
  CUDA_OK(first, cudaStreamSynchronize(grp->stream));
  return ETXB_OK;
}

int etxb_group_read_film(etxb_group* grp, uint32_t layer, float* dst_rgba, uint64_t dst_bytes) {
  if (!grp || !dst_rgba || (layer > ETXB_FILM_LIGHT)) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = group_combine_into(grp, layer, grp->combined, nullptr)) return rc;
  etxb_ctx* first = grp->lanes[0];
  const uint64_t bytes = uint64_t(first->path_count) * 16u;
  if (dst_bytes < bytes) return fail(first, ETXB_ERR_INVALID_ARGUMENT, "film buffer too small");
  CUDA_OK(first, cudaMemcpy(dst_rgba, grp->combined.ptr, bytes, cudaMemcpyDeviceToHost));
  return ETXB_OK;
}
