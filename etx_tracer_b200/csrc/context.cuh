// context.cuh — the context behind the C interface (struct etxb_ctx) and the host helpers of the units that drive it: module.cu (the
// product: context, passes, film, NCCL), scene_upload.cu (the scene upload and update), group.cu (the iteration group, etxb_group) and
// test_hooks.cu (the test hooks that run the d*.cuh routines on host-given queries).  No kernels*.cuh here: their non-template kernels have
// host stubs with external linkage, and a second unit that included them would not link; etxb_ctx names two of their types by declaration only.
#pragma once
#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <mutex>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include <nccl.h>

#include "dvcm.cuh"

namespace etxb {
struct DeviceCounters;  // kernels.cuh
struct ErrorSums;       // kernels_view.cuh
}  // namespace etxb

// C++ internals shared by the library's units, kept out of its exports
namespace etxb_internal __attribute__((visibility("hidden"))) {

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
inline const char* kKernelNames[K_COUNT] = {"light_begin", "trace_closest(light)", "light_bounce", "lv_scan", "lv_reorder", "grid_bbox", "grid_keys", "grid_sort", "grid_build",
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

// a 128-bit content hash (hash128, scene_upload.cu)
struct Hash128 {
  uint64_t lo = 0, hi = 0;
  bool operator==(const Hash128& o) const { return (lo == o.lo) && (hi == o.hi); }
};

// what the last upload / update of a context copied, by content (etxb_update_scene keeps what did not change)
struct SceneHashes {
  bool valid = false;  // set once the whole scene is on the device
  Hash128 geometry;    // vertex array + triangle array: device vertices, triangles, BVH2 (+ the 4-wide tree)
  std::vector<Hash128> images, grids;  // per image; per medium (zero for media without a density grid)
};

}  // namespace etxb_internal

using namespace etxb;
using namespace etxb_internal;

// The C interface's handle.  Its default visibility is stated, as its members' types are hidden (GCC warns otherwise); a hidden etxb_ctx
// would hide the etxb_* functions that take it, since GCC gives a function no more visibility than its parameter types.
struct __attribute__((visibility("default"))) etxb_ctx {
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
  DevBuf<float4> film_view;                                  // the float4 frame of etxb_read_film_view (the RGBA8 one goes to film_ldr)
  DevBuf<float4> reference;                                  // the viewer's reference image: W x H in storage order, empty when none is set
  double reference_mean_rgb = 0.0;                           // its mean over pixels and RGB channels, the scale of rel_mse's epsilon
  DevBuf<ErrorSums> error_blocks;                            // etxb_film_error: one record per block, then the final record
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

namespace etxb_internal __attribute__((visibility("hidden"))) {

inline int fail(etxb_ctx* ctx, int code, const char* fmt, ...) {
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

template <class T>
int upload(etxb_ctx* ctx, DevBuf<T>& buf, const T* host, size_t n) {
  CUDA_OK(ctx, buf.alloc(std::max<size_t>(n, 1)));
  if (n) CUDA_OK(ctx, cudaMemcpyAsync(buf.ptr, host, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  return ETXB_OK;
}

// takes ownership of a cudaMalloc'd array of n elements
template <class T>
void adopt(DevBuf<T>& buf, T* ptr, size_t n) {
  buf.release();
  buf.ptr = ptr;
  buf.count = n;
}

inline uint32_t blocks_for(uint32_t n, uint32_t block) { return (n + block - 1u) / block; }

inline double seconds_since(std::chrono::steady_clock::time_point t0) { return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count(); }

// ---- the scene upload and update (scene_upload.cu) ----------------------------------------------------------------------------------------
// etxb_upload_scene, etxb_update_scene and etxb_group_update_scene run the same stages: validate_scene makes every check and touches nothing
// on the device, prepare_scene hashes the bulk arrays (prepare_bvh uploads a new geometry and builds its BVH2 on the device), commit_scene
// commits to the device.  An update keeps the device copies whose content hashes did not change; everything small is derived from the PODs
// again on every call.
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

int check_scene_args(etxb_ctx* ctx, uint64_t scene_bytes, uint64_t camera_bytes);
int prepare_scene(etxb_ctx* ctx, const etxb_scene& s, const etxb_camera& cam, ScenePrep& p);
int prepare_bvh(etxb_ctx* ctx, const etxb_scene& s, ScenePrep& p);
bool geometry_kept(const etxb_ctx* ctx, const ScenePrep& p, bool reuse);
int commit_scene(etxb_ctx* ctx, const etxb_scene& s, const etxb_camera& cam, ScenePrep& p, bool reuse, etxb_update_info* info);

// ---- the driver (module.cu) ------------------------------------------------------------------------------------------------------------------
// commit_scene's last step: the film and path-state buffers for the committed scene class and film size (Film::allocate), counting the
// allocations it makes (none: an update kept the path state)
int commit_path_state(etxb_ctx* ctx, const etxb_camera& cam, bool reuse, uint32_t* allocations);
// one whole iteration on the calling thread; returns when it has finished (the bounce loops read queue sizes back)
int run_iteration_blocking(etxb_ctx* ctx);
// blocks until every queued iteration of the context's worker has finished; returns (and clears) the first error one of them hit
int ctx_drain(etxb_ctx* ctx);
// Film::layer's read-out of `layer` (film.cxx:381-418) from `raw`, the buffer the layer is made from: Result = max(0, raw + light) and
// Normals = raw * 0.5 + 0.5 are written to `out`, which is returned; every other layer is `raw` as it is.  Asynchronous on `stream`.
const float4* film_layer_finish(uint32_t layer, float4* raw, float4* light, uint32_t width, uint32_t height, float4* out, cudaStream_t stream);

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
// the bound library, or null where it could not be loaded
NcclApi* nccl_api();

#define NCCL_OK(ctx, call)                                                                                                 \
  do {                                                                                                                     \
    ncclResult_t res__ = (call);                                                                                           \
    if (res__ != ncclSuccess) return fail(ctx, ETXB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, nccl_api()->GetErrorString(res__), __FILE__, __LINE__); \
  } while (0)

// Joins rank `rank` of a `world`-rank communicator on the current device; `id` holds the ncclUniqueId rank 0 made.  Collective.
int comm_init_rank(etxb_ctx* ctx, ncclComm_t* comm, uint32_t world, uint32_t rank, const void* id);
// A stream at the device's highest priority, so that its few blocks do not queue behind the lanes' large kernels
cudaError_t create_priority_stream(cudaStream_t* stream);

// The end of a film reduce to rank 0 on `stream`: a rank other than 0 waits for its part and returns; rank 0 checks the host buffer, finishes
// the layer (`finish(&src)` leaves the device buffer that holds it in src) and copies it to `dst`.  Errors go to `ctx`.
template <class Finish>
int end_rank0_reduce(etxb_ctx* ctx, cudaStream_t stream, uint32_t rank, float* dst, uint64_t dst_bytes, size_t pixels, Finish&& finish) {
  if (rank != 0u) {
    CUDA_OK(ctx, cudaStreamSynchronize(stream));
    return ETXB_OK;
  }
  if (!dst || (dst_bytes < pixels * 16u)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "film buffer too small");
  const float4* src = nullptr;
  if (int rc = finish(&src)) return rc;
  CUDA_OK(ctx, cudaMemcpyAsync(dst, src, pixels * 16u, cudaMemcpyDeviceToHost, stream));
  CUDA_OK(ctx, cudaStreamSynchronize(stream));
  return ETXB_OK;
}

}  // namespace etxb_internal
