// module.cu — C ABI (include/etx_b200.h) over the wavefront kernels: context, iteration driver, film, NCCL.
// Host-side counterpart of CPUVCMImpl (sources/etx/rt/integrators/vcm_cpu.cxx:30-241).  The context is declared in context.cuh; the scene
// upload and update are in scene_upload.cu (its last step, the path-state buffers the kernels size, is commit_path_state here), the iteration
// group in group.cu, and the test hooks that run the d*.cuh routines on host-given queries in test_hooks.cu.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <ctime>

#include <dlfcn.h>

#include "bvh_build.h"
#include "bvh_build_device.h"
#include "context.cuh"
#include "kernels.cuh"
#include "kernels_pt.cuh"
#include "kernels_denoise.cuh"
#include "kernels_view.cuh"

#if defined(ETXB_PARITY) && ETXB_PARITY
static const char* kFlavor = "parity";
#else
static const char* kFlavor = "fast";
#endif

namespace etxb_internal __attribute__((visibility("hidden"))) {

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

int comm_init_rank(etxb_ctx* ctx, ncclComm_t* comm, uint32_t world, uint32_t rank, const void* id) {
  NcclApi* n = nccl_api();
  if (!n) return fail(ctx, ETXB_ERR_NOT_READY, "libnccl.so.2 could not be loaded");
  ncclUniqueId uid;
  memcpy(&uid, id, sizeof(uid));
  NCCL_OK(ctx, n->CommInitRank(comm, int(world), uid, int(rank)));
  return ETXB_OK;
}

cudaError_t create_priority_stream(cudaStream_t* stream) {
  int prio_low = 0, prio_high = 0;
  if (cudaError_t err = cudaDeviceGetStreamPriorityRange(&prio_low, &prio_high)) return err;
  return cudaStreamCreateWithPriority(stream, cudaStreamNonBlocking, prio_high);
}

}  // namespace etxb_internal

namespace {

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

// Buffers that only some scene classes use, each with the count the scene asks for: sized by `size(buffer, count)` when `needed`, released
// otherwise.  Stops at the first error.
template <class Size, class... T>
cudaError_t size_if_needed(bool needed, Size&& size, std::pair<DevBuf<T>*, size_t>... bufs) {
  cudaError_t err = cudaSuccess;
  if (needed) {
    ((err = (err == cudaSuccess) ? size(*bufs.first, bufs.second) : err), ...);
  } else {
    (bufs.first->release(), ...);
  }
  return err;
}

}  // namespace

namespace etxb_internal __attribute__((visibility("hidden"))) {

// Film + queues (Film::allocate, film.cxx).  An update keeps every buffer whose size is what the upload would allocate (DevBuf::ensure).
int commit_path_state(etxb_ctx* ctx, const etxb_camera& cam, bool reuse, uint32_t* allocations) {
  auto sized = [&](auto& b, size_t count) -> cudaError_t {
    if (reuse) return b.ensure(count, *allocations);
    *allocations += 1;
    return b.alloc(count);
  };
  if ((ctx->width != cam.film_size[0]) || (ctx->height != cam.film_size[1])) {  // Denoised starts over at a new film size; the reference no longer fits
    ctx->film_denoised.release();
    ctx->reference.release();
  }
  ctx->width = cam.film_size[0];
  ctx->height = cam.film_size[1];
  ctx->path_count = ctx->width * ctx->height;
  size_t n = ctx->path_count;
  if (!reuse) {
    ctx->film_normals.release();  // sized by the film: re-allocated by the next path-tracer run
  } else if (ctx->film_normals.ptr && (ctx->film_normals.count != n)) {
    if (int rc = pt_ensure_film(ctx)) return rc;  // the path tracer's layers and per-pixel history at the new film size
    *allocations += 1;
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
  // the material sorts of path queues and connection lists (scenes with stochastic BSDFs)
  CUDA_OK(ctx, size_if_needed(ctx->has_stochastic_merge, sized, std::pair{&ctx->conn_list_sorted, cap}, std::pair{&ctx->queue_sorted, n}, std::pair{&ctx->queue_keys, n},
                              std::pair{&ctx->queue_keys_sorted, n}));
#if defined(ETXB_PARITY) && ETXB_PARITY
  ctx->conn_rec.release();
#else
  // the connection stage's per-path camera vertex records (make_params: connect_stage = has_stochastic_merge)
  CUDA_OK(ctx, size_if_needed(ctx->has_stochastic_merge, sized, std::pair{&ctx->conn_rec, n * (ctx->spectral ? kConnRecRows<true> : kConnRecRows<false>)}));
#endif
  CUDA_OK(ctx, sized(ctx->trace_cursor, 1));
  // the shadow segments of deferred shadow rays and of the atomic mode: a camera bounce queues its vertex connections (<= cap, the pair list's
  // capacity) plus, in atomic mode, one emitter segment per path
  const bool atomic_candidate = ctx->opaque_scene && ctx->plain_scene && ctx->has_stochastic_merge;
  const uint64_t shadow_cap = std::min<uint64_t>(cap + (atomic_candidate ? n : 0), 0x7fffffffull);
  CUDA_OK(ctx, size_if_needed(ctx->dscene.deferred_shadow_rays || atomic_candidate, sized, std::pair{&ctx->shadow_span, n}, std::pair{&ctx->shadow_p0, shadow_cap},
                              std::pair{&ctx->shadow_p1, shadow_cap}, std::pair{&ctx->shadow_value, shadow_cap}, std::pair{&ctx->shadow_result, shadow_cap},
                              std::pair{&ctx->shadow_count, size_t(2)}));
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
  return ETXB_OK;
}

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

int ctx_drain(etxb_ctx* ctx) {
  std::unique_lock<std::mutex> lock(ctx->worker_m);
  ctx->worker_idle.wait(lock, [&] { return (ctx->worker_queued == 0) && !ctx->worker_busy; });
  int rc = ctx->worker_error;
  ctx->worker_error = ETXB_OK;
  return rc;
}

const float4* film_layer_finish(uint32_t layer, float4* raw, float4* light, uint32_t width, uint32_t height, float4* out, cudaStream_t stream) {
  const uint32_t n = width * height;
  if (layer == ETXB_FILM_RESULT) {
    FilmBuffers film = {raw, light, nullptr, width, height};
    k_film_resolve<<<blocks_for(n, 256), 256, 0, stream>>>(film, out);
    return out;
  }
  if (layer == ETXB_FILM_NORMALS) {  // the VCM integrator leaves them empty; shown as n * 0.5 + 0.5
    k_film_layer_normals<<<blocks_for(n, 256), 256, 0, stream>>>(raw, out, n);
    return out;
  }
  return raw;
}

}  // namespace etxb_internal

namespace {

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

// Film::layer (film.cxx:381-418), step 1: the context's per-pixel buffer that `layer` is made from (the camera image for Result)
int film_layer_raw(etxb_ctx* ctx, uint32_t layer, float4** out) {
  switch (layer) {
    case ETXB_FILM_RESULT:
    case ETXB_FILM_CAMERA:
      *out = ctx->film_camera.ptr;
      return ETXB_OK;
    case ETXB_FILM_LIGHT:
      *out = ctx->film_light.ptr;
      return ETXB_OK;
    case ETXB_FILM_LIGHT_ITERATION:
      *out = ctx->film_light_iteration.ptr;
      return ETXB_OK;
    case ETXB_FILM_CAMERA_ADAPTIVE:
      if (int rc = film_ensure_adaptive(ctx)) return rc;
      *out = ctx->film_adaptive.ptr;
      return ETXB_OK;
    case ETXB_FILM_DENOISED:
      if (ctx->film_denoised.count != ctx->path_count) {
        CUDA_OK(ctx, ctx->film_denoised.alloc(ctx->path_count));
        CUDA_OK(ctx, cudaMemsetAsync(ctx->film_denoised.ptr, 0, ctx->film_denoised.bytes(), ctx->stream));
      }
      *out = ctx->film_denoised.ptr;
      return ETXB_OK;
    case ETXB_FILM_NORMALS:
    case ETXB_FILM_ALBEDO:
      if (int rc = pt_ensure_film(ctx)) return rc;
      *out = (layer == ETXB_FILM_NORMALS) ? ctx->film_normals.ptr : ctx->film_albedo.ptr;
      return ETXB_OK;
    default:
      return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "unknown film layer %u", layer);
  }
}

// step 2 on the context's stream, into its film_out, with the context's light image: `raw` is step 1's buffer or its sum over the ranks
const float4* film_layer_read_out(etxb_ctx* ctx, uint32_t layer, float4* raw) {
  const float4* src = film_layer_finish(layer, raw, ctx->film_light.ptr, ctx->width, ctx->height, ctx->film_out.ptr, ctx->stream);
  if (src != raw) ctx->kernel_launches += 1;
  return src;
}

// the device buffer that holds `layer` as float4 (computed into film_out where the layer is derived)
int film_layer_source(etxb_ctx* ctx, uint32_t layer, const float4** out_src) {
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  cudaSetDevice(ctx->device);
  float4* raw = nullptr;
  if (int rc = film_layer_raw(ctx, layer, &raw)) return rc;
  *out_src = film_layer_read_out(ctx, layer, raw);
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

// ---- the viewer (DESIGN §14) -------------------------------------------------------------------------------------------------------------
int check_view(etxb_ctx* ctx, const etxb_view* v) {
  if (!v) return ETXB_ERR_INVALID_ARGUMENT;
  if ((v->view > ETXB_VIEW_ABSOLUTE) || (v->options & ~(ETXB_VIEW_OPT_TONEMAPPING | ETXB_VIEW_OPT_SRGB | ETXB_VIEW_OPT_SKIP_COLOR_CONVERSION)) ||
      !std::isfinite(v->exposure) || (v->rgba8 > 1u))
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "film view: view %u (0-5), options 0x%x (bits 0-2), exposure %g (finite), rgba8 %u (0 or 1)", v->view, v->options,
                double(v->exposure), v->rgba8);
  return ETXB_OK;
}

int check_whole_film(etxb_ctx* ctx, const char* what) {
  if (!ctx->scene_ready) return fail(ctx, ETXB_ERR_NOT_READY, "no scene uploaded");
  if ((ctx->comm != nullptr) || (ctx->world > 1u)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "%s: the film of a context with pixel tiles holds only its own tiles", what);
  return ETXB_OK;
}

bool has_reference(const etxb_ctx* ctx) { return (ctx->reference.ptr != nullptr) && (ctx->reference.count == ctx->path_count); }

// k_film_view over n pixels into the context's own frame buffer, then to `dst`; synchronous
int run_film_view(etxb_ctx* ctx, const float4* layer, const float4* ref, size_t n, const etxb_view& v, void* dst) {
  float4* out_f = nullptr;
  uint32_t* out_rgba8 = nullptr;
  if (v.rgba8) {
    if (ctx->film_ldr.count != n) CUDA_OK(ctx, ctx->film_ldr.alloc(n));
    out_rgba8 = ctx->film_ldr.ptr;
  } else {
    if (ctx->film_view.count != n) CUDA_OK(ctx, ctx->film_view.alloc(n));
    out_f = ctx->film_view.ptr;
  }
  k_film_view<<<blocks_for(uint32_t(n), 256), 256, 0, ctx->stream>>>(layer, ref, uint32_t(n), v.view, v.options, v.exposure, out_f, out_rgba8);
  ctx->kernel_launches += 1;
  const void* src = v.rgba8 ? static_cast<const void*>(out_rgba8) : static_cast<const void*>(out_f);
  CUDA_OK(ctx, cudaMemcpyAsync(dst, src, n * (v.rgba8 ? 4u : 16u), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  return ETXB_OK;
}

// the two passes of the error reduction over n > 0 pixels (MeanOnly: the reference's r + g + b); synchronous
template <bool MeanOnly>
int run_film_error(etxb_ctx* ctx, const float4* layer, const float4* ref, uint32_t n, double eps, ErrorSums* out) {
  const uint32_t blocks = (n + kErrorChunk - 1u) / kErrorChunk;
  if (ctx->error_blocks.count < blocks + 1u) CUDA_OK(ctx, ctx->error_blocks.alloc(blocks + 1u));
  ErrorSums* final_record = ctx->error_blocks.ptr + blocks;
  k_film_error_blocks<MeanOnly><<<blocks, kErrorThreads, 0, ctx->stream>>>(layer, ref, n, eps, ctx->error_blocks.ptr);
  k_film_error_final<<<1, kErrorThreads, 0, ctx->stream>>>(ctx->error_blocks.ptr, blocks, final_record);
  ctx->kernel_launches += 2;
  CUDA_OK(ctx, cudaMemcpyAsync(out, final_record, sizeof(ErrorSums), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
  return ETXB_OK;
}

// mean_rgb of a reference of n pixels
int reference_mean_rgb(etxb_ctx* ctx, const float4* ref, uint32_t n, double* out) {
  ErrorSums s = {};
  if (int rc = run_film_error<true>(ctx, nullptr, ref, n, 0.0, &s)) return rc;
  *out = s.se / (3.0 * double(n));
  return ETXB_OK;
}

// the reference slot has just been filled: its mean, or the slot emptied again when that fails
int commit_reference(etxb_ctx* ctx) {
  if (int rc = reference_mean_rgb(ctx, ctx->reference.ptr, ctx->path_count, &ctx->reference_mean_rgb)) {
    ctx->reference.release();
    return rc;
  }
  return ETXB_OK;
}

int film_error_of(etxb_ctx* ctx, const float4* layer, const float4* ref, uint32_t n, double mean_rgb, etxb_film_error_info* out) {
  ErrorSums s = {};
  const double eps = (0.01 * mean_rgb) * (0.01 * mean_rgb);
  if (int rc = run_film_error<false>(ctx, layer, ref, n, eps, &s)) return rc;
  const double finite = double(s.finite);
  memset(out, 0, sizeof(*out));
  out->pixels = n;
  out->nonfinite = s.nonfinite;
  out->negative = s.negative;
  out->lum_above = s.above;
  out->lum_below = s.below;
  out->mse = s.se / (3.0 * finite);
  out->rel_mse = s.rel / (3.0 * finite);
  out->mean_abs_lum = s.abs_lum / finite;
  out->mean_lum = s.lum / finite;
  out->reference_mean_lum = s.ref_lum / finite;
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
  cudaSetDevice(ctx->device);
  const size_t px = ctx->path_count;
  if (ctx->film_reduced.count < px) CUDA_OK(ctx, ctx->film_reduced.alloc(px));
  if (layer != ETXB_FILM_LIGHT) {
    // the tiled layers: each rank holds its own tiles and zeros elsewhere (k_pt_accumulate and k_film_adaptive_vcm write owned pixels only)
    float4* tiles = nullptr;
    if (int rc = film_layer_raw(ctx, layer, &tiles)) return rc;
    NCCL_OK(ctx, nccl_api()->Reduce(tiles, ctx->film_reduced.ptr, px * 4u, ncclFloat, ncclSum, 0, ctx->comm, ctx->stream));
  }
  return end_rank0_reduce(ctx, ctx->stream, ctx->rank, dst_rgba, dst_bytes, px, [&](const float4** src) -> int {
    *src = (layer == ETXB_FILM_LIGHT) ? ctx->film_light.ptr : film_layer_read_out(ctx, layer, ctx->film_reduced.ptr);
    return ETXB_OK;
  });
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

// ImagePool::add_from_data into the viewer's reference slot (app.cxx:243-250 with a file read by the caller)
int etxb_set_reference_image(etxb_ctx* ctx, const float* rgba, uint32_t width, uint32_t height) {
  if (!ctx || !rgba) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = check_whole_film(ctx, "etxb_set_reference_image")) return rc;
  // the reference's HLSL and Metal shaders disagree on a reference of another size (a zero Load against a bilinear uv sample): neither is taken
  if ((width != ctx->width) || (height != ctx->height))
    return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "etxb_set_reference_image: a %ux%u image for a %ux%u film", width, height, ctx->width, ctx->height);
  cudaSetDevice(ctx->device);
  if (ctx->reference.count != ctx->path_count) CUDA_OK(ctx, ctx->reference.alloc(ctx->path_count));
  CUDA_OK(ctx, cudaMemcpyAsync(ctx->reference.ptr, rgba, ctx->reference.bytes(), cudaMemcpyHostToDevice, ctx->stream));
  return commit_reference(ctx);
}

// Use as Reference (app.cxx:252-259): the layer as it stands, copied on the device
int etxb_use_film_as_reference(etxb_ctx* ctx, uint32_t layer) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = check_whole_film(ctx, "etxb_use_film_as_reference")) return rc;
  const float4* src = nullptr;
  if (int rc = film_layer_source(ctx, layer, &src)) return rc;
  if (ctx->reference.count != ctx->path_count) CUDA_OK(ctx, ctx->reference.alloc(ctx->path_count));
  CUDA_OK(ctx, cudaMemcpyAsync(ctx->reference.ptr, src, ctx->reference.bytes(), cudaMemcpyDeviceToDevice, ctx->stream));
  return commit_reference(ctx);
}

int etxb_clear_reference(etxb_ctx* ctx) {
  if (!ctx) return ETXB_ERR_INVALID_ARGUMENT;
  if ((ctx->comm != nullptr) || (ctx->world > 1u)) return fail(ctx, ETXB_ERR_UNSUPPORTED, "etxb_clear_reference: the film of a context with pixel tiles holds only its own tiles");
  cudaSetDevice(ctx->device);
  ctx->reference.release();
  return ETXB_OK;
}

// RenderContext's fragment shader (render.cxx:252-388) over the whole layer
int etxb_read_film_view(etxb_ctx* ctx, uint32_t layer, const etxb_view* view, void* dst, uint64_t dst_bytes) {
  if (!ctx || !dst) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = check_view(ctx, view)) return rc;
  if (int rc = check_whole_film(ctx, "etxb_read_film_view")) return rc;
  if ((view->view >= ETXB_VIEW_REFERENCE) && !has_reference(ctx)) return fail(ctx, ETXB_ERR_NOT_READY, "etxb_read_film_view: view %u needs a reference image", view->view);
  const size_t n = ctx->path_count;
  if (dst_bytes < n * (view->rgba8 ? 4u : 16u)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "film buffer too small");
  const float4* src = nullptr;
  if (int rc = film_layer_source(ctx, layer, &src)) return rc;
  return run_film_view(ctx, src, (view->view >= ETXB_VIEW_REFERENCE) ? ctx->reference.ptr : nullptr, n, *view, dst);
}

int etxb_film_error(etxb_ctx* ctx, uint32_t layer, etxb_film_error_info* out) {
  if (!ctx || !out) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = check_whole_film(ctx, "etxb_film_error")) return rc;
  if (!has_reference(ctx)) return fail(ctx, ETXB_ERR_NOT_READY, "etxb_film_error: no reference image");
  if (int rc = ctx_drain(ctx)) return rc;
  const float4* src = nullptr;
  if (int rc = film_layer_source(ctx, layer, &src)) return rc;
  if (int rc = film_error_of(ctx, src, ctx->reference.ptr, ctx->path_count, ctx->reference_mean_rgb, out)) return rc;
  out->iterations = ctx->completed;
  return ETXB_OK;
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

// Test hook: etxb_read_film_view's kernel on host arrays
int etxb_debug_film_view(etxb_ctx* ctx, const float* layer, const float* reference, uint32_t count, const etxb_view* view, void* out) {
  if (!ctx || !layer || !out || !count) return ETXB_ERR_INVALID_ARGUMENT;
  if (int rc = check_view(ctx, view)) return rc;
  if ((view->view >= ETXB_VIEW_REFERENCE) && !reference) return fail(ctx, ETXB_ERR_NOT_READY, "etxb_debug_film_view: view %u needs a reference image", view->view);
  cudaSetDevice(ctx->device);
  DevBuf<float4> dl, dr;
  if (int rc = upload(ctx, dl, reinterpret_cast<const float4*>(layer), count)) return rc;
  if (reference)
    if (int rc = upload(ctx, dr, reinterpret_cast<const float4*>(reference), count)) return rc;
  return run_film_view(ctx, dl.ptr, reference ? dr.ptr : nullptr, count, *view, out);
}

// Test hook: etxb_film_error's kernels on host arrays (the reference's mean taken as etxb_set_reference_image takes it)
int etxb_debug_film_error(etxb_ctx* ctx, const float* layer, const float* reference, uint32_t width, uint32_t height, etxb_film_error_info* out) {
  if (!ctx || !layer || !reference || !out || !width || !height) return ETXB_ERR_INVALID_ARGUMENT;
  if (uint64_t(width) * height > (1ull << 26)) return fail(ctx, ETXB_ERR_INVALID_ARGUMENT, "etxb_debug_film_error: film too large");
  cudaSetDevice(ctx->device);
  const uint32_t n = width * height;
  DevBuf<float4> dl, dr;
  if (int rc = upload(ctx, dl, reinterpret_cast<const float4*>(layer), n)) return rc;
  if (int rc = upload(ctx, dr, reinterpret_cast<const float4*>(reference), n)) return rc;
  double mean_rgb = 0.0;
  if (int rc = reference_mean_rgb(ctx, dr.ptr, n, &mean_rgb)) return rc;
  return film_error_of(ctx, dl.ptr, dr.ptr, n, mean_rgb, out);
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
