// group.cu — the iteration group of the C interface (etxb_group, include/etx_b200.h): L contexts on one device whose lanes render iterations
// in flight, the work plan that deals the iterations to the lanes, the film combine, and the group's communicators over NCCL.  It reaches
// the contexts through the C interface and the internals context.cuh declares; the kernels of the film combine are its own.
#include <cstring>
#include <deque>

#include "context.cuh"

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

// The C interface's group handle: its default visibility is stated as etxb_ctx's is (context.cuh), its members' types being hidden
struct __attribute__((visibility("default"))) etxb_group {
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

  // a C++ symbol, kept out of the library's exports (the interface is etxb_group_destroy)
  __attribute__((visibility("hidden"))) ~etxb_group() = default;
};

namespace {

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

// A call on a lane failed with `code`: the lane's etxb_last_error becomes etxb_group_last_error
int group_fail(etxb_group* grp, const etxb_ctx* lane, int code) {
  std::lock_guard<std::mutex> lock(grp->m);
  grp->error_text = etxb_last_error(lane);
  return code;
}

// A call the group refuses in its present state: the reason goes to etxb_group_last_error and to lane 0's etxb_last_error
int group_refuse(etxb_group* grp, const char* why, int code = ETXB_ERR_INVALID_ARGUMENT) { return group_fail(grp, grp->lanes[0], fail(grp->lanes[0], code, "%s", why)); }

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
  for (auto* c : grp->lanes)
    if (int rc = etxb_set_film_pixel_size(c, size)) return group_fail(grp, c, rc);
  return ETXB_OK;
}

int etxb_group_update_scene(etxb_group* grp, const void* scene_blob, uint64_t scene_bytes, const void* camera_blob, uint64_t camera_bytes, etxb_update_info* info) {
  const auto t0 = std::chrono::steady_clock::now();
  if (info) memset(info, 0, sizeof(*info));
  if (!grp || !scene_blob || !camera_blob) return ETXB_ERR_INVALID_ARGUMENT;
  etxb_ctx* first = grp->lanes[0];
  bool comm = grp->plan.mode != GroupMode::local;
  for (auto* c : grp->lanes) comm = comm || (c->comm != nullptr);
  if (comm) return group_refuse(grp, "etxb_group_update_scene: a group with communicators takes a new scene through etxb_upload_scene on each lane", ETXB_ERR_UNSUPPORTED);
  if (int rc = check_scene_args(first, scene_bytes, camera_bytes)) return group_fail(grp, first, rc);
  if (int rc = etxb_group_wait(grp)) return rc;
  const etxb_scene& s = *static_cast<const etxb_scene*>(scene_blob);
  const etxb_camera& cam = *static_cast<const etxb_camera*>(camera_blob);
  cudaSetDevice(grp->device);
  // hashed and validated once; a new geometry's BVH is built once, and its depth checked, before any lane changes
  ScenePrep p;
  if (int rc = prepare_scene(first, s, cam, p)) return group_fail(grp, first, rc);
  for (auto* c : grp->lanes)
    if (!geometry_kept(c, p, c->scene_ready))
      if (int rc = prepare_bvh(first, s, p)) return group_fail(grp, first, rc);
  uint32_t kept = ~0u;
  for (size_t l = 0; l < grp->lanes.size(); ++l) {
    etxb_ctx* c = grp->lanes[l];
    etxb_update_info lane = {};
    ctx_drain(c);
    if (int rc = commit_scene(c, s, cam, p, c->scene_ready, &lane)) return group_fail(grp, c, rc);
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
  for (size_t l = 0; l < grp->lanes.size(); ++l)
    if (int rc = etxb_comm_init(grp->lanes[l], world, rank, bytes + l * sizeof(ncclUniqueId), sizeof(ncclUniqueId))) return group_fail(grp, grp->lanes[l], rc);
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
    return end_rank0_reduce(first, grp->stream, grp->plan.rank, dst_rgba, dst_bytes, px, [&](const float4** src) -> int {
      k_film_finish_mean<<<blocks_for(uint32_t(px), 256), 256, 0, grp->stream>>>(grp->reduced.ptr, grp->combined.ptr, uint32_t(px), (layer == ETXB_FILM_RESULT) ? 1u : 0u);
      *src = grp->combined.ptr;
      return ETXB_OK;
    });
  }
  if (layer != ETXB_FILM_LIGHT) {
    if (int rc = group_combine_into(grp, ETXB_FILM_CAMERA, grp->combined, nullptr)) return rc;
    if (grp->reduced.count < px) CUDA_OK(first, grp->reduced.alloc(px));
    NCCL_OK(first, n->Reduce(grp->combined.ptr, grp->reduced.ptr, px * 4u, ncclFloat, ncclSum, 0, grp->reduce_comm, grp->stream));
  }
  // rank 0 finishes the summed camera tiles with the light layer as etxb_read_film finishes a context's own
  return end_rank0_reduce(first, grp->stream, grp->plan.rank, dst_rgba, dst_bytes, px, [&](const float4** src) -> int {
    if (layer != ETXB_FILM_CAMERA)
      if (int rc = group_combine_into(grp, ETXB_FILM_LIGHT, grp->combined_light, nullptr)) return rc;
    *src = (layer == ETXB_FILM_LIGHT) ? grp->combined_light.ptr
                                      : film_layer_finish(layer, grp->reduced.ptr, grp->combined_light.ptr, first->width, first->height, grp->combined.ptr, grp->stream);
    return ETXB_OK;
  });
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