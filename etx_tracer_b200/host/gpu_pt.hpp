// gpu_pt.hpp — host-side C++ mirror of the reference's unidirectional path-tracing plugin (SURVEY 8(f) N3).
//
// `etxb::GPUPathTracing` has the member functions, threading contract and option ids of `etx::CPUPathTracing`
// (sources/etx/rt/integrators/path_tracing.hxx, path_tracing.cxx:122-170) and of its base `etx::Integrator`
// (sources/etx/rt/integrators/integrator.hxx:12-98) and forwards them to the C ABI in include/etx_b200.h
// (etxb_set_integrator(ETXB_INTEGRATOR_PT) + the calls the VCM adapter uses).  Like gpu_vcm.hpp it is self-contained here because
// `integrator.hxx -> util/options.hxx` does not compile with gcc; INTEGRATION.md shows the derivation a maintainer adds.
//
// Contract kept from the reference:
//  * run() first stops immediately, then (if a scene is committed) reads the options, clears the camera data of the film and schedules
//    iteration 0                                                                                              (path_tracing.cxx:35-48, 141-148)
//  * update() never blocks; when the task of the current iteration has completed it accounts the iteration, lets the film estimate the
//    noise levels, and either stops (scene.samples reached, WaitingForCompletion, or an iteration that processed no pixel because all
//    have converged) or schedules the next iteration                                                          (path_tracing.cxx:85-110)
//  * stop(WaitForCompletion) lets the current iteration finish, stop(Immediate) waits for the task            (path_tracing.cxx:154-166)
//  * update_options() restarts a running render                                                               (path_tracing.cxx:168-172)
//  * option ids "direct", "nee", "mis", "bn"                                                                  (path_tracing.cxx:36-39, 112-119)
#pragma once
#include <atomic>
#include <cstdint>

#include "../../include/etx_b200.h"

namespace etxb {

class GPUPathTracing {
 public:
  enum class State : uint32_t { Stopped, Running, WaitingForCompletion };  // Integrator::State (integrator.hxx:14-18)
  enum class Stop : uint32_t { Immediate, WaitForCompletion };             // Integrator::Stop (integrator.hxx:20-23)
  struct Status {                                                          // Integrator::Status (integrator.hxx:24-37)
    double last_iteration_time = 0.0;
    double total_time = 0.0;
    uint32_t completed_iterations = 0;
    uint32_t current_iteration = 0;
  };

  explicit GPUPathTracing(int device_index = 0) {
    etxb_device_config cfg = {};
    cfg.device_index = device_index;
    _create_result = etxb_create(&_ctx, &cfg);
    if (_create_result == ETXB_OK) _create_result = etxb_set_integrator(_ctx, ETXB_INTEGRATOR_PT);
    etxb_pt_options_default(&_options);
  }
  ~GPUPathTracing() {
    stop(Stop::Immediate);
    if (_ctx) etxb_destroy(_ctx);
  }
  GPUPathTracing(const GPUPathTracing&) = delete;
  GPUPathTracing& operator=(const GPUPathTracing&) = delete;

  const char* name() const { return "Path Tracing (B200)"; }
  bool enabled() const { return _create_result == ETXB_OK; }
  const char* status_str() const { return _ctx ? etxb_last_error(_ctx) : "no CUDA device"; }
  State state() const { return _state.load(); }
  bool can_run() const { return enabled() && _scene_committed; }

  // Raytracing::link_scene / link_camera / commit_changes: `scene` / `camera` are the reference PODs; scene.samples, noise_threshold and
  // radiance_clamp travel inside the Scene record
  int commit_scene(const void* scene, uint64_t scene_bytes, const void* camera, uint64_t camera_bytes) {
    stop(Stop::Immediate);
    _scene_committed = false;
    if (!enabled()) return _create_result;
    int rc = etxb_upload_scene(_ctx, scene, scene_bytes, camera, camera_bytes);
    _scene_committed = (rc == ETXB_OK);
    if (_scene_committed && (scene_bytes == sizeof(etxb_scene))) _samples = static_cast<const etxb_scene*>(scene)->samples;
    return rc;
  }
  // a scene file read by the module's loader (etxb_scene_file_load): tables + scene + camera in one call
  int commit_scene_file(const etxb_scene_file* file) {
    stop(Stop::Immediate);
    _scene_committed = false;
    if (!enabled()) return _create_result;
    int rc = etxb_scene_file_commit(_ctx, file);
    _scene_committed = (rc == ETXB_OK);
    if (_scene_committed) _samples = etxb_scene_file_scene(file)->samples;
    return rc;
  }
  // The application's restart after it edited the committed PODs (camera moves, material / medium / emitter / settings edits,
  // app.cxx:131-141, 368-403): etxb_update_scene keeps on the device what the edit did not change.  A render that was running starts again
  // from iteration 0; a refused edit leaves the previous scene committed (and restarts it).
  int update_scene(const void* scene, uint64_t scene_bytes, const void* camera, uint64_t camera_bytes, uint32_t samples, etxb_update_info* info = nullptr) {
    const bool was_running = (_state.load() != State::Stopped);
    stop(Stop::Immediate);
    if (!enabled()) return _create_result;
    int rc = etxb_update_scene(_ctx, scene, scene_bytes, camera, camera_bytes, info);
    if (rc == ETXB_OK) {
      _scene_committed = true;
      _samples = samples;
    }
    if (was_running) run();
    return rc;
  }
  int upload_tables(const float* xyz_441x3, const float* rgb_response_391x3, const uint8_t* sobol, const uint8_t* scrambling, const uint8_t* ranking) {
    if (!enabled()) return _create_result;
    int rc = etxb_upload_color_tables(_ctx, xyz_441x3, rgb_response_391x3);
    if (rc == ETXB_OK && sobol) rc = etxb_upload_blue_noise(_ctx, sobol, scrambling, ranking);
    return rc;
  }

  int set_option(const char* key, double value) { return etxb_pt_options_set_key(&_options, key, value); }
  const etxb_pt_options& options() const { return _options; }

  void run() {
    stop(Stop::Immediate);
    if (!can_run()) return;
    if (etxb_pt_set_options(_ctx, &_options) != ETXB_OK) return;
    if (etxb_begin(_ctx, 0) != ETXB_OK) return;
    if (etxb_enqueue_iteration(_ctx) != ETXB_OK) return;  // start() schedules the first task itself (path_tracing.cxx:47)
    _status = {};
    _seen_iterations = 0;
    _have_camera_image = true;
    _state = State::Running;
  }

  void update() {
    if (_state.load() == State::Stopped) return;
    etxb_status st = {};
    if (etxb_poll(_ctx, &st) != ETXB_OK) {
      _state = State::Stopped;
      return;
    }
    if (st.iteration_in_flight) return;  // the task has not completed (path_tracing.cxx:86-88)
    _status.last_iteration_time = st.last_iteration_time;
    _status.total_time = st.total_time;
    _status.completed_iterations = st.completed_iterations;
    _status.current_iteration = st.current_iteration;
    if (st.completed_iterations > _seen_iterations) {
      _seen_iterations = st.completed_iterations;
      _have_camera_image = true;
    }
    etxb_pt_status pt = {};
    etxb_pt_get_status(_ctx, &pt);
    if (pt.pixels_processed == 0u) _state = State::WaitingForCompletion;  // every pixel has converged (path_tracing.cxx:90-92)
    if ((_state.load() == State::WaitingForCompletion) || (st.completed_iterations >= _samples)) {
      _state = State::Stopped;
      return;
    }
    if (etxb_enqueue_iteration(_ctx) != ETXB_OK) _state = State::Stopped;
  }

  void stop(Stop st) {
    if (_state.load() == State::Stopped) return;
    _state = (st == Stop::Immediate) ? State::Stopped : State::WaitingForCompletion;
    if (_state.load() == State::Stopped && _ctx) etxb_stop(_ctx, 0);
  }

  void update_options() {
    if (_state.load() == State::Running) run();
  }

  bool have_updated_camera_image() const {
    bool r = _have_camera_image;
    _have_camera_image = false;
    return r;
  }
  bool have_updated_light_image() const { return false; }  // the path tracer never writes the light image
  const Status& status() const { return _status; }

  // Film::layer: ETXB_FILM_RESULT / CAMERA / NORMALS / ALBEDO / CAMERA_ADAPTIVE, row-major float4, y flipped in storage like the reference
  int read_film(uint32_t layer, float* rgba, uint64_t bytes) { return enabled() ? etxb_read_film(_ctx, layer, rgba, bytes) : _create_result; }
  // Film::noise_level / active_pixel_count (film.cxx:430, 461)
  float noise_level() const {
    etxb_pt_status pt = {};
    return (_ctx && (etxb_pt_get_status(_ctx, &pt) == ETXB_OK)) ? pt.noise_level : 0.0f;
  }
  etxb_ctx* context() { return _ctx; }

 private:
  etxb_ctx* _ctx = nullptr;
  int _create_result = ETXB_ERR_NO_DEVICE;
  etxb_pt_options _options = {};
  std::atomic<State> _state{State::Stopped};
  Status _status;
  uint32_t _samples = 0, _seen_iterations = 0;
  bool _scene_committed = false;
  mutable bool _have_camera_image = false;
};

}  // namespace etxb
