// gpu_vcm.hpp — host-side C++ mirror of the reference's Integrator plugin for this path.
//
// `etxb::GPUVCM` has the member functions, threading contract and option keys of `etx::CPUVCM`
// (sources/etx/rt/integrators/vcm_cpu.hxx:7-27, vcm_cpu.cxx:247-310) and of its base `etx::Integrator`
// (sources/etx/rt/integrators/integrator.hxx:12-98), and forwards them to the C ABI in include/etx_b200.h.
// In the reference tree the class would derive from `etx::Integrator` (see INTEGRATION.md for the 3-line diff); here it is
// self-contained because `integrator.hxx -> util/options.hxx` does not compile with gcc (options.hxx:77-88).
//
// Contract kept from the reference:
//  * run() first stops immediately, then (if a scene is committed) clears the film and starts at iteration 0   (vcm_cpu.cxx:255-262)
//  * update() is called once per UI frame from the thread that pumps IntegratorThread; it advances the render and
//    fills Status; when `scene.samples` iterations are done the state becomes Stopped                          (vcm_cpu.cxx:264-276, 227-241)
//  * stop(WaitForCompletion) lets the current iteration finish, stop(Immediate) returns after the queue drained (vcm_cpu.cxx:278-288)
//  * update_options() restarts a running render                                                                (vcm_cpu.cxx:290-294)
//  * options are the reference's `vcm-*` keys                                                                  (vcm_shared.cxx:15-28)
#pragma once
#include <atomic>
#include <cstdint>
#include <string>

#include "../../include/etx_b200.h"

namespace etxb {

class GPUVCM {
 public:
  enum class State : uint32_t { Stopped, Running, WaitingForCompletion };  // Integrator::State (integrator.hxx:14-18)
  enum class Stop : uint32_t { Immediate, WaitForCompletion };             // Integrator::Stop (integrator.hxx:20-23)

  struct Status {  // Integrator::Status (integrator.hxx:24-37)
    double last_iteration_time = 0.0;
    double total_time = 0.0;
    uint32_t completed_iterations = 0;
    uint32_t current_iteration = 0;
  };

  explicit GPUVCM(int device_index = 0) {
    etxb_device_config cfg = {};
    cfg.device_index = device_index;
    _create_result = etxb_create(&_ctx, &cfg);
    etxb_options_default(&_options);
  }
  ~GPUVCM() {
    stop(Stop::Immediate);
    if (_ctx) etxb_destroy(_ctx);
  }
  GPUVCM(const GPUVCM&) = delete;
  GPUVCM& operator=(const GPUVCM&) = delete;

  const char* name() const { return "VCM (B200)"; }
  bool enabled() const { return _create_result == ETXB_OK; }
  const char* status_str() const { return _ctx ? etxb_last_error(_ctx) : "no CUDA device"; }
  State state() const { return _state.load(); }
  bool can_run() const { return enabled() && _scene_committed; }

  // Raytracing::link_scene / link_camera / commit_changes (rt.cxx:58-64, 323): `scene`/`camera` are the reference PODs.
  int commit_scene(const void* scene, uint64_t scene_bytes, const void* camera, uint64_t camera_bytes, uint32_t samples) {
    stop(Stop::Immediate);
    _scene_committed = false;
    if (!enabled()) return _create_result;
    int rc = etxb_upload_scene(_ctx, scene, scene_bytes, camera, camera_bytes);
    _scene_committed = (rc == ETXB_OK);
    _samples = samples;
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

  // Integrator::options(): the reference's keys
  int set_option(const char* key, double value) { return etxb_options_set_key(&_options, key, value); }
  const etxb_vcm_options& options() const { return _options; }

  void run() {
    stop(Stop::Immediate);
    if (!can_run()) return;
    if (etxb_set_options(_ctx, &_options) != ETXB_OK) return;
    if (etxb_begin(_ctx, 0) != ETXB_OK) return;
    _status = {};
    _seen_iterations = 0;
    _have_camera_image = _have_light_image = true;
    _state = State::Running;
  }

  // Non-blocking, like CPUVCM::update (vcm_cpu.cxx:264-276): while the iteration queued earlier is still running this only refreshes the status;
  // when it has completed, the next one is queued (etxb_enqueue_iteration returns at once: the module runs it on its own worker thread).
  void update() {
    if (_state.load() == State::Stopped) return;
    etxb_status st = {};
    if (etxb_poll(_ctx, &st) != ETXB_OK) {
      _state = State::Stopped;
      return;
    }
    _status.last_iteration_time = st.last_iteration_time;
    _status.total_time = st.total_time;
    _status.completed_iterations = st.completed_iterations;
    _status.current_iteration = st.current_iteration;
    if (st.iteration_in_flight) return;
    if (st.completed_iterations > _seen_iterations) {
      _seen_iterations = st.completed_iterations;
      _have_camera_image = _have_light_image = true;
    }
    // complete_camera_vertices (vcm_cpu.cxx:227-241)
    if ((_state.load() == State::WaitingForCompletion) || (st.completed_iterations >= _samples)) {
      _state = State::Stopped;
      return;
    }
    if (etxb_enqueue_iteration(_ctx) != ETXB_OK) _state = State::Stopped;
  }

  void stop(Stop st) {
    if (_state.load() == State::Stopped) return;
    _state = (st == Stop::Immediate) ? State::Stopped : State::WaitingForCompletion;
    if (_state.load() == State::Stopped && _ctx) etxb_stop(_ctx, 0);  // drops what is queued; the iteration in flight completes (its film update is whole)
  }

  void update_options() {
    if (_state.load() == State::Running) run();
  }

  bool have_updated_camera_image() const {
    bool r = _have_camera_image;
    _have_camera_image = false;
    return r;
  }
  bool have_updated_light_image() const {
    bool r = _have_light_image;
    _have_light_image = false;
    return r;
  }
  const Status& status() const { return _status; }

  // Film::layer(Result) (film.cxx:381-418): row-major float4, y flipped in storage like the reference
  int read_film(uint32_t layer, float* rgba, uint64_t bytes) { return enabled() ? etxb_read_film(_ctx, layer, rgba, bytes) : _create_result; }
  etxb_ctx* context() { return _ctx; }

 private:
  etxb_ctx* _ctx = nullptr;
  int _create_result = ETXB_ERR_NO_DEVICE;
  etxb_vcm_options _options = {};
  std::atomic<State> _state{State::Stopped};
  Status _status;
  uint32_t _samples = 0, _seen_iterations = 0;
  bool _scene_committed = false;
  mutable bool _have_camera_image = false, _have_light_image = false;
};

}  // namespace etxb
