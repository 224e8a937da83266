// integrator_adapter.hpp — what the two host adapters (gpu_vcm.hpp, gpu_pt.hpp) share: the members, types and state machine of the reference's
// `etx::Integrator` (sources/etx/rt/integrators/integrator.hxx:12-98) over one module context, forwarded to the C ABI in include/etx_b200.h.
// The adapters add their options, commit_scene(), run() and update(): that is where CPUVCM and CPUPathTracing differ.
//
// Contract kept from the reference:
//  * stop(WaitForCompletion) lets the current iteration finish, stop(Immediate) returns after the queue drained (vcm_cpu.cxx:278-288,
//    path_tracing.cxx:154-166)
//  * update_options() restarts a running render                                                              (vcm_cpu.cxx:290-294, path_tracing.cxx:168-172)
#pragma once
#include <atomic>
#include <cstdint>

#include "../../include/etx_b200.h"

namespace etxb {

class IntegratorAdapter {
 public:
  enum class State : uint32_t { Stopped, Running, WaitingForCompletion };  // Integrator::State (integrator.hxx:14-18)
  enum class Stop : uint32_t { Immediate, WaitForCompletion };             // Integrator::Stop (integrator.hxx:20-23)

  struct Status {  // Integrator::Status (integrator.hxx:24-37)
    double last_iteration_time = 0.0;
    double total_time = 0.0;
    uint32_t completed_iterations = 0;
    uint32_t current_iteration = 0;
  };

  explicit IntegratorAdapter(int device_index) {
    etxb_device_config cfg = {};
    cfg.device_index = device_index;
    _create_result = etxb_create(&_ctx, &cfg);
  }
  virtual ~IntegratorAdapter() {
    stop(Stop::Immediate);
    if (_ctx) etxb_destroy(_ctx);
  }
  IntegratorAdapter(const IntegratorAdapter&) = delete;
  IntegratorAdapter& operator=(const IntegratorAdapter&) = delete;

  bool enabled() const { return _create_result == ETXB_OK; }
  const char* status_str() const { return _ctx ? etxb_last_error(_ctx) : "no CUDA device"; }
  State state() const { return _state.load(); }
  bool can_run() const { return enabled() && _scene_committed; }

  // stops immediately, then (if a scene is committed) starts the render at iteration 0
  virtual void run() = 0;

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
  // Film::set_pixel_size + restart, as the application does when the camera starts (8) and stops (1) moving (app.cxx:131-141): the size is
  // taken by the next run(), which a running render gets at once
  int set_film_pixel_size(uint32_t size) {
    if (!enabled()) return _create_result;
    const bool was_running = (_state.load() != State::Stopped);
    int rc = etxb_set_film_pixel_size(_ctx, size);
    if ((rc == ETXB_OK) && was_running) run();
    return rc;
  }
  int upload_tables(const float* xyz_441x3, const float* rgb_response_391x3, const uint8_t* sobol, const uint8_t* scrambling, const uint8_t* ranking) {
    if (!enabled()) return _create_result;
    int rc = etxb_upload_color_tables(_ctx, xyz_441x3, rgb_response_391x3);
    if (rc == ETXB_OK && sobol) rc = etxb_upload_blue_noise(_ctx, sobol, scrambling, ranking);
    return rc;
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
  const Status& status() const { return _status; }

  // Film::layer (film.cxx:381-418; the path tracer adds NORMALS / ALBEDO / CAMERA_ADAPTIVE): row-major float4, y flipped in storage like the reference
  int read_film(uint32_t layer, float* rgba, uint64_t bytes) { return enabled() ? etxb_read_film(_ctx, layer, rgba, bytes) : _create_result; }
  // Film::denoise (film.cxx:420-423, the application's Denoise button): `layer` (RESULT or CAMERA) into ETXB_FILM_DENOISED, on the device; waits for
  // the iteration in flight.  The filter is the module's own (DESIGN §13), not OpenImageDenoise.
  int denoise(uint32_t layer) { return enabled() ? etxb_denoise(_ctx, layer) : _create_result; }
  // The viewer (DESIGN §14): its reference image (Open Reference Image / Use as Reference), its six output views, and the error against the
  // reference (waits for the iteration in flight)
  int set_reference(const float* rgba, uint32_t width, uint32_t height) { return enabled() ? etxb_set_reference_image(_ctx, rgba, width, height) : _create_result; }
  int use_as_reference(uint32_t layer = ETXB_FILM_RESULT) { return enabled() ? etxb_use_film_as_reference(_ctx, layer) : _create_result; }
  int clear_reference() { return enabled() ? etxb_clear_reference(_ctx) : _create_result; }
  int view(uint32_t layer, const etxb_view& v, void* dst, uint64_t bytes) { return enabled() ? etxb_read_film_view(_ctx, layer, &v, dst, bytes) : _create_result; }
  int film_error(uint32_t layer, etxb_film_error_info* out) { return enabled() ? etxb_film_error(_ctx, layer, out) : _create_result; }
  etxb_ctx* context() { return _ctx; }

 protected:
  // Raytracing::link_scene / link_camera / commit_changes (rt.cxx:58-64, 323): `scene` / `camera` are the reference PODs
  int upload_scene(const void* scene, uint64_t scene_bytes, const void* camera, uint64_t camera_bytes) {
    stop(Stop::Immediate);
    _scene_committed = false;
    if (!enabled()) return _create_result;
    int rc = etxb_upload_scene(_ctx, scene, scene_bytes, camera, camera_bytes);
    _scene_committed = (rc == ETXB_OK);
    return rc;
  }
  // update()'s steps: poll the running render (false when it is stopped or the poll failed), note a newly completed iteration, and
  // either stop (scene.samples reached or WaitingForCompletion) or queue the next iteration (etxb_enqueue_iteration returns at once)
  bool poll(etxb_status& st) {
    if (_state.load() == State::Stopped) return false;
    if (etxb_poll(_ctx, &st) == ETXB_OK) return true;
    _state = State::Stopped;
    return false;
  }
  void copy_status(const etxb_status& st) { _status = {st.last_iteration_time, st.total_time, st.completed_iterations, st.current_iteration}; }
  bool iteration_completed(const etxb_status& st) {
    if (st.completed_iterations <= _seen_iterations) return false;
    _seen_iterations = st.completed_iterations;
    return true;
  }
  void finish_or_enqueue(const etxb_status& st) {
    if ((_state.load() == State::WaitingForCompletion) || (st.completed_iterations >= _samples)) {
      _state = State::Stopped;
      return;
    }
    if (etxb_enqueue_iteration(_ctx) != ETXB_OK) _state = State::Stopped;
  }

  etxb_ctx* _ctx = nullptr;
  int _create_result = ETXB_ERR_NO_DEVICE;
  std::atomic<State> _state{State::Stopped};
  Status _status;
  uint32_t _samples = 0, _seen_iterations = 0;
  bool _scene_committed = false;
  mutable bool _have_camera_image = false;
};

}  // namespace etxb
