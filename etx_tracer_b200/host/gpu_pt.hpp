// gpu_pt.hpp — host-side C++ mirror of the reference's unidirectional path-tracing plugin (SURVEY 8(f) N3).
//
// `etxb::GPUPathTracing` has the member functions, threading contract and option ids of `etx::CPUPathTracing`
// (sources/etx/rt/integrators/path_tracing.hxx, path_tracing.cxx:122-170) and of its base `etx::Integrator`
// (sources/etx/rt/integrators/integrator.hxx:12-98) and forwards them to the C ABI in include/etx_b200.h
// (etxb_set_integrator(ETXB_INTEGRATOR_PT) + the calls the VCM adapter uses).  Like gpu_vcm.hpp it derives from integrator_adapter.hpp's mirror
// of the base because `integrator.hxx -> util/options.hxx` does not compile with gcc; INTEGRATION.md shows the derivation a maintainer adds.
//
// Contract kept from the reference (stop() and update_options() are the base's):
//  * run() first stops immediately, then (if a scene is committed) reads the options, clears the camera data of the film and schedules
//    iteration 0                                                                                              (path_tracing.cxx:35-48, 141-148)
//  * update() never blocks; when the task of the current iteration has completed it accounts the iteration, lets the film estimate the
//    noise levels, and either stops (scene.samples reached, WaitingForCompletion, or an iteration that processed no pixel because all
//    have converged) or schedules the next iteration                                                          (path_tracing.cxx:85-110)
//  * option ids "direct", "nee", "mis", "bn"                                                                  (path_tracing.cxx:36-39, 112-119)
#pragma once
#include "integrator_adapter.hpp"

namespace etxb {

class GPUPathTracing : public IntegratorAdapter {
 public:
  explicit GPUPathTracing(int device_index = 0) : IntegratorAdapter(device_index) {
    if (_create_result == ETXB_OK) _create_result = etxb_set_integrator(_ctx, ETXB_INTEGRATOR_PT);
    etxb_pt_options_default(&_options);
  }

  const char* name() const { return "Path Tracing (B200)"; }

  // scene.samples, noise_threshold and radiance_clamp travel inside the Scene record
  int commit_scene(const void* scene, uint64_t scene_bytes, const void* camera, uint64_t camera_bytes) {
    int rc = upload_scene(scene, scene_bytes, camera, camera_bytes);
    if (_scene_committed && (scene_bytes == sizeof(etxb_scene))) _samples = static_cast<const etxb_scene*>(scene)->samples;
    return rc;
  }

  int set_option(const char* key, double value) { return etxb_pt_options_set_key(&_options, key, value); }
  const etxb_pt_options& options() const { return _options; }

  void run() override {
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
    etxb_status st = {};
    if (!poll(st)) return;
    if (st.iteration_in_flight) return;  // the task has not completed (path_tracing.cxx:86-88)
    copy_status(st);
    if (iteration_completed(st)) _have_camera_image = true;
    etxb_pt_status pt = {};
    etxb_pt_get_status(_ctx, &pt);
    if (pt.pixels_processed == 0u) _state = State::WaitingForCompletion;  // every pixel has converged (path_tracing.cxx:90-92)
    finish_or_enqueue(st);
  }

  bool have_updated_light_image() const { return false; }  // the path tracer never writes the light image
  // Film::noise_level / active_pixel_count (film.cxx:430, 461)
  float noise_level() const {
    etxb_pt_status pt = {};
    return (_ctx && (etxb_pt_get_status(_ctx, &pt) == ETXB_OK)) ? pt.noise_level : 0.0f;
  }

 private:
  etxb_pt_options _options = {};
};

}  // namespace etxb
