// gpu_vcm.hpp — host-side C++ mirror of the reference's Integrator plugin for this path.
//
// `etxb::GPUVCM` has the member functions, threading contract and option keys of `etx::CPUVCM`
// (sources/etx/rt/integrators/vcm_cpu.hxx:7-27, vcm_cpu.cxx:247-310) and of its base `etx::Integrator`
// (sources/etx/rt/integrators/integrator.hxx:12-98), and forwards them to the C ABI in include/etx_b200.h.
// In the reference tree the class would derive from `etx::Integrator` (see INTEGRATION.md for the 3-line diff); here it derives from
// integrator_adapter.hpp's mirror of it because `integrator.hxx -> util/options.hxx` does not compile with gcc (options.hxx:77-88).
//
// Contract kept from the reference (stop() and update_options() are the base's):
//  * run() first stops immediately, then (if a scene is committed) clears the film and starts at iteration 0   (vcm_cpu.cxx:255-262)
//  * update() is called once per UI frame from the thread that pumps IntegratorThread; it advances the render and
//    fills Status; when `scene.samples` iterations are done the state becomes Stopped                          (vcm_cpu.cxx:264-276, 227-241)
//  * options are the reference's `vcm-*` keys                                                                  (vcm_shared.cxx:15-28)
#pragma once
#include "integrator_adapter.hpp"

namespace etxb {

class GPUVCM : public IntegratorAdapter {
 public:
  explicit GPUVCM(int device_index = 0) : IntegratorAdapter(device_index) { etxb_options_default(&_options); }

  const char* name() const { return "VCM (B200)"; }

  int commit_scene(const void* scene, uint64_t scene_bytes, const void* camera, uint64_t camera_bytes, uint32_t samples) {
    int rc = upload_scene(scene, scene_bytes, camera, camera_bytes);
    if (enabled()) _samples = samples;
    return rc;
  }

  // Integrator::options(): the reference's keys
  int set_option(const char* key, double value) { return etxb_options_set_key(&_options, key, value); }
  const etxb_vcm_options& options() const { return _options; }

  void run() override {
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
  // when it has completed, the next one is queued (the module runs it on its own worker thread).
  void update() {
    etxb_status st = {};
    if (!poll(st)) return;
    copy_status(st);
    if (st.iteration_in_flight) return;
    if (iteration_completed(st)) _have_camera_image = _have_light_image = true;
    finish_or_enqueue(st);  // complete_camera_vertices (vcm_cpu.cxx:227-241)
  }

  bool have_updated_light_image() const {
    bool r = _have_light_image;
    _have_light_image = false;
    return r;
  }

 private:
  etxb_vcm_options _options = {};
  mutable bool _have_light_image = false;
};

}  // namespace etxb
