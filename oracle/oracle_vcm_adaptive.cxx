// oracle_vcm_adaptive.cxx — the VCM's CameraAdaptive layer restated on top of the oracle.  TEST INFRASTRUCTURE.
//
// The reference's Film keeps CameraAdaptive, the mean of the even-indexed samples, for every integrator: CPUVCM's camera pass calls
// Film::accumulate_camera_image like the path tracer does (vcm_cpu.cxx:195-198, film.cxx:173-230), and the device's VCM keeps it for the
// denoiser's variance estimate (DESIGN §13).  oracle_preview.cxx (which compiles oracle_vcm.cxx) is compiled here as it is; this file adds
// oracle_adaptive_run_iterations: the same iterations, and after each VCM iteration film.cxx's even-sample lerp of every film pixel from its
// path's camera value (the pixel's block at pixel size > 1), with that pixel's own sample count.  The path tracer already keeps the layer.
// Built into liboracle_vcm_adaptive_parity.so by build_oracle_vcm_adaptive.sh.
#include "oracle_preview.cxx"

namespace etx {
namespace {

// film.cxx:173-230, the CameraAdaptive part: `sample_index` is the pixel's count before this sample
void film_accumulate_adaptive(Oracle& o, const uint2& pixel, const float3& color) {
  if ((pixel.x >= o.width) || (pixel.y >= o.height))
    return;
  const uint32_t i = pixel.x + (o.height - 1u - pixel.y) * o.width;
  const uint32_t sample_index = o.film_samples[i] - 1u;  // film_accumulate_camera has counted this sample already
  if (sample_index == 0) {
    o.film_adaptive[i] = color;
  } else if ((sample_index % 2) == 0) {
    const double ds = double(sample_index);
    const float t = float(ds / (ds + 2.0));
    o.film_adaptive[i] = {lerp(color.x, o.film_adaptive[i].x, t), lerp(color.y, o.film_adaptive[i].y, t), lerp(color.z, o.film_adaptive[i].z, t)};
  }
}

}  // namespace
}  // namespace etx

extern "C" {

double oracle_adaptive_run_iterations(void* h, uint32_t count, uint32_t threads) {
  auto* o = static_cast<Oracle*>(h);
  for (uint32_t k = 0; k < count; ++k) {
    const uint32_t iteration = o->iteration.iteration;
    oracle_run_iterations(h, 1u, threads);
    if (o->integrator == ETXB_INTEGRATOR_PT)
      continue;
    const uint32_t s = preview_of(h).pixel_size;
    for (uint32_t pi = 0, n = static_cast<uint32_t>(o->camera_value.size()); pi < n; ++pi) {
      uint2 pixel = {pi % o->width, pi / o->width};  // Film::active_pixel at pixel size 1
      if (s != 1u)
        active_pixel(*o, s, pi, iteration, pixel);
      for_block(*o, s, pixel, [&](const uint2& p) { film_accumulate_adaptive(*o, p, o->camera_value[pi]); });
    }
  }
  return o->total_time;
}

}  // extern "C"
