// render_main.cpp — the headless renderer as a native program: scene file in, image file out.
//
// What the reference application does between File > Open and File > Save (sources/raytracer/app.cxx: load_scene_file :318-352, the integrator chosen
// by options.json "integrator" :88-99, IntegratorThread pumping Integrator::update, on_save_image_selected :261-295), without its window, on the module's
// C ABI: etxb_scene_file_load -> GPUVCM / GPUPathTracing::commit_scene_file -> run() -> update() until Stopped -> etxb_save_film.
// etx_tracer_b200/render.py is the same program through the ctypes mirror.
//
//   g++ -std=c++17 -O2 -pthread -I<repo> etx_tracer_b200/host/render_main.cpp <repo>/etx_tracer_b200/libetx_b200.so -Wl,-rpath,<repo>/etx_tracer_b200 -o etx_render
//   etx_render scene.json -o out.exr [--integrator vcm|pt] [--spp N] [--option key=value]... [--png-exposure E] [--layer N] [--denoise]
//   etx_render --options bin/options.json -o out.exr        the application's own options file names the scene and the integrator
//   --denoise filters the Result layer on the device (Film::denoise, the application's Denoise button) and saves the Denoised layer unless
//   --layer names another
//   --reference FILE     the viewer's reference image (also options.json's "ref"): prints the final error against it as one JSON line
//   --view NAME          write an output view of the layer (tonemapped, alpha, hdr, reference, relative, absolute): 8-bit to a .png, float to an .exr
//   --error-every N      with a reference: one JSON error line per N completed iterations
//
// Exit codes: 0 rendered and saved; 2 usage; 3 the scene could not be loaded; 4 no CUDA device (the module has no CPU path); 5 device error; 6 save failed.
#include <chrono>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "gpu_pt.hpp"
#include "gpu_vcm.hpp"

namespace {

struct Arguments {
  std::string scene, output = "out.exr", integrator = "vcm", options_file, reference;
  bool integrator_given = false, layer_given = false, denoise = false;
  std::vector<std::pair<std::string, double>> options;
  uint32_t spp = 0, layer = ETXB_FILM_RESULT, error_every = 0;
  int view = -1;
  float exposure = 1.0f;
  bool ok = false;
};

Arguments parse(int argc, char** argv) {
  Arguments a;
  for (int i = 1; i < argc; ++i) {
    std::string s = argv[i];
    auto next = [&]() -> const char* { return (i + 1 < argc) ? argv[++i] : nullptr; };
    if (s == "-o" || s == "--output") {
      const char* v = next();
      if (!v) return a;
      a.output = v;
    } else if (s == "--integrator") {
      const char* v = next();
      if (!v || (strcmp(v, "vcm") != 0 && strcmp(v, "pt") != 0)) return a;
      a.integrator = v;
      a.integrator_given = true;
    } else if (s == "--spp") {
      const char* v = next();
      if (!v) return a;
      a.spp = uint32_t(strtoul(v, nullptr, 10));
    } else if (s == "--layer") {
      const char* v = next();
      if (!v) return a;
      a.layer = uint32_t(strtoul(v, nullptr, 10));
      a.layer_given = true;
    } else if (s == "--denoise") {
      a.denoise = true;
    } else if (s == "--png-exposure") {
      const char* v = next();
      if (!v) return a;
      a.exposure = float(atof(v));
    } else if (s == "--reference") {
      const char* v = next();
      if (!v) return a;
      a.reference = v;
    } else if (s == "--view") {
      static const char* names[] = {"tonemapped", "alpha", "hdr", "reference", "relative", "absolute"};
      const char* v = next();
      if (!v) return a;
      for (int k = 0; k < 6; ++k)
        if (strcmp(v, names[k]) == 0) a.view = k;
      if (a.view < 0) return a;
    } else if (s == "--error-every") {
      const char* v = next();
      if (!v) return a;
      a.error_every = uint32_t(strtoul(v, nullptr, 10));
    } else if (s == "--options") {  // the application's options.json: "scene" and "integrator" (raytracer/app.cxx:88-105)
      const char* v = next();
      if (!v) return a;
      a.options_file = v;
    } else if (s == "--option") {
      const char* v = next();
      const char* eq = v ? strchr(v, '=') : nullptr;
      if (!eq) return a;
      a.options.push_back({std::string(v, eq), atof(eq + 1)});
    } else if (!s.empty() && s[0] == '-') {
      return a;
    } else {
      a.scene = s;
    }
  }
  if (!a.options_file.empty()) {
    char value[2048] = {};
    if (a.scene.empty() && etxb_options_file_string(a.options_file.c_str(), "scene", value, sizeof(value)) > 0) {
      // the application stores the path relative to its working directory, which is the folder of options.json
      std::string folder = a.options_file.substr(0, a.options_file.find_last_of('/') == std::string::npos ? 0 : a.options_file.find_last_of('/') + 1);
      a.scene = (value[0] == '/') ? std::string(value) : (folder + value);
    }
    if (a.reference.empty() && etxb_options_file_string(a.options_file.c_str(), "ref", value, sizeof(value)) > 0) {  // app.cxx:106-109
      std::string folder = a.options_file.substr(0, a.options_file.find_last_of('/') == std::string::npos ? 0 : a.options_file.find_last_of('/') + 1);
      a.reference = (value[0] == '/') ? std::string(value) : (folder + value);
    }
    if (!a.integrator_given && etxb_options_file_string(a.options_file.c_str(), "integrator", value, sizeof(value)) > 0) {
      // "VCM (CPU)" / "VCM (B200)" -> vcm, "Path Tracing (CPU)" / "Path Tracing (B200)" -> pt; the bidirectional integrator has no device twin:
      // VCM with merging off is the reference's own equivalent (vcm_shared.hxx:33)
      const std::string name = value;
      if (name.compare(0, 12, "Path Tracing") == 0) {
        a.integrator = "pt";
      } else if (name.compare(0, 13, "Bidirectional") == 0) {
        a.integrator = "vcm";
        a.options.insert(a.options.begin(), {"vcm-merging", 0.0});
      } else {
        a.integrator = "vcm";
      }
    }
  }
  if (a.denoise && !a.layer_given) a.layer = ETXB_FILM_DENOISED;
  a.ok = !a.scene.empty() && ((a.error_every == 0) || !a.reference.empty());
  return a;
}

bool ends_with(const std::string& s, const char* tail) {
  size_t n = strlen(tail);
  return s.size() >= n && s.compare(s.size() - n, n, tail) == 0;
}

// the Result layer's error against the reference as one JSON line (the fields and order of render.py's); `iterations` gets the film's
// iteration count.  A failure (which may be the error an iteration hit: the call waits for them) is returned, not printed.
template <class Integrator>
int print_error(Integrator& integrator, uint32_t& iterations) {
  etxb_film_error_info e = {};
  if (int rc = integrator.film_error(ETXB_FILM_RESULT, &e)) return rc;
  etxb_status st = {};
  etxb_poll(integrator.context(), &st);
  std::printf("{\"iteration\": %u, \"seconds\": %.17g, \"pixels\": %" PRIu64 ", \"nonfinite\": %" PRIu64 ", \"negative\": %" PRIu64
              ", \"lum_above\": %" PRIu64 ", \"lum_below\": %" PRIu64 ", \"mse\": %.17g, \"rel_mse\": %.17g, \"mean_abs_lum\": %.17g, \"mean_lum\": %.17g, "
              "\"reference_mean_lum\": %.17g, \"iterations\": %u}\n",
              e.iterations, st.total_time, e.pixels, e.nonfinite, e.negative, e.lum_above, e.lum_below, e.mse, e.rel_mse, e.mean_abs_lum, e.mean_lum,
              e.reference_mean_lum, e.iterations);
  std::fflush(stdout);
  iterations = e.iterations;
  return ETXB_OK;
}

// Open Reference Image (app.cxx:243-250): the file as the image pool holds it, into the integrator's reference slot
template <class Integrator>
int load_reference(Integrator& integrator, const std::string& file) {
  uint32_t w = 0, h = 0;
  char warning[1024] = {};
  if (etxb_reference_image_file_read(file.c_str(), &w, &h, nullptr, 0, warning, sizeof(warning)) != ETXB_OK) return ETXB_ERR_INVALID_ARGUMENT;
  std::vector<float> rgba(size_t(w) * h * 4u);
  if (etxb_reference_image_file_read(file.c_str(), &w, &h, rgba.data(), rgba.size() * 4u, warning, sizeof(warning)) != ETXB_OK) return ETXB_ERR_INVALID_ARGUMENT;
  if (warning[0]) std::fprintf(stderr, "warning: %s\n", warning);
  return integrator.set_reference(rgba.data(), w, h);
}

// IntegratorThread's loop (sources/etx/rt/integrators/integrator_thread.cxx): update() until the integrator reports Stopped
template <class Integrator>
int pump(Integrator& integrator, const Arguments& args, etxb_scene_file* file, uint32_t samples) {
  if (!integrator.enabled()) {
    std::fprintf(stderr, "%s: no CUDA device (the module has no CPU path)\n", integrator.name());
    return 4;
  }
  for (const auto& kv : args.options) {
    if (integrator.set_option(kv.first.c_str(), kv.second) != 0) {
      std::fprintf(stderr, "unknown option `%s` for %s\n", kv.first.c_str(), integrator.name());
      return 2;
    }
  }
  if (integrator.commit_scene_file(file) != ETXB_OK) {
    std::fprintf(stderr, "%s: %s\n", integrator.name(), integrator.status_str());
    return 5;
  }
  if (!args.reference.empty() && (load_reference(integrator, args.reference) != ETXB_OK)) {
    std::fprintf(stderr, "could not use %s as the reference: %s\n", args.reference.c_str(), integrator.status_str());
    return 5;
  }
  integrator.run();
  auto t0 = std::chrono::steady_clock::now();
  uint32_t reported = 0;
  while (integrator.state() != Integrator::State::Stopped) {
    integrator.update();
    if ((args.error_every != 0) && (integrator.status().completed_iterations >= reported + args.error_every) && (print_error(integrator, reported) != ETXB_OK)) {
      std::fprintf(stderr, "%s: the error against the reference failed: %s\n", integrator.name(), integrator.status_str());
      return 5;
    }
    std::this_thread::sleep_for(std::chrono::microseconds(200));
  }
  double seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  const auto& st = integrator.status();
  if (st.completed_iterations == 0) {
    std::fprintf(stderr, "%s: %s\n", integrator.name(), integrator.status_str());
    return 5;
  }
  const etxb_camera* cam = etxb_scene_file_camera(file);
  std::printf("%s: %u of %u iterations, %u x %u, %.3f s\n", integrator.name(), st.completed_iterations, samples, cam->film_size[0], cam->film_size[1], seconds);
  if (args.denoise && (integrator.denoise(ETXB_FILM_RESULT) != ETXB_OK)) {
    std::fprintf(stderr, "could not denoise: %s\n", integrator.status_str());
    return 5;
  }
  if (!args.reference.empty() && (print_error(integrator, reported) != ETXB_OK)) {
    std::fprintf(stderr, "%s: the error against the reference failed: %s\n", integrator.name(), integrator.status_str());
    return 5;
  }
  uint32_t mode = ends_with(args.output, ".png") ? ETXB_SAVE_PNG_TONEMAPPED : ETXB_SAVE_EXR;
  if (args.view >= 0) {
    const etxb_view v = {uint32_t(args.view), ETXB_VIEW_OPT_TONEMAPPING | ETXB_VIEW_OPT_SRGB, args.exposure, mode == ETXB_SAVE_PNG_TONEMAPPED ? 1u : 0u};
    const size_t n = size_t(cam->film_size[0]) * cam->film_size[1];
    std::vector<float> pixels(n * 4u);  // float4, or RGBA8 in its first quarter
    int rc = integrator.view(args.layer, v, pixels.data(), pixels.size() * 4u);
    if (rc == ETXB_OK)
      rc = v.rgba8 ? etxb_write_png(args.output.c_str(), reinterpret_cast<const uint8_t*>(pixels.data()), cam->film_size[0], cam->film_size[1])
                   : etxb_write_exr(args.output.c_str(), pixels.data(), cam->film_size[0], cam->film_size[1]);
    if (rc != ETXB_OK) {
      std::fprintf(stderr, "could not write the view to %s: %s\n", args.output.c_str(), integrator.status_str());
      return 6;
    }
    return 0;
  }
  if (etxb_save_film(integrator.context(), args.layer, args.output.c_str(), mode, args.exposure) != ETXB_OK) {
    std::fprintf(stderr, "could not save %s: %s\n", args.output.c_str(), integrator.status_str());
    return 6;
  }
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  Arguments args = parse(argc, argv);
  if (!args.ok) {
    std::fprintf(stderr, "usage: %s scene.json [-o out.exr|out.png] [--integrator vcm|pt] [--spp N] [--option key=value] [--options options.json] [--png-exposure E] [--layer N] [--denoise] [--reference FILE] [--view NAME] [--error-every N]\n", argv[0]);
    return 2;
  }
  char error[1024] = {};
  etxb_scene_file* file = nullptr;
  if (etxb_scene_file_load(args.scene.c_str(), nullptr, &file, error, sizeof(error)) != ETXB_OK) {
    std::fprintf(stderr, "%s\n", error);
    return 3;
  }
  for (uint32_t i = 0; i < etxb_scene_file_warning_count(file); ++i) std::fprintf(stderr, "warning: %s\n", etxb_scene_file_warning(file, i));
  if (args.spp != 0) etxb_scene_file_set_samples(file, args.spp);
  uint32_t samples = etxb_scene_file_scene(file)->samples;
  int rc;
  if (args.integrator == "pt") {
    etxb::GPUPathTracing integrator(0);
    rc = pump(integrator, args, file, samples);
  } else {
    etxb::GPUVCM integrator(0);
    rc = pump(integrator, args, file, samples);
  }
  etxb_scene_file_free(file);
  return rc;
}
