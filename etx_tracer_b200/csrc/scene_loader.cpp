// scene_loader.cpp — the reference's scene files read into the Scene / Camera PODs, host code of the module (SURVEY 8(f) N2; no CUDA here).
//
// What it replaces: SceneRepresentation::load_from_file and what it calls (sources/etx/render/host/scene_representation.cxx: load_from_file :679-838,
// load_from_obj :964-1052, parse_camera :1054-1159, parse_medium :1161-1306, parse_directional_light :1308-1343, parse_env_light :1345-1378,
// parse_spectrum :1496-1611, load_reflectance_spectrum / load_illuminant_spectrum :1613-1680, parse_material :1682-2079, validate_materials :262-302,
// validate_normals / validate_tangents :304-418, commit :420-455, add_area_emitters_for_triangle :840-905, build_emitters_distribution :2460-2497),
// the spectrum builders of render/host/spectrum.cxx:11-154, ImagePool's loading + sampling tables (render/host/image_pool.cxx:162-259) and
// MediumPool / SceneLoaderContext::add_medium (scene_data.hxx:125-147) — for the `.json` + `.obj` + `.mtl` dialect.  The .mtl reader follows the
// reference's patched tinyobjloader (thirdparty/tinyobjloader/tiny_obj_loader.hxx:1900-2190, quads :1464-1527).
//
// tests/test_loader.py loads the same files with the reference's OWN loader (compiled in place, test infrastructure) and compares array by array —
// hand-written scenes, the shipped Cornell asset, and seeded random material / geometry files.
// Parts (each .inl is included below, inside this file's anonymous namespace):
//   scene_loader_formats.inl     DEFLATE, PNG (every form stb_image decodes), TGA, BMP, OpenEXR scan lines (none / RLE / ZIPS / ZIP / PIZ), Radiance HDR,
//                                the reference's PFM variant, JSON, the .mtl / .obj dialect of the patched tinyobjloader (ear-clipped polygons)
//   scene_loader_jpeg.inl        baseline / progressive JPEG with stb_image's IDCT, upsampling and colour conversion (same bytes)
//   scene_loader_tangents.inl    the tangent-space generator the reference calls for meshes with texture coordinates (identical frames)
//   scene_loader_nvdb.inl        NanoVDB 32.x float grids -> the dense grid of a heterogeneous medium
//   scene_loader_atmosphere.inl  `et::atmosphere`, and the default sun + sky of a file without distant emitters (render/host/scattering.cxx)
//   scene_loader_build.inl       the directives -> Scene / Camera PODs
// Refused with a message: glTF (DESIGN.md 10 says why), BLOSC-compressed volumes.  Textures in a format that is not read (GIF, PSD, CMYK JPEG, lossy EXR
// codecs) become the 1 x 1 white placeholder the reference uses for files it cannot read.  The data tables the reference derives at start-up (CIE /
// RGB-response tables, the IOR database on the 1 nm grid, the atmosphere spectra, blue-noise tiles) ship as etx_tracer_b200/data/tables.bin
// (tools/make_tables_bin.py).  etx_tracer_b200/loader.py is the same loader in Python, sharing the readers above through the C ABI.
#include <algorithm>
#include <atomic>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include <dlfcn.h>
#include <unistd.h>

#include "../../include/etx_b200.h"

namespace {

constexpr uint32_t kInvalid = 0xffffffffu;
constexpr float kPiF = 3.1415926535897932384626433832795f;
constexpr float kEps = 1.192092896e-07f;  // kEpsilon (math.hxx:107)
enum : uint32_t { IMG_BUILD_TABLE = 1, IMG_REPEAT_U = 2, IMG_REPEAT_V = 4, IMG_SKIP_SRGB = 8, IMG_HAS_ALPHA = 16, IMG_UNIFORM_TABLE = 32, IMG_PERFORM_LOADING = 64 };
enum : uint32_t { SPD_INVALID = 0, SPD_REFLECTANCE = 1, SPD_CONDUCTOR = 2, SPD_DIELECTRIC = 3, SPD_ILLUMINANT = 4 };

struct LoadError {
  std::string text;
};
[[noreturn]] void fail(const std::string& text) { throw LoadError{text}; }

struct F3 {
  float x = 0.0f, y = 0.0f, z = 0.0f;
};
inline F3 operator+(F3 a, F3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
inline F3 operator-(F3 a, F3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline F3 operator*(F3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
inline F3 operator/(F3 a, float s) { return {a.x / s, a.y / s, a.z / s}; }
inline float dot(F3 a, F3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline F3 cross(F3 a, F3 b) { return {a.y * b.z - b.y * a.z, a.z * b.x - b.z * a.x, a.x * b.y - b.x * a.y}; }
inline float length(F3 a) { return sqrtf(dot(a, a)); }
inline F3 normalize(F3 a) { return a / length(a); }
inline bool finite3(F3 a) { return std::isfinite(a.x) && std::isfinite(a.y) && std::isfinite(a.z); }
inline bool valid_vector(F3 a) { return finite3(a) && (dot(a, a) > 0.0f); }  // math.hxx:877-879
inline F3 load3(const float* p) { return {p[0], p[1], p[2]}; }
inline void store3(float* p, F3 v) { p[0] = v.x, p[1] = v.y, p[2] = v.z; }
inline float luminance(F3 v) { return v.x * 0.212671f + v.y * 0.715160f + v.z * 0.072169f; }  // math.hxx:729
inline float saturate(float v) { return v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v); }
inline float clampf(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

// ---- the module's data tables (etx_tracer_b200/data/tables.bin) -----------------------------------------------------------------------------------
struct Tables {
  std::map<std::string, std::vector<float>> f32;
  std::map<std::string, std::vector<uint32_t>> u32;
  std::map<std::string, std::vector<uint8_t>> u8;
  const std::vector<float>& get(const std::string& name) const {
    auto i = f32.find(name);
    if (i == f32.end()) fail("data table `" + name + "` is missing from tables.bin");
    return i->second;
  }
  bool has(const std::string& name) const { return f32.count(name) != 0; }
};

std::string module_directory() {
  Dl_info info = {};
  if (dladdr(reinterpret_cast<const void*>(&module_directory), &info) && info.dli_fname) {
    std::string path = info.dli_fname;
    size_t slash = path.find_last_of('/');
    if (slash != std::string::npos) return path.substr(0, slash);
  }
  return ".";
}

std::shared_ptr<Tables> load_tables(const char* data_folder) {
  static std::mutex guard;  // loads may come from several host threads
  static std::map<std::string, std::shared_ptr<Tables>> cache;
  std::lock_guard<std::mutex> lock(guard);
  std::string folder = (data_folder && data_folder[0]) ? std::string(data_folder) : (module_directory() + "/data");
  auto hit = cache.find(folder);
  if (hit != cache.end()) return hit->second;
  std::string path = folder + "/tables.bin";
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) fail("cannot open " + path + " (tools/make_data.py writes it)");
  auto t = std::make_shared<Tables>();
  uint32_t header[2] = {};
  if (fread(header, 4, 2, f) != 2 || header[0] != 0x54585445u) {
    fclose(f);
    fail(path + " is not a table file");
  }
  for (uint32_t k = 0; k < header[1]; ++k) {
    uint16_t name_len = 0;
    uint32_t meta[2] = {};
    std::string name;
    if (fread(&name_len, 2, 1, f) != 1) break;
    name.resize(name_len);
    if (fread(&name[0], 1, name_len, f) != name_len || fread(meta, 4, 2, f) != 2) break;
    if (meta[0] == 0u) {
      auto& v = t->f32[name];
      v.resize(meta[1]);
      if (fread(v.data(), 4, meta[1], f) != meta[1]) break;
    } else if (meta[0] == 1u) {
      auto& v = t->u32[name];
      v.resize(meta[1]);
      if (fread(v.data(), 4, meta[1], f) != meta[1]) break;
    } else {
      auto& v = t->u8[name];
      v.resize(meta[1]);
      if (fread(v.data(), 1, meta[1], f) != meta[1]) break;
    }
  }
  fclose(f);
  cache[folder] = t;
  return t;
}

// ---- spectra (render/host/spectrum.cxx) ---------------------------------------------------------------------------------------------------------------
using Spd = etxb_spectrum;

Spd spd_from_power(const float* power441, const float* integrated) {
  Spd s = {};
  for (int i = 0; i < 441; ++i) {
    s.entries[i].wavelength = float(390 + i);
    s.entries[i].power = power441[i];
  }
  s.entry_count = 441;
  if (integrated) memcpy(s.integrated, integrated, 12);
  return s;
}

F3 xyz_to_rgb(F3 xyz) {  // spectrum.hxx:142-148
  return {3.24045420f * xyz.x - 1.5371385f * xyz.y - 0.4985314f * xyz.z, -0.9692660f * xyz.x + 1.8760108f * xyz.y + 0.0415560f * xyz.z,
          0.05564340f * xyz.x - 0.2040259f * xyz.y + 1.0572252f * xyz.z};
}

// SpectralDistribution::integrate_to_xyz (spectrum.cxx:348-377) on the 1 nm grid
F3 integrate_to_xyz(const Tables& t, const Spd& s) {
  const std::vector<float>& xyz = t.get("color_tables/xyz_441x3");
  const float k_y = 1.0f / t.get("color_tables/y_integral")[0];
  auto to_xyz = [&](int i, float value) -> F3 {
    if (value == 0.0f) return {};
    F3 c = {xyz[3 * i + 0], xyz[3 * i + 1], xyz[3 * i + 2]};
    return c * (value * k_y);
  };
  F3 result = {};
  for (int i = 0; i + 1 < 441; ++i) {
    F3 v0 = to_xyz(i, s.entries[i].power), v1 = to_xyz(i + 1, s.entries[i + 1].power);
    result = result + (v0 + (v1 - v0) * 0.5f) * 1.0f;
  }
  return result;
}

Spd spd_integrated(const Tables& t, const float* power441) {
  Spd s = spd_from_power(power441, nullptr);
  F3 rgb = xyz_to_rgb(integrate_to_xyz(t, s));
  store3(s.integrated, rgb);
  return s;
}

Spd spd_constant(float value) {  // spectrum.cxx:108-116
  float p[441];
  for (float& v : p) v = value;
  float rgb[3] = {value, value, value};
  return spd_from_power(p, rgb);
}

Spd spd_rgb_reflectance(const Tables& t, F3 rgb) {  // spectrum.cxx:135-148 via rgb_response (spectrum.cxx:399-)
  if (luminance(rgb) == 0.0f) return spd_constant(0.0f);
  const std::vector<float>& w = t.get("color_tables/rgb_response_391x3");
  float p[441];
  for (int i = 0; i < 391; ++i) p[i] = rgb.x * w[3 * i + 0] + rgb.y * w[3 * i + 1] + rgb.z * w[3 * i + 2];
  for (int i = 391; i < 441; ++i) p[i] = p[390];  // from_samples holds the last sample
  float integrated[3] = {rgb.x, rgb.y, rgb.z};
  return spd_from_power(p, integrated);
}

Spd spd_rgb_luminance(const Tables& t, F3 rgb) {  // spectrum.cxx:150-154; kRGBLuminanceScale spectrum.hxx:450
  Spd s = spd_rgb_reflectance(t, {rgb.x * 0.817660332f, rgb.y * 1.05418909f, rgb.z * 1.09945524f});
  store3(s.integrated, rgb);
  return s;
}

void spd_scale(Spd& s, float factor) {  // spectrum.cxx:97-102
  for (uint32_t i = 0; i < s.entry_count; ++i) s.entries[i].power *= factor;
  for (float& v : s.integrated) v *= factor;
}

float spd_max_power(const Spd& s) {  // spectrum.cxx:340-346
  float r = s.entries[0].power;
  for (uint32_t i = 0; i < s.entry_count; ++i) r = std::max(r, s.entries[i].power);
  return r;
}

float black_body_radiation(float wavelength_nm, float t_kelvins) {  // spectrum.hxx:171-189
  constexpr float Lc1 = 3.7417712e+5f, Lc2 = 1.4387752e+4f;
  wavelength_nm *= 1.0f / 1000.0f;
  float wl5 = wavelength_nm * (wavelength_nm * wavelength_nm) * (wavelength_nm * wavelength_nm);
  float e0 = expf(Lc2 / (wavelength_nm * t_kelvins));
  float d = wl5 * (e0 - 1.0f);
  return std::isinf(d) ? 0.0f : (Lc1 / d);
}

Spd spd_black_body(const Tables& t, float temperature, float scale) {  // spectrum.cxx:118-125
  float p[441];
  for (int i = 0; i < 441; ++i) p[i] = black_body_radiation(float(i + 390), temperature) * scale;
  return spd_integrated(t, p);
}

Spd spd_normalized_black_body(const Tables& t, float temperature, float scale) {  // spectrum.cxx:127-133
  float w = 2.8977729e+6f / temperature;
  float r = black_body_radiation(w, temperature);
  Spd s = spd_black_body(t, temperature, 1.0f / r);
  spd_scale(s, scale / luminance(load3(s.integrated)));
  return s;
}

// SpectralDistribution::from_samples (spectrum.cxx:11-95)
Spd spd_from_samples(const Tables& t, const std::vector<std::pair<float, float>>& in) {
  if (in.empty()) return spd_constant(0.0f);
  float mult = 1.0f;
  while ((in[0].first * mult) < 100.0f) mult *= 10.0f;
  std::vector<std::pair<float, float>> pts;
  for (const auto& s : in) {
    float w = s.first * mult, p = s.second;
    if (!std::isfinite(w) || !std::isfinite(p)) continue;
    pts.push_back({clampf(w, 390.0f, 830.0f), p});
  }
  if (pts.empty()) return spd_constant(0.0f);
  std::sort(pts.begin(), pts.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  std::vector<std::pair<float, float>> u;
  for (const auto& s : pts) {
    if (u.empty() || fabsf(s.first - u.back().first) > 1.0e-4f) {
      u.push_back(s);
    } else {
      u.back().second = s.second;
    }
  }
  if (u.size() == 1) u.push_back(u.front());
  float power[441];
  size_t seg = 0;
  for (int i = 0; i < 441; ++i) {
    float wl = float(390 + i), p = 0.0f;
    if (wl <= u.front().first) {
      p = u.front().second;
    } else if (wl >= u.back().first) {
      p = u.back().second;
    } else {
      while ((seg + 1 < u.size()) && (u[seg + 1].first < wl)) ++seg;
      float den = u[seg + 1].first - u[seg].first;
      float tt = (den > 0.0f) ? (wl - u[seg].first) / den : 0.0f;
      tt = saturate(tt);
      p = u[seg].second * (1.0f - tt) + u[seg + 1].second * tt;
    }
    power[i] = p;
  }
  return spd_integrated(t, power);
}

// ---- text helpers with the C library's semantics -----------------------------------------------------------------------------------------------------------
std::vector<std::string> split(const std::string& s) {
  std::vector<std::string> out;
  size_t i = 0;
  while (i < s.size()) {
    while (i < s.size() && isspace(static_cast<unsigned char>(s[i]))) ++i;
    size_t b = i;
    while (i < s.size() && !isspace(static_cast<unsigned char>(s[i]))) ++i;
    if (i > b) out.push_back(s.substr(b, i - b));
  }
  return out;
}
// split_params (scene_representation.cxx:463-478): cut at every single space, empty pieces kept (two spaces in a row make an empty parameter,
// which atof reads as 0 and which shifts the positions of what follows) — the reference's tokenizer for every multi-word directive value
std::vector<std::string> split_params(const std::string& s) {
  std::vector<std::string> out;
  size_t begin = 0;
  for (size_t i = 0; i < s.size(); ++i) {
    if (s[i] == ' ') {
      out.push_back(s.substr(begin, i - begin));
      begin = i + 1;
    }
  }
  out.push_back(s.substr(begin));
  return out;
}

std::string lower(std::string s) {
  for (char& c : s) c = char(tolower(static_cast<unsigned char>(c)));
  return s;
}
std::string trim(const std::string& s) {
  size_t b = 0, e = s.size();
  while (b < e && isspace(static_cast<unsigned char>(s[b]))) ++b;
  while (e > b && isspace(static_cast<unsigned char>(s[e - 1]))) --e;
  return s.substr(b, e - b);
}
float c_atof(const std::string& s) { return static_cast<float>(atof(s.c_str())); }
// sscanf("%f %f ...") : as many leading floats as parse (a token must parse completely up to a separator, like %f stops at the first bad character)
std::vector<float> leading_floats(const std::string& text, size_t limit) {
  std::vector<float> out;
  const char* p = text.c_str();
  while (out.size() < limit) {
    char* end = nullptr;
    float v = strtof(p, &end);
    if (end == p) break;
    out.push_back(v);
    p = end;
  }
  return out;
}
bool leading_uint(const std::string& s, uint32_t& out) {
  auto t = split(s);
  if (t.empty() || !isdigit(static_cast<unsigned char>(t[0][0]))) return false;
  out = uint32_t(strtoul(t[0].c_str(), nullptr, 10));
  return true;
}

F3 gamma_to_linear(F3 v) {  // math.hxx gamma_to_linear
  auto g = [](float c) { return c <= 0.04045f ? c / 12.92f : powf((c + 0.055f) / 1.055f, 2.4f); };
  return {g(v.x), g(v.y), g(v.z)};
}

std::string read_file(const std::string& path) {
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) fail("cannot open " + path);
  std::string data;
  char buffer[1 << 16];
  size_t n;
  while ((n = fread(buffer, 1, sizeof(buffer), f)) > 0) data.append(buffer, n);
  fclose(f);
  return data;
}
std::string folder_of(const std::string& path) {
  size_t slash = path.find_last_of('/');
  return slash == std::string::npos ? std::string("") : path.substr(0, slash);
}
std::string join(const std::string& folder, const std::string& name) {
  if (!name.empty() && name[0] == '/') return name;
  return folder.empty() ? name : (folder + "/" + name);
}

#include "scene_loader_formats.inl"
#include "scene_loader_tangents.inl"
#include "scene_loader_nvdb.inl"
#include "scene_loader_build.inl"

}  // namespace

// ---- the C ABI (include/etx_b200.h "scene files") ------------------------------------------------------------------------------------------------------
namespace {
void put_error(char* err, uint64_t err_bytes, const std::string& text) {
  if (err == nullptr || err_bytes == 0) return;
  size_t n = std::min<size_t>(text.size(), size_t(err_bytes) - 1u);
  memcpy(err, text.data(), n);
  err[n] = 0;
}
}  // namespace

struct etxb_scene_file : etxb_scene_file_impl {};

extern "C" {

int etxb_scene_file_load(const char* file_name, const char* data_folder, etxb_scene_file** out, char* err, uint64_t err_bytes) {
  if (out == nullptr || file_name == nullptr) return ETXB_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  std::unique_ptr<etxb_scene_file> sf(new (std::nothrow) etxb_scene_file());
  if (!sf) return ETXB_ERR_OUT_OF_MEMORY;
  try {
    sf->tables = load_tables(data_folder);
    sf->data_folder = (data_folder && data_folder[0]) ? std::string(data_folder) : (module_directory() + "/data");
    sf->load(file_name);
  } catch (const LoadError& e) {
    put_error(err, err_bytes, e.text);
    return ETXB_ERR_UNSUPPORTED;
  } catch (const std::exception& e) {
    put_error(err, err_bytes, std::string(file_name) + ": " + e.what());
    return ETXB_ERR_INVALID_ARGUMENT;
  }
  *out = sf.release();
  return ETXB_OK;
}

const etxb_scene* etxb_scene_file_scene(const etxb_scene_file* sf) { return sf ? &sf->scene : nullptr; }
const etxb_camera* etxb_scene_file_camera(const etxb_scene_file* sf) { return sf ? &sf->camera : nullptr; }
uint32_t etxb_scene_file_warning_count(const etxb_scene_file* sf) { return sf ? uint32_t(sf->warnings.size()) : 0u; }
const char* etxb_scene_file_warning(const etxb_scene_file* sf, uint32_t index) { return (sf && index < sf->warnings.size()) ? sf->warnings[index].c_str() : nullptr; }
uint32_t etxb_scene_file_material_count(const etxb_scene_file* sf) { return sf ? uint32_t(sf->material_names.size()) : 0u; }
const char* etxb_scene_file_material_name(const etxb_scene_file* sf, uint32_t index) {
  return (sf && index < sf->material_names.size()) ? sf->material_names[index].c_str() : nullptr;
}
void etxb_scene_file_free(etxb_scene_file* sf) { delete sf; }
void etxb_scene_file_set_samples(etxb_scene_file* sf, uint32_t samples) {
  if (sf) sf->scene.samples = std::max(samples, 1u);
}

const void* etxb_scene_file_table(const etxb_scene_file* sf, const char* name, uint64_t* bytes) {
  if (bytes) *bytes = 0;
  if (sf == nullptr || name == nullptr || !sf->tables) return nullptr;
  const Tables& t = *sf->tables;
  if (auto i = t.f32.find(name); i != t.f32.end()) {
    if (bytes) *bytes = i->second.size() * 4u;
    return i->second.data();
  }
  if (auto i = t.u32.find(name); i != t.u32.end()) {
    if (bytes) *bytes = i->second.size() * 4u;
    return i->second.data();
  }
  if (auto i = t.u8.find(name); i != t.u8.end()) {
    if (bytes) *bytes = i->second.size();
    return i->second.data();
  }
  return nullptr;
}

// A string value of the application's options file (util/options.cxx: {"values": [{"class", "description", "id", "meta", "value"}, ...]}), e.g. the ids
// "integrator" and "scene" RTApplication::init reads at start-up (raytracer/app.cxx:88-105).  Returns the length, 0 when the id is absent, < 0 on error.
int etxb_options_file_string(const char* file_name, const char* id, char* out, uint64_t out_bytes) {
  if (file_name == nullptr || id == nullptr) return ETXB_ERR_INVALID_ARGUMENT;
  try {
    const std::string text = read_file(file_name);
    JsonParser parser{text};
    const Json root = parser.value();
    for (const auto& member : root.members) {
      if (member.first != "values" || member.second.kind != Json::Array) continue;
      for (const Json& entry : member.second.items) {
        const Json *entry_id = nullptr, *entry_value = nullptr;
        for (const auto& field : entry.members) {
          if (field.first == "id") entry_id = &field.second;
          if (field.first == "value") entry_value = &field.second;
        }
        if (entry_id == nullptr || entry_value == nullptr || entry_id->kind != Json::String || entry_id->text != id || entry_value->kind != Json::String) continue;
        put_error(out, out_bytes, entry_value->text);
        return int(std::min<size_t>(entry_value->text.size(), 0x7fffffffu));
      }
    }
  } catch (const LoadError&) {
    return ETXB_ERR_UNSUPPORTED;
  }
  return 0;
}

// The image readers on their own (PNG in every form, OpenEXR, Radiance HDR, PFM): rows in file order, RGBA8 (`eight_bit` = 1, 4 bytes per pixel, the file's
// own values: no sRGB step) or RGBA32F (16 bytes per pixel).  Call with pixels = NULL for the size, then with a buffer.
int etxb_image_file_read(const char* file_name, uint32_t* width, uint32_t* height, uint32_t* eight_bit, void* pixels, uint64_t capacity, char* err, uint64_t err_bytes) {
  if (file_name == nullptr || width == nullptr || height == nullptr || eight_bit == nullptr) return ETXB_ERR_INVALID_ARGUMENT;
  try {
    const Pixels px = read_image(file_name);
    *width = px.w, *height = px.h, *eight_bit = px.eight_bit ? 1u : 0u;
    if (pixels != nullptr) {
      const uint64_t bytes = uint64_t(px.w) * px.h * (px.eight_bit ? 4u : 16u);
      if (capacity < bytes) return ETXB_ERR_OVERFLOW;
      memcpy(pixels, px.eight_bit ? static_cast<const void*>(px.u8.data()) : static_cast<const void*>(px.f32.data()), size_t(bytes));
    }
  } catch (const LoadError& e) {
    put_error(err, err_bytes, e.text);
    return ETXB_ERR_UNSUPPORTED;
  } catch (const std::exception& e) {
    put_error(err, err_bytes, std::string(file_name) + ": " + e.what());
    return ETXB_ERR_UNSUPPORTED;
  }
  return ETXB_OK;
}

// The viewer's reference image as ImagePool::add_from_file(file, 0, {}, {1, 1}) leaves it (image_pool.cxx:51-67, 162-224, 271-385): float4 per
// pixel, rows in file order, 8-bit files read back as UNORM after the pool's sRGB -> linear and truncation.  A file that cannot be read is the
// 1 x 1 white placeholder, with the reason in `err`, and ETXB_OK, as the pool takes it.  Call with rgba = NULL for the size.
int etxb_reference_image_file_read(const char* file_name, uint32_t* width, uint32_t* height, float* rgba, uint64_t capacity, char* err, uint64_t err_bytes) {
  if (file_name == nullptr || width == nullptr || height == nullptr) return ETXB_ERR_INVALID_ARGUMENT;
  put_error(err, err_bytes, "");
  Pixels px;
  std::string problem;
  if (!pool_read(file_name, px, problem)) put_error(err, err_bytes, problem + "; using the 1x1 white placeholder");
  pool_convert(px, true, exr_file(file_name));
  *width = px.w, *height = px.h;
  if (rgba != nullptr) {
    const size_t n = size_t(px.w) * px.h;
    if (capacity < uint64_t(n) * 16u) return ETXB_ERR_OVERFLOW;
    if (px.eight_bit) {
      for (size_t i = 0; i < n * 4u; ++i) rgba[i] = px.u8[i] / 255.0f;
    } else {
      memcpy(rgba, px.f32.data(), n * 16u);
    }
  }
  return ETXB_OK;
}

// The tangent-space generator and the NanoVDB reader on their own, for a caller that assembles the scene itself (the Python twin)
int etxb_mesh_tangents(etxb_vertex* vertices, uint64_t vertex_count, const etxb_triangle* triangles, uint64_t triangle_count) {
  if ((vertices == nullptr && vertex_count != 0) || (triangles == nullptr && triangle_count != 0)) return ETXB_ERR_INVALID_ARGUMENT;
  for (uint64_t t = 0; t < triangle_count; ++t)
    for (int k = 0; k < 3; ++k)
      if (triangles[t].i[k] >= vertex_count) return ETXB_ERR_INVALID_ARGUMENT;
  std::vector<etxb_vertex> v(vertices, vertices + vertex_count);
  std::vector<etxb_triangle> tris(triangles, triangles + triangle_count);
  tangents::generate(v, tris);
  if (vertex_count) memcpy(vertices, v.data(), vertex_count * sizeof(etxb_vertex));
  return ETXB_OK;
}

int etxb_nvdb_density(const char* file_name, uint32_t dimensions[3], float* values, uint64_t value_capacity, char* err, uint64_t err_bytes) {
  if (file_name == nullptr || dimensions == nullptr) return ETXB_ERR_INVALID_ARGUMENT;
  try {
    std::vector<std::string> warnings;
    DensityGrid grid = read_nvdb_density(file_name, warnings);
    memcpy(dimensions, grid.dim, sizeof(grid.dim));
    if (values != nullptr) {
      if (value_capacity < grid.values.size()) return ETXB_ERR_OVERFLOW;
      if (!grid.values.empty()) memcpy(values, grid.values.data(), grid.values.size() * sizeof(float));
    }
  } catch (const LoadError& e) {
    put_error(err, err_bytes, e.text);
    return ETXB_ERR_UNSUPPORTED;
  } catch (const std::exception& e) {
    put_error(err, err_bytes, std::string(file_name) + ": " + e.what());
    return ETXB_ERR_UNSUPPORTED;
  }
  return ETXB_OK;
}

// The two images of an atmosphere block for a caller that assembles the emitters itself (etx_tracer_b200/loader.py, the Python twin of this file)
int etxb_atmosphere_images(const char* data_folder, const float direction[3], float angular_size, const float parameters[5], uint32_t sky_width, uint32_t sky_height,
                           float* sun_rgba_128x128, float* sky_rgba) {
  if (direction == nullptr || parameters == nullptr) return ETXB_ERR_INVALID_ARGUMENT;
  try {
    std::shared_ptr<Tables> tables = load_tables(data_folder);
    const std::string folder = (data_folder && data_folder[0]) ? std::string(data_folder) : (module_directory() + "/data");
    const atmosphere::Medium medium = {tables->get("spectra/atmosphere_rayleigh.power").data(), tables->get("spectra/atmosphere_mie.power").data(),
                                       tables->get("spectra/atmosphere_ozone.power").data()};
    AtmosphereParameters prm;
    prm.altitude = parameters[0], prm.anisotropy = parameters[1], prm.rayleigh_scale = parameters[2], prm.mie_scale = parameters[3], prm.ozone_scale = parameters[4];
    const F3 light = load3(direction);
    if (sun_rgba_128x128 != nullptr) atmosphere::sun_image(*tables, medium, prm, light, angular_size, 128, 128, sun_rgba_128x128);
    if (sky_rgba != nullptr && sky_width * sky_height != 0u) {
      auto table = atmosphere::optical_length_table(folder);
      atmosphere::sky_image(*tables, medium, *table, prm, light, sky_width, sky_height, sky_rgba);
    }
  } catch (const LoadError&) {
    return ETXB_ERR_UNSUPPORTED;
  }
  return ETXB_OK;
}

// Raytracing::link_scene / link_camera / commit_changes for a loaded file, with the two table uploads every context needs first: the colour tables and
// the blue-noise variant BNSampler would pick for scene.samples, next_power(min(samples, 256)) (thirdparty/bluenoise/bluenoise.cxx:73-95).
int etxb_scene_file_commit(etxb_ctx* ctx, const etxb_scene_file* sf) {
  if (ctx == nullptr || sf == nullptr || !sf->tables) return ETXB_ERR_INVALID_ARGUMENT;
  const Tables& t = *sf->tables;
  uint32_t spp = 1;
  while (spp < std::min(std::max(sf->scene.samples, 1u), 256u)) spp *= 2;
  auto xyz = t.f32.find("color_tables/xyz_441x3"), rgb = t.f32.find("color_tables/rgb_response_391x3");
  auto sobol = t.u8.find("bluenoise/sobol"), scr = t.u8.find("bluenoise/scrambling_" + std::to_string(spp)), rank = t.u8.find("bluenoise/ranking_" + std::to_string(spp));
  if (xyz == t.f32.end() || rgb == t.f32.end() || sobol == t.u8.end() || scr == t.u8.end() || rank == t.u8.end()) return ETXB_ERR_UNSUPPORTED;
  if (xyz->second.size() != 441u * 3u || rgb->second.size() != 391u * 3u || sobol->second.size() != 256u * 256u || scr->second.size() != 128u * 128u * 8u ||
      rank->second.size() != 128u * 128u * 8u)
    return ETXB_ERR_UNSUPPORTED;
  int rc = etxb_upload_color_tables(ctx, xyz->second.data(), rgb->second.data());
  if (rc == ETXB_OK) rc = etxb_upload_blue_noise(ctx, sobol->second.data(), scr->second.data(), rank->second.data());
  if (rc == ETXB_OK) rc = etxb_upload_scene(ctx, &sf->scene, sizeof(etxb_scene), &sf->camera, sizeof(etxb_camera));
  return rc;
}

}  // extern "C"
