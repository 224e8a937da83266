// dscene.cuh — the scene as it lives in HBM, and the geometry helpers of sources/etx/render/shared/scene.hxx.
//
// HBM layout (all arrays 16-byte aligned, read through the read-only path):
//   vertices   : DVertex[V]   64 B  = 4 x float4 {pos|u, nrm|v, tan, btn}      (reference Vertex is 56 B AoS)
//   triangles  : DTriangle[T] 32 B  = 2 x uint4  {i0,i1,i2,mat | geo_n,pad}    (same bytes as the reference)
//   tri_emitter: uint32[T]
//   materials  : etxb_material[M] 200 B (reference layout; a handful of records, L1/L2 resident)
//   spectra    : DSpectrum[S] = float power[441] on the fixed 390..830 nm grid + rgb  (reference: 3552 B with
//                a binary search; every SpectralDistribution the loader makes is resampled to this grid,
//                render/host/spectrum.cxx:11-95, so the search collapses to an index)
//   bvh_nodes  : BvhNode[...] 64 B, bvh_tris: float4[3*slots]
#pragma once
#include "../../include/etx_b200.h"
#include "bvh.h"
#include "dcore.cuh"
#include "dimage.cuh"

namespace etxb {

struct alignas(16) DVertex {
  float4 pos_u;  // pos.xyz, tex.x
  float4 nrm_v;  // nrm.xyz, tex.y
  float4 tan;
  float4 btn;
};
struct alignas(16) DTriangle {
  uint32_t i0, i1, i2, material_index;
  float gnx, gny, gnz, pad;
};
struct DSpectrum {
  float power[441];
  float rgb[3];
};

struct DeviceScene {
  const DVertex* vertices;
  const DTriangle* triangles;
  const uint32_t* tri_emitter;
  const etxb_material* materials;
  const etxb_emitter_profile* emitter_profiles;
  const etxb_emitter* emitters;
  const DSpectrum* spectra;
  const etxb_distribution_entry* emitter_dist;  // E + 1 entries
  const BvhNode* bvh_nodes;  // the first 512 nodes are the top levels, breadth-first (dtrav.cuh stages them in shared memory); below: depth-first
  const float4* bvh_tris;
  uint32_t bvh_node_count;
  const WideNode* wide_nodes;  // product build, scenes with stochastic BSDFs: the 4-wide quantised form of the same tree (dwide.cuh); else null
  uint32_t wide_node_count;
  const float* xyz_table;           // 441 x 3
  const float* rgb_response_table;  // 391 x 3
  const uint8_t* bn_sobol;          // 256 x 256
  const uint8_t* bn_scrambling;     // 128*128*8
  const uint8_t* bn_ranking;        // 128*128*8
  const DImage* images;
  uint32_t image_count;
  const struct DMedium* mediums;
  uint32_t medium_count;
  uint32_t spectrum_count;
  uint32_t deferred_shadow_rays;  // camera-vertex shadow rays may run in their own kernel (see k_shadow_trace)
  uint32_t has_subsurface;  // some material has subsurface scattering enabled
  uint32_t subsurface_exit_material;
  uint32_t has_boundaries;  // some material is of class Boundary (shadow rays may cross medium interfaces)
  uint32_t emitter_count;
  uint32_t triangle_count;
  float emitter_total_weight;
  float y_scale;  // 1 / kYIntegral
  uint32_t env_emitters[63];
  uint32_t env_emitter_count;
  V3 bounding_sphere_center;
  float bounding_sphere_radius;
  uint32_t min_path_length, max_path_length, samples, random_path_termination;
  uint32_t spectral;
  uint32_t has_blue_noise;
  uint32_t default_dielectric_eta, default_conductor_eta, default_conductor_k;
  etxb_camera camera;
};

// ---- loads ---------------------------------------------------------------------------------------------
DEV float4 ldg4(const float4* p) { return __ldg(p); }

struct VertexRec {
  V3 pos, nrm, tan, btn;
  V2 tex;
};
DEV VertexRec load_vertex(const DeviceScene& sc, uint32_t i) {
  const float4* p = reinterpret_cast<const float4*>(sc.vertices + i);
  float4 a = ldg4(p + 0), b = ldg4(p + 1), c = ldg4(p + 2), d = ldg4(p + 3);
  VertexRec v;
  v.pos = {a.x, a.y, a.z};
  v.nrm = {b.x, b.y, b.z};
  v.tan = {c.x, c.y, c.z};
  v.btn = {d.x, d.y, d.z};
  v.tex = {a.w, b.w};
  return v;
}
DEV V3 load_vertex_pos(const DeviceScene& sc, uint32_t i) {
  float4 a = ldg4(reinterpret_cast<const float4*>(sc.vertices + i));
  return {a.x, a.y, a.z};
}
DEV V3 load_vertex_nrm(const DeviceScene& sc, uint32_t i) {
  float4 a = ldg4(reinterpret_cast<const float4*>(sc.vertices + i) + 1);
  return {a.x, a.y, a.z};
}
struct TriRec {
  uint32_t i0, i1, i2, material_index;
  V3 geo_n;
};
DEV TriRec load_triangle(const DeviceScene& sc, uint32_t i) {
  const uint4* p = reinterpret_cast<const uint4*>(sc.triangles + i);
  uint4 a = __ldg(p);
  float4 b = ldg4(reinterpret_cast<const float4*>(p + 1));
  return {a.x, a.y, a.z, a.w, {b.x, b.y, b.z}};
}
DEV uint32_t load_triangle_material(const DeviceScene& sc, uint32_t i) { return __ldg(&sc.triangles[i].material_index); }

// ---- surface point (Intersection, math.hxx:672-689) -----------------------------------------------------
struct Isect {
  V3 pos, nrm, tan, btn;
  V2 tex;
  V3 barycentric;
  uint32_t triangle_index;
  V3 w_i;
  float t;
  uint32_t material_index;
  uint32_t emitter_index;
};

// scene.hxx:113-132 lerp_vertex
DEV void lerp_vertex(const DeviceScene& sc, const TriRec& tri, V3 bc, V3& pos, V3& nrm, V3& tan, V3& btn, V2& tex) {
  VertexRec v0 = load_vertex(sc, tri.i0), v1 = load_vertex(sc, tri.i1), v2 = load_vertex(sc, tri.i2);
  pos = v0.pos * bc.x + v1.pos * bc.y + v2.pos * bc.z;
  nrm = v0.nrm * bc.x + v1.nrm * bc.y + v2.nrm * bc.z;
  tan = v0.tan * bc.x + v1.tan * bc.y + v2.tan * bc.z;
  V3 b = v0.btn * bc.x + v1.btn * bc.y + v2.btn * bc.z;
  tex = {v0.tex.x * bc.x + v1.tex.x * bc.y + v2.tex.x * bc.z, v0.tex.y * bc.x + v1.tex.y * bc.y + v2.tex.y * bc.z};
  nrm = normalize(nrm);
  tan = normalize(tan - dot(tan, nrm) * nrm);
  V3 cb = cross(nrm, tan);
  btn = normalize(cb * (dot(cb, b) > 0.0f ? 1.0f : -1.0f));
}
DEV V3 lerp_pos(const DeviceScene& sc, const TriRec& tri, V3 bc) {
  return load_vertex_pos(sc, tri.i0) * bc.x + load_vertex_pos(sc, tri.i1) * bc.y + load_vertex_pos(sc, tri.i2) * bc.z;
}
DEV V3 lerp_normal(const DeviceScene& sc, const TriRec& tri, V3 bc) {
  return normalize(load_vertex_nrm(sc, tri.i0) * bc.x + load_vertex_nrm(sc, tri.i1) * bc.y + load_vertex_nrm(sc, tri.i2) * bc.z);
}
DEV V2 lerp_uv(const DeviceScene& sc, const TriRec& tri, V3 b) {
  float4 a0 = ldg4(reinterpret_cast<const float4*>(sc.vertices + tri.i0)), b0 = ldg4(reinterpret_cast<const float4*>(sc.vertices + tri.i0) + 1);
  float4 a1 = ldg4(reinterpret_cast<const float4*>(sc.vertices + tri.i1)), b1 = ldg4(reinterpret_cast<const float4*>(sc.vertices + tri.i1) + 1);
  float4 a2 = ldg4(reinterpret_cast<const float4*>(sc.vertices + tri.i2)), b2 = ldg4(reinterpret_cast<const float4*>(sc.vertices + tri.i2) + 1);
  return {a0.w * b.x + a1.w * b.y + a2.w * b.z, b0.w * b.x + b1.w * b.y + b2.w * b.z};
}

// scene.hxx:172-186 shading_pos
DEV V3 shading_pos_project(V3 position, V3 origin, V3 normal) { return position - dot(position - origin, normal) * normal; }
struct ShadingVerts {
  V3 p0, p1, p2, n0, n1, n2;
  V3 geo_pos, sh_normal;
};
DEV ShadingVerts load_shading_verts(const DeviceScene& sc, const TriRec& tri, V3 bc) {
  ShadingVerts v;
  v.p0 = load_vertex_pos(sc, tri.i0), v.p1 = load_vertex_pos(sc, tri.i1), v.p2 = load_vertex_pos(sc, tri.i2);
  v.n0 = load_vertex_nrm(sc, tri.i0), v.n1 = load_vertex_nrm(sc, tri.i1), v.n2 = load_vertex_nrm(sc, tri.i2);
  v.geo_pos = v.p0 * bc.x + v.p1 * bc.y + v.p2 * bc.z;
  v.sh_normal = normalize(v.n0 * bc.x + v.n1 * bc.y + v.n2 * bc.z);
  return v;
}
// the origin on one side of the surface: direction = +1 when w_o leaves on the side of the shading normal, -1 otherwise
DEV V3 shading_pos_side(const ShadingVerts& v, const TriRec& tri, V3 bc, float direction) {
  V3 p0 = shading_pos_project(v.geo_pos, v.p0, direction * v.n0);
  V3 p1 = shading_pos_project(v.geo_pos, v.p1, direction * v.n1);
  V3 p2 = shading_pos_project(v.geo_pos, v.p2, direction * v.n2);
  V3 sh_pos = p0 * bc.x + p1 * bc.y + p2 * bc.z;
  bool convex = dot(sh_pos - v.geo_pos, v.sh_normal) * direction > 0.0f;
  return offset_ray(convex ? sh_pos : v.geo_pos, tri.geo_n * direction);
}
DEV float shading_pos_direction(V3 sh_normal, V3 w_o) { return (dot(sh_normal, w_o) >= 0.0f) ? +1.0f : -1.0f; }
DEV V3 shading_pos(const DeviceScene& sc, const TriRec& tri, V3 bc, V3 w_o) {
  ShadingVerts v = load_shading_verts(sc, tri, bc);
  return shading_pos_side(v, tri, bc, shading_pos_direction(v.sh_normal, w_o));
}

// scene.hxx:202-226 make_intersection (incl. normal mapping)
DEV Isect make_intersection(const DeviceScene& sc, V3 w_i, uint32_t triangle_index, float u, float v, float t) {
  Isect r;
  V3 bc = barycentrics_uv(u, v);
  TriRec tri = load_triangle(sc, triangle_index);
  lerp_vertex(sc, tri, bc, r.pos, r.nrm, r.tan, r.btn, r.tex);
  r.barycentric = bc;
  r.triangle_index = triangle_index;
  r.w_i = w_i;
  r.t = t;
  r.material_index = tri.material_index;
  r.emitter_index = __ldg(&sc.tri_emitter[triangle_index]);
  const etxb_material& mat = sc.materials[r.material_index];
  if ((mat.normal_image_index != kInvalidIndex) && (mat.normal_scale > kEpsilon)) {
    // Image::evaluate_normal (image.hxx:109-116) + orient_normals_to_hemisphere (scene.hxx:188-200)
    F4v value = image_evaluate(sc.images[mat.normal_image_index], r.tex, nullptr);
    float scale = mat.normal_scale;
    V3 sn = {scale * (value.x * 2.0f - 1.0f), scale * (value.y * 2.0f - 1.0f), scale * (value.z * 2.0f - 1.0f) + (1.0f - scale)};
    V3 n_s = normalize(r.tan * sn.x + r.btn * sn.y + r.nrm * sn.z);
    const float i_dot_g = dot(w_i, tri.geo_n);
    float i_dot_s = dot(w_i, n_s);
    for (uint32_t k = 0; ((i_dot_s * i_dot_g) <= kEpsilon) && (k < 16u); ++k) {
      n_s = normalize(8.0f * n_s + tri.geo_n);
      i_dot_s = dot(w_i, n_s);
    }
    r.nrm = n_s;
    r.tan = normalize(r.tan - dot(r.tan, r.nrm) * r.nrm);
    r.btn = normalize(cross(r.nrm, r.tan));
  }
  return r;
}

// ---- spectra --------------------------------------------------------------------------------------------
// SpectralDistribution::query (spectrum.hxx:468-507) on the fixed integer grid
template <bool SP>
DEV Spec<SP> spectrum_query(const DeviceScene& sc, uint32_t index, float wavelength) {
  const DSpectrum& s = sc.spectra[index];
  if constexpr (!SP) {
    return Spec<false>{__ldg(&s.rgb[0]), __ldg(&s.rgb[1]), __ldg(&s.rgb[2])};
  } else {
    if (wavelength < 390.0f) return {0.0f};
    float fl = floorf(wavelength);
    uint32_t i = static_cast<uint32_t>(fl) - 390u;
    if (i > 440u) i = 440u;
    float wi = static_cast<float>(390u + i);
    if ((i == 440u) && (wavelength > wi)) return {0.0f};
    uint32_t j = umin(i + 1u, 440u);
    float tt = (i == j) ? 0.0f : (wavelength - wi) / (static_cast<float>(390u + j) - wi);
    float p = lerpf(__ldg(&s.power[i]), __ldg(&s.power[j]), tt);
    return {p};
  }
}

// SpectralResponse::to_rgb (spectrum.hxx:271-293)
template <bool SP>
DEV V3 spec_to_rgb(const DeviceScene& sc, Spec<SP> s, float wavelength) {
  if constexpr (!SP) {
    return {s.x, s.y, s.z};
  } else {
    if ((s.v == 0.0f) || (wavelength < 390.0f) || (wavelength > 830.0f)) return xyz_to_rgb({0.0f, 0.0f, 0.0f});
    float w = floorf(wavelength);
    float dw = wavelength - w;
    uint32_t i = static_cast<uint32_t>(w - 390.0f);
    uint32_t j = umin(i + 1u, 440u);
    V3 xyz0 = {__ldg(&sc.xyz_table[i * 3 + 0]), __ldg(&sc.xyz_table[i * 3 + 1]), __ldg(&sc.xyz_table[i * 3 + 2])};
    V3 xyz1 = {__ldg(&sc.xyz_table[j * 3 + 0]), __ldg(&sc.xyz_table[j * 3 + 1]), __ldg(&sc.xyz_table[j * 3 + 2])};
    V3 xyz = (xyz0 * (1.0f - dw) + xyz1 * dw) * (s.v * sc.y_scale);
    return xyz_to_rgb(xyz);
  }
}

// rgb_response (render/host/spectrum.cxx:399-): RGB -> reflectance at one wavelength through the 391-entry response table
DEV float rgb_response(const DeviceScene& sc, float wavelength, V3 rgb) {
  if (luminance(rgb) == 0.0f) return 0.0f;
  if ((wavelength < 390.0f) || (wavelength > 780.0f)) return 0.0f;
  uint32_t wi = uint32_t(wavelength - 390.0f);
  uint32_t wj = umin(wi + 1u, 390u);
  float dw = wavelength - floorf(wavelength);
  const float* t = sc.rgb_response_table;
  V3 w = lerp3({__ldg(&t[wi * 3 + 0]), __ldg(&t[wi * 3 + 1]), __ldg(&t[wi * 3 + 2])}, {__ldg(&t[wj * 3 + 0]), __ldg(&t[wj * 3 + 1]), __ldg(&t[wj * 3 + 2])}, dw);
  return rgb.x * w.x + rgb.y * w.y + rgb.z * w.z;
}
// apply_rgb (scene.hxx:251-263)
template <bool SP>
DEV Spec<SP> apply_rgb(const DeviceScene& sc, float wavelength, Spec<SP> response, F4v value) {
  if constexpr (SP) {
    float scale = rgb_response(sc, wavelength, {value.x, value.y, value.z});
    response *= scale;
    return response;
  } else {
    return {response.x * value.x, response.y * value.y, response.z * value.z};
  }
}
// apply_image (scene.hxx:291-305)
template <bool SP>
DEV Spec<SP> apply_image(const DeviceScene& sc, const etxb_spectral_image& img, V2 uv, float wavelength, float* image_pdf = nullptr) {
  if (image_pdf) *image_pdf = 0.0f;
  Spec<SP> result = spectrum_query<SP>(sc, img.spectrum_index, wavelength);
  if (img.image_index == kInvalidIndex) return result;
  F4v eval = image_evaluate(sc.images[img.image_index], uv, image_pdf);
  return apply_rgb<SP>(sc, wavelength, result, eval);
}

// RefractiveIndex::Sample (spectrum.hxx:557-586) via evaluate_refractive_index (scene.hxx:307-313)
template <bool SP>
struct IorSample {
  uint32_t cls;
  Spec<SP> eta, k;
};
template <bool SP>
DEV IorSample<SP> evaluate_ior(const DeviceScene& sc, const etxb_refractive_index& ri, float wavelength) {
  IorSample<SP> r;
  r.cls = ri.cls;
  r.eta = (ri.eta_index == kInvalidIndex) ? Spec<SP>::make(1.0f) : spectrum_query<SP>(sc, ri.eta_index, wavelength);
  r.k = (ri.k_index == kInvalidIndex) ? Spec<SP>::make(0.0f) : spectrum_query<SP>(sc, ri.k_index, wavelength);
  return r;
}

// evaluate_image / evaluate_roughness / evaluate_metalness (scene.hxx:265-289)
DEV float evaluate_image_channel(const DeviceScene& sc, const etxb_sampled_image& img, V2 uv, float default_value) {
  if ((img.image_index == kInvalidIndex) || (img.channel >= 4u)) return default_value;
  F4v e = image_evaluate(sc.images[img.image_index], uv, nullptr);
  return img.channel == 0u ? e.x : (img.channel == 1u ? e.y : (img.channel == 2u ? e.z : e.w));
}
DEV V2 evaluate_roughness(const DeviceScene& sc, const etxb_material& m, V2 uv) {
  float s = evaluate_image_channel(sc, m.roughness, uv, 1.0f);
  return {m.roughness.value[0] * s, m.roughness.value[1] * s};
}
DEV float evaluate_metalness(const DeviceScene& sc, const etxb_material& m, V2 uv) { return m.metalness.value[0] * evaluate_image_channel(sc, m.metalness, uv, 1.0f); }

// scene.hxx:228-249 random_continue
template <bool SP>
DEV bool random_continue(uint32_t path_length, uint32_t start_path_length, float eta_scale, Smp& smp, Spec<SP>& throughput) {
  float max_t = throughput.maximum();
  if (max_t == 0.0f) return false;
  if (path_length < start_path_length) return true;
  max_t *= sqr(eta_scale);
  if (valid_value(max_t) == false) return false;
  float q = tmin(0.95f, max_t);
  if ((q > 0.0f) && (smp.next() < q)) {
    throughput *= (1.0f / q);
    return true;
  }
  return false;
}

// thirdparty/bluenoise sampler*_spp.hpp (integer table lookups) + rt/integrators/path_tracing.cxx:173-178
DEV V2 sample_blue_noise(const DeviceScene& sc, uint32_t px, uint32_t py, uint32_t current_sample, uint32_t dimension) {
  float out[2];
#pragma unroll
  for (uint32_t k = 0; k < 2; ++k) {
    uint32_t dim = (dimension + k) & 7u;
    uint32_t pi = px & 127u, pj = py & 127u;
    uint32_t si = current_sample & 255u;
    uint32_t tile = dim + (pi + pj * 128u) * 8u;
    uint32_t ranked = si ^ uint32_t(__ldg(&sc.bn_ranking[tile]));
    uint32_t value = uint32_t(__ldg(&sc.bn_sobol[dim + ranked * 256u]));
    value = value ^ uint32_t(__ldg(&sc.bn_scrambling[tile]));
    out[k] = (0.5f + float(int(value))) / 256.0f;
  }
  return {out[0], out[1]};
}

}  // namespace etxb
