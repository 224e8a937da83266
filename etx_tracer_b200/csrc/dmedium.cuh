// dmedium.cuh — participating media: homogeneous (closed-form free flight with spectral-channel MIS) and heterogeneous (dense
// float grid, trilinear taps, delta tracking / ratio tracking), Henyey-Greenstein phase function.
// Restates sources/etx/render/shared/scene_medium.hxx (line refs inline) and medium.hxx:8-47.
#pragma once
#include "dscene.cuh"

namespace etxb {

struct DMedium {
  const float* density;  // dx*dy*dz floats, normalised to max 1 (host prep: medium_pool.cxx:44-55)
  V3 bounds_min, bounds_max;
  uint32_t cls;  // 0 homogeneous, 1 heterogeneous
  uint32_t enable_explicit_connections;
  uint32_t absorption_index, scattering_index;
  float phase_function_g, max_sigma;
  uint32_t dim_x, dim_y, dim_z;
};

template <bool SP>
struct MediumSample {  // Medium::Sample (medium.hxx:27-40)
  Spec<SP> weight;
  V3 pos;
  float sampled_medium_t;
  DEV bool sampled_medium() const { return sampled_medium_t > 0.0f; }
};

// scene_medium.hxx:7-55
DEV bool medium_bounds(V3 in_pos, V3 in_dir, float max_t, float& t_min, float& t_max) {
  constexpr float e = kEpsilon * 0.5f;
  constexpr float gamma3 = (3 * e) / (1.0f - 3 * e);
  constexpr float g3 = 1.0f + 2.0f * gamma3;
  float pos[3] = {in_pos.x, in_pos.y, in_pos.z};
  float dir[3] = {in_dir.x, in_dir.y, in_dir.z};
  t_min = 0.0f;
  t_max = max_t;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    float t_near = (0.0f - pos[i]) / dir[i];
    float t_far = (1.0f - pos[i]) / dir[i];
    if (t_near > t_far) {
      float t = t_far;
      t_far = t_near;
      t_near = t;
    }
    t_far *= g3;
    t_min = t_near > t_min ? t_near : t_min;
    t_max = t_far < t_max ? t_far : t_max;
    if (t_min > t_max) return false;
  }
  return true;
}
DEV V3 bounds_to_local(const DMedium& m, V3 p) { return (p - m.bounds_min) / (m.bounds_max - m.bounds_min); }
DEV bool medium_intersects_bounds(const DMedium& medium, V3 in_pos, V3 in_direction, float in_max_t, V3& medium_pos, V3& medium_dir, float& t_min, float& t_max) {
  if (in_max_t >= kMaxFloat) return false;
  V3 end_pos = in_pos + in_direction * in_max_t;
  V3 medium_end_pos = bounds_to_local(medium, end_pos);
  medium_pos = bounds_to_local(medium, in_pos);
  // __fsub_rn: the product build would otherwise contract the difference of the two local points with one of their products into an FMA,
  // and a component along which the ray does not move would keep that product's rounding error (~1e-8) instead of being exactly 0 --
  // the slab of a ray parallel to a face then ends at t = 0 instead of being skipped as 0 / 0.  Without -fmad this is the plain difference.
  const V3 delta = {__fsub_rn(medium_end_pos.x, medium_pos.x), __fsub_rn(medium_end_pos.y, medium_pos.y), __fsub_rn(medium_end_pos.z, medium_pos.z)};
  medium_dir = normalize(delta);
  float segment = length(delta);
  return medium_bounds(medium_pos, medium_dir, segment, t_min, t_max);
}

// scene_medium.hxx:58-95 — 8 trilinear taps
DEV float medium_sample_density(const DMedium& m, V3 coord) {
  if ((coord.x < 0.0f) || (coord.y < 0.0f) || (coord.z < 0.0f) || (coord.x >= 1.0f) || (coord.y >= 1.0f) || (coord.z >= 1.0f)) return 0.0f;
  float px = clampf(coord.x * float(m.dim_x) - 0.5f, 0.0f, float(m.dim_x) - 1.0f);
  float py = clampf(coord.y * float(m.dim_y) - 0.5f, 0.0f, float(m.dim_y) - 1.0f);
  float pz = clampf(coord.z * float(m.dim_z) - 0.5f, 0.0f, float(m.dim_z) - 1.0f);
  uint32_t ix = umin(m.dim_x - 1u, static_cast<uint32_t>(px)), nx = umin(m.dim_x - 1u, ix + 1u);
  uint32_t iy = umin(m.dim_y - 1u, static_cast<uint32_t>(py)), ny = umin(m.dim_y - 1u, iy + 1u);
  uint32_t iz = umin(m.dim_z - 1u, static_cast<uint32_t>(pz)), nz = umin(m.dim_z - 1u, iz + 1u);
  const float* d = m.density;
  uint32_t sx = m.dim_x, sxy = m.dim_x * m.dim_y;
  float d000 = __ldg(&d[ix + iy * sx + iz * sxy]);
  float d001 = __ldg(&d[nx + iy * sx + iz * sxy]);
  float d010 = __ldg(&d[ix + ny * sx + iz * sxy]);
  float d011 = __ldg(&d[nx + ny * sx + iz * sxy]);
  float d100 = __ldg(&d[ix + iy * sx + nz * sxy]);
  float d101 = __ldg(&d[nx + iy * sx + nz * sxy]);
  float d110 = __ldg(&d[ix + ny * sx + nz * sxy]);
  float d111 = __ldg(&d[nx + ny * sx + nz * sxy]);
  float dx = px - floorf(px), dy = py - floorf(py), dz = pz - floorf(pz);
  float d_bottom = lerpf(lerpf(d000, d001, dx), lerpf(d010, d011, dx), dy);
  float d_top = lerpf(lerpf(d100, d101, dx), lerpf(d110, d111, dx), dy);
  return lerpf(d_bottom, d_top, dz);
}

// scene_medium.hxx:99-123
template <bool SP>
DEV uint32_t sample_spectrum_component(Spec<SP> albedo, Spec<SP> throughput, float rnd, Spec<SP>& pdf) {
  if constexpr (SP) {
    pdf = {1.0f};
    return 0;
  } else {
    Spec<false> at = albedo * throughput;
    if (at.is_zero()) {
      pdf = Spec<false>::make(1.0f / 3.0f);
      return uint32_t(3.0f * rnd);
    }
    pdf = at / at.sum();
    return 2u - uint32_t(rnd < pdf.x + pdf.y) - uint32_t(rnd < pdf.x);
  }
}
template <bool SP>
DEV Spec<SP> calculate_albedo(Spec<SP> scattering, Spec<SP> extinction) {
  if constexpr (SP) {
    return {extinction.v > 0.0f ? (scattering.v / extinction.v) : 0.0f};
  } else {
    return {extinction.x > 0.0f ? (scattering.x / extinction.x) : 0.0f, extinction.y > 0.0f ? (scattering.y / extinction.y) : 0.0f,
      extinction.z > 0.0f ? (scattering.z / extinction.z) : 0.0f};
  }
}

// scene_medium.hxx:125-145 — Henyey-Greenstein
DEV float phase_function(V3 w_i, V3 w_o, float g) {
  float cos_t = dot(w_i, w_o);
  float d = 1.0f + g * g - 2.0f * g * cos_t;
  return (1.0f / (4.0f * kPi)) * (1.0f - g * g) / (d * sqrtf(d));
}
DEV V3 sample_phase_function(V3 w_i, float g, V2 smp_rnd) {
  float cos_theta;
  if (fabsf(g) < 1e-3f) {
    cos_theta = 1.0f - 2.0f * smp_rnd.x;
  } else {
    float sqr_term = (1.0f - g * g) / (1.0f + g * (2.0f * smp_rnd.x - 1.0f));
    cos_theta = (1.0f + g * g - sqr_term * sqr_term) / (2.0f * g);
  }
  float sin_theta = sqrtf(tmax(0.0f, 1.0f - cos_theta * cos_theta));
  float phi = kDoublePi * smp_rnd.y;
  Basis basis = orthonormal_basis(w_i);
  return (basis.u * m_cos(phi) + basis.v * m_sin(phi)) * sin_theta - w_i * cos_theta;
}

template <bool SP>
DEV Spec<SP> medium_absorption(const DeviceScene& sc, const DMedium& m, float wavelength) {
  if ((m.absorption_index == kInvalidIndex) || (m.absorption_index >= sc.spectrum_count)) return Spec<SP>::make(0.0f);
  return spectrum_query<SP>(sc, m.absorption_index, wavelength);
}
template <bool SP>
DEV Spec<SP> medium_scattering(const DeviceScene& sc, const DMedium& m, float wavelength) {
  if ((m.scattering_index == kInvalidIndex) || (m.scattering_index >= sc.spectrum_count)) return Spec<SP>::make(0.0f);
  return spectrum_query<SP>(sc, m.scattering_index, wavelength);
}
template <bool SP>
DEV Spec<SP> medium_extinction(const DeviceScene& sc, const DMedium& m, float wavelength) {
  return medium_absorption<SP>(sc, m, wavelength) + medium_scattering<SP>(sc, m, wavelength);
}

// scene_medium.hxx:191-239 — transmittance along a segment (heterogeneous: ratio tracking with Russian roulette)
template <bool SP>
DEV Spec<SP> medium_transmittance(const DeviceScene& sc, const DMedium& medium, float wavelength, Smp& smp, V3 pos, V3 direction, float distance) {
  if (medium.cls == 0u) {
    return spec_exp(medium_extinction<SP>(sc, medium, wavelength) * (-distance));
  }
  if (medium.max_sigma <= 0.0f) return Spec<SP>::make(1.0f);
  V3 medium_pos = pos, medium_dir = direction;
  float t_min = 0.0f, t_max = 0.0f;
  if (medium_intersects_bounds(medium, pos, direction, distance, medium_pos, medium_dir, t_min, t_max) == false) return Spec<SP>::make(1.0f);
  const float rr_threshold = 0.1f;
  float transmittance = 1.0f;
  float t = t_min;
  while (true) {
    t -= m_log(1.0f - smp.next()) / medium.max_sigma;
    if (t >= t_max) break;
    float density_value = medium_sample_density(medium, medium_pos + medium_dir * t);
    transmittance *= tmax(0.0f, 1.0f - density_value);
    if (transmittance < rr_threshold) {
      float q = tmax(0.05f, 1.0f - transmittance);
      if (smp.next() < q) return Spec<SP>::make(0.0f);
      transmittance /= (1.0f - q);
    }
  }
  return Spec<SP>::make(transmittance);
}

// scene_medium.hxx:241-351 — free-flight sampling
template <bool SP>
DEV MediumSample<SP> sample_medium(const DeviceScene& sc, const DMedium& medium, float wavelength, Spec<SP> throughput, Smp& smp, V3 pos, V3 w_i, float max_t) {
  MediumSample<SP> result;
  result.weight = Spec<SP>::make(0.0f);
  result.pos = {0.0f, 0.0f, 0.0f};
  result.sampled_medium_t = 0.0f;
  if (medium.cls == 0u) {
    Spec<SP> scattering_value = medium_scattering<SP>(sc, medium, wavelength);
    Spec<SP> absorption_value = medium_absorption<SP>(sc, medium, wavelength);
    Spec<SP> extinction_value = scattering_value + absorption_value;
    Spec<SP> albedo = calculate_albedo<SP>(scattering_value, extinction_value);
    float t = 0.0f;
    Spec<SP> pdf = Spec<SP>::make(0.0f);
    while (t < kRayEpsilon) {
      uint32_t channel = sample_spectrum_component<SP>(albedo, throughput, smp.next(), pdf);
      float sample_t = extinction_value.component(channel);
      t = (sample_t > 0.0f) ? -m_log(1.0f - smp.next()) / sample_t : max_t;
    }
    t = tmin(t, max_t);
    bool sampled_medium = t < max_t;
    Spec<SP> tr = spec_exp(-t * extinction_value);
    pdf *= sampled_medium ? tr * extinction_value : tr;
    if (pdf.is_zero()) return result;
    result.pos = pos + w_i * t;
    result.sampled_medium_t = sampled_medium ? t : 0.0f;
    result.weight = (sampled_medium ? tr * scattering_value : tr) / pdf.sum();
    return result;
  }
  if (medium.max_sigma <= 0.0f) return result;
  V3 medium_pos = pos, medium_dir = w_i;
  float t_min = 0.0f, t_max = 0.0f;
  if (medium_intersects_bounds(medium, pos, w_i, max_t, medium_pos, medium_dir, t_min, t_max) == false) return result;
  Spec<SP> scattering_value = medium_scattering<SP>(sc, medium, wavelength);
  Spec<SP> extinction_value = medium_extinction<SP>(sc, medium, wavelength);
  Spec<SP> albedo = calculate_albedo<SP>(scattering_value, extinction_value);
  float t = t_min;
  float previous_t = t_min;
  Spec<SP> accumulated_transmittance = Spec<SP>::make(1.0f);
  while (true) {
    t -= m_log(1.0f - smp.next()) / medium.max_sigma;
    if (t >= t_max) break;
    float distance = tmax(0.0f, t - previous_t);
    accumulated_transmittance *= spec_exp(-extinction_value * distance);
    previous_t = t;
    float density_value = medium_sample_density(medium, medium_pos + medium_dir * t);
    if (density_value * medium.max_sigma == 0.0f) continue;
    Spec<SP> pdf = Spec<SP>::make(0.0f);
    uint32_t channel = sample_spectrum_component<SP>(albedo, scattering_value, smp.next(), pdf);
    float sigma_t = extinction_value.component(channel);
    float random = smp.next();
    if ((sigma_t > 0.0f) && (random < density_value)) {
      float pdf_sum = pdf.sum();
      if (pdf_sum > 0.0f) {
        result.weight = (scattering_value * accumulated_transmittance) / pdf_sum;
      } else {
        result.weight = scattering_value * accumulated_transmittance;
      }
      result.pos = medium_pos + medium_dir * t;  // (sic) the reference reports the position in the medium's local frame
      result.sampled_medium_t = t - t_min;
      return result;
    }
  }
  float remaining_distance = tmax(0.0f, t_max - previous_t);
  accumulated_transmittance *= spec_exp(-extinction_value * remaining_distance);
  result.weight = accumulated_transmittance;
  return result;
}

}  // namespace etxb
