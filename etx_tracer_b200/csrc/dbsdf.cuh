// dbsdf.cuh — BSDF sample / evaluate / pdf for the material classes on the hot path.
//
// Follows sources/etx/render/shared/{bsdf.hxx, scene_bsdf.hxx, bsdf_various.hxx, bsdf_dielectric.hxx,
// bsdf_conductor.hxx, bsdf_external.hxx}.  The microfacet classes use the Heitz et al. multiple-scattering
// random walk on the microsurface; its evaluate() is stochastic and consumes the path's sampler, so the order
// of sampler draws below is part of the contract (SURVEY.md Appendix C).
#pragma once
#include "dscene.cuh"

namespace etxb {

enum : uint32_t { kPathCamera = 1u, kPathLight = 2u };  // PathSource (bsdf.hxx:14-18)

enum : uint32_t {  // BSDFSample::Properties (bsdf.hxx:63-69)
  kBsdfDiffuse = 1u << 0u,
  kBsdfReflection = 1u << 1u,
  kBsdfTransmission = 1u << 2u,
  kBsdfMediumChanged = 1u << 3u,
  kBsdfDelta = 1u << 4u,
};

// BSDFData (bsdf.hxx:20-45): the surface point + incoming direction + query
struct BData {
  V3 pos, nrm, tan, btn;
  V2 tex;
  V3 w_i;
  float wavelength;
  uint32_t path_source;
  uint32_t current_medium;
};
DEV BData make_bdata(const Isect& i, V3 w_i, float wavelength, uint32_t medium, uint32_t source) {
  return {i.pos, i.nrm, i.tan, i.btn, i.tex, w_i, wavelength, source, medium};
}

template <bool SP>
struct BEval {
  Spec<SP> func, bsdf;
  float pdf;
  float eta;
  DEV bool valid() const { return pdf > 0.0f; }
};
template <bool SP>
DEV BEval<SP> beval_zero() {
  return {Spec<SP>::make(0.0f), Spec<SP>::make(0.0f), 0.0f, 1.0f};
}

template <bool SP>
struct BSample {
  Spec<SP> weight;
  V3 w_o;
  float pdf;
  float eta;
  uint32_t properties;
  uint32_t medium_index;
  DEV bool valid() const { return pdf > 0.0f; }
  DEV bool is_delta() const { return (properties & kBsdfDelta) == kBsdfDelta; }
};
template <bool SP>
DEV BSample<SP> bsample_zero() {
  return {Spec<SP>::make(0.0f), {0.0f, 0.0f, 0.0f}, 0.0f, 1.0f, 0u, kInvalidIndex};
}

// LocalFrame (math.hxx:614-643)
struct Frame {
  V3 tan, btn, nrm;
  bool entering;
  DEV V3 to_local(V3 v) const {
    return {tan.x * v.x + tan.y * v.y + tan.z * v.z, btn.x * v.x + btn.y * v.y + btn.z * v.z, nrm.x * v.x + nrm.y * v.y + nrm.z * v.z};
  }
  DEV V3 from_local(V3 v) const {
    return {tan.x * v.x + btn.x * v.y + nrm.x * v.z, tan.y * v.x + btn.y * v.y + nrm.y * v.z, tan.z * v.x + btn.z * v.y + nrm.z * v.z};
  }
};
// BSDFData::get_normal_frame (bsdf.hxx:34-37)
DEV Frame normal_frame(const BData& d) {
  bool entering = dot(d.nrm, d.w_i) < 0.0f;
  return entering ? Frame{d.tan, d.btn, d.nrm, true} : Frame{-d.tan, -d.btn, -d.nrm, false};
}
DEV V3 front_facing_normal(const BData& d) { return dot(d.nrm, d.w_i) < 0.0f ? d.nrm : -d.nrm; }

// bsdf.hxx:232-239
DEV float fix_shading_normal(V3 n_g, V3 n_s, V3 w_i, V3 w_o) {
  float w_i_g = dot(w_i, n_g);
  float w_i_s = dot(w_i, n_s);
  float w_o_g = dot(w_o, n_g);
  float w_o_s = dot(w_o, n_s);
  float den = fmaxf(kInvMaxHalf, fabsf(w_o_s * w_i_g));
  return fabsf(w_o_g * w_i_s) / den;
}

// ---- Fresnel (bsdf.hxx:241-377) ---------------------------------------------------------------------------
template <bool SP>
struct ThinfilmEval {
  IorSample<SP> ior;
  V3 rgb_wavelengths;
  float thickness;
};

struct RsRp {
  Cx a, b;
};
DEV Cx cx_div_conj(Cx a, Cx b) {
  Cx num = a * cx_conj(b);
  float denom = cx_norm(b);
  return {num.re / denom, num.im / denom};
}
DEV RsRp fresnel_reflectance(Cx ni, Cx ci, Cx nj, Cx cj) {
  if ((ci.re == 0.0f) && (cj.re == 0.0f) && (ci.im == 0.0f) && (cj.im == 0.0f)) return {cx(1.0f), cx(1.0f)};
  if (ni == nj) return {cx(0.0f), cx(0.0f)};
  Cx rs = cx_div_conj(ni * ci - nj * cj, ni * ci + nj * cj);
  Cx rp = cx_div_conj(nj * ci - ni * cj, nj * ci + ni * cj);
  return {rs, rp};
}
DEV RsRp fresnel_transmittance(Cx ni, Cx ci, Cx nj, Cx cj) {
  if ((ci.re == 0.0f) && (cj.re == 0.0f) && (ci.im == 0.0f) && (cj.im == 0.0f)) return {cx(0.0f), cx(0.0f)};
  if (ni == nj) return {cx(1.0f), cx(1.0f)};
  Cx ts = cx_div_conj((2.0f * ni) * ci, ni * ci + nj * cj);
  Cx tp = cx_div_conj((2.0f * ni) * ci, ni * cj + nj * ci);
  return {ts, tp};
}
DEVN float fresnel_generic(float cos_theta_i, Cx ext_ior, Cx int_ior) {
#if !(defined(ETXB_PARITY) && ETXB_PARITY)
  if ((ext_ior.im == 0.0f) && (int_ior.im == 0.0f)) {
    // two dielectrics: the same Fresnel equations in real arithmetic (total internal reflection = the complex cosine turning imaginary)
    const float q = __fdividef(ext_ior.re, int_ior.re);
    const float sin2_o = q * q * (1.0f - cos_theta_i * cos_theta_i);
    if (sin2_o >= 1.0f) return 1.0f;
    const float cos_o = sqrtf(1.0f - sin2_o);
    const float a = ext_ior.re * cos_theta_i, b = int_ior.re * cos_o, c = int_ior.re * cos_theta_i, d = ext_ior.re * cos_o;
    if ((a + b == 0.0f) || (c + d == 0.0f)) return 1.0f;
    const float rs = __fdividef(a - b, a + b), rp = __fdividef(c - d, c + d);
    return 0.5f * (rs * rs + rp * rp);
  }
#endif
  Cx q = ext_ior / int_ior;
  Cx sin_theta_o_squared = (q * q) * (1.0f - cos_theta_i * cos_theta_i);
  Cx cos_theta_o = cx_sqrt(1.0f - sin_theta_o_squared);
  RsRp r = fresnel_reflectance(ext_ior, cx(cos_theta_i), int_ior, cos_theta_o);
  return 0.5f * (cx_norm(r.a) + cx_norm(r.b));
}
DEVN float fresnel_thinfilm(float wavelength, float cos_theta_0, Cx ext_ior, Cx film_ior, Cx int_ior, float thickness) {
  const Cx i = {0.0f, 1.0f};
  if (cos_theta_0 == 0.0f) return 0.0f;
  Cx q1 = ext_ior / film_ior;
  Cx sin_theta_1_squared = (q1 * q1) * (1.0f - cos_theta_0 * cos_theta_0);
  if (sin_theta_1_squared.re >= 1.0f) return 1.0f;
  Cx cos_theta_1 = cx_sqrt(1.0f - sin_theta_1_squared);
  Cx q2 = film_ior / int_ior;
  Cx sin_theta_2_squared = (q2 * q2) * (1.0f - cos_theta_1 * cos_theta_1);
  if (sin_theta_2_squared.re >= 1.0f) return 1.0f;
  Cx cos_theta_2 = cx_sqrt(1.0f - sin_theta_2_squared);
  Cx ratio = (int_ior * cos_theta_2) / (ext_ior * cos_theta_0);
  float delta_10 = ext_ior.re < film_ior.re ? kPi : 0.0f;
  float delta_21 = film_ior.re < int_ior.re ? kPi : 0.0f;
  float phase_shift = delta_10 + delta_21;
  RsRp r01 = fresnel_reflectance(ext_ior, cx(cos_theta_0), film_ior, cos_theta_1);
  RsRp t01 = fresnel_transmittance(ext_ior, cx(cos_theta_0), film_ior, cos_theta_1);
  RsRp r12 = fresnel_reflectance(film_ior, cos_theta_1, int_ior, cos_theta_2);
  RsRp t12 = fresnel_transmittance(film_ior, cos_theta_1, int_ior, cos_theta_2);
  Cx phi = ((kDoublePi * 2.0f * thickness) * cos_theta_1 + phase_shift * film_ior) / wavelength;
  Cx exp_i_phi = cx_exp(i * phi);
  Cx tpq = t01.b * t12.b / (1.0f - r01.b * r12.b * exp_i_phi);
  Cx tp = tpq * tpq;
  Cx tsq = t01.a * t12.a / (1.0f - r01.a * r12.a * exp_i_phi);
  Cx ts = tsq * tsq;
  return cx_abs(1.0f - ratio * 0.5f * (tp + ts));
}

constexpr uint32_t kSpdClassConductor = 2u;  // SpectralDistribution::Class::Conductor (spectrum.hxx:455)

template <bool SP>
DEV Spec<SP> fresnel_calculate(float wavelength, float cos_theta, const IorSample<SP>& ext_ior, const IorSample<SP>& int_ior, const ThinfilmEval<SP>& thinfilm) {
  cos_theta = fabsf(cos_theta);
  bool plain = (thinfilm.thickness == 0.0f) || thinfilm.ior.eta.is_zero();
  if constexpr (SP) {
    float value;
    if (plain) {
      value = fresnel_generic(cos_theta, cx(ext_ior.eta.v, ext_ior.k.v), cx(int_ior.eta.v, int_ior.k.v));
    } else {
      value = fresnel_thinfilm(wavelength, cos_theta, cx(ext_ior.eta.v, ext_ior.k.v), cx(thinfilm.ior.eta.v, thinfilm.ior.k.v), cx(int_ior.eta.v, int_ior.k.v),
        thinfilm.thickness);
    }
    return {saturatef(value)};
  } else {
    V3 values;
    if (plain) {
      values.x = fresnel_generic(cos_theta, cx(ext_ior.eta.x, ext_ior.k.x), cx(int_ior.eta.x, int_ior.k.x));
      values.y = fresnel_generic(cos_theta, cx(ext_ior.eta.y, ext_ior.k.y), cx(int_ior.eta.y, int_ior.k.y));
      values.z = fresnel_generic(cos_theta, cx(ext_ior.eta.z, ext_ior.k.z), cx(int_ior.eta.z, int_ior.k.z));
      if (int_ior.cls == kSpdClassConductor) {
        values = xyz_to_rgb(values) * V3{0.817660332f, 1.05418909f, 1.09945524f};
      }
    } else {
      values.x = fresnel_thinfilm(thinfilm.rgb_wavelengths.x, cos_theta, cx(ext_ior.eta.x, ext_ior.k.x), cx(thinfilm.ior.eta.x, thinfilm.ior.k.x),
        cx(int_ior.eta.x, int_ior.k.x), thinfilm.thickness);
      values.y = fresnel_thinfilm(thinfilm.rgb_wavelengths.y, cos_theta, cx(ext_ior.eta.y, ext_ior.k.y), cx(thinfilm.ior.eta.y, thinfilm.ior.k.y),
        cx(int_ior.eta.y, int_ior.k.y), thinfilm.thickness);
      values.z = fresnel_thinfilm(thinfilm.rgb_wavelengths.z, cos_theta, cx(ext_ior.eta.z, ext_ior.k.z), cx(thinfilm.ior.eta.z, thinfilm.ior.k.z),
        cx(int_ior.eta.z, int_ior.k.z), thinfilm.thickness);
    }
    return {saturatef(values.x), saturatef(values.y), saturatef(values.z)};
  }
}

// scene_bsdf.hxx:110-126 evaluate_thinfilm
template <bool SP>
DEV ThinfilmEval<SP> evaluate_thinfilm(const DeviceScene& sc, float wavelength, const etxb_thinfilm& film, V2 uv, Smp& smp) {
  ThinfilmEval<SP> r;
  r.rgb_wavelengths = {610.0f, 537.0f, 450.0f};
  if (film.max_thickness * film.min_thickness <= 0.0f) {
    r.ior.cls = 0u;
    r.ior.eta = Spec<SP>::make(0.0f);
    r.ior.k = Spec<SP>::make(0.0f);
    r.thickness = 0.0f;
    return r;
  }
  float t = (film.thickness_image == kInvalidIndex) ? 1.0f : image_evaluate(sc.images[film.thickness_image], uv, nullptr).x;
  r.thickness = lerpf(film.min_thickness, film.max_thickness, t);
  if constexpr (SP) {
    r.rgb_wavelengths = {wavelength, wavelength, wavelength};
  } else {
    r.rgb_wavelengths.x = 610.0f + 45.0f * (2.0f * smp.next() - 1.0f);
    r.rgb_wavelengths.y = 537.0f + 47.0f * (2.0f * smp.next() - 1.0f);
    r.rgb_wavelengths.z = 450.0f + 23.5f * (2.0f * smp.next() - 1.0f);
  }
  r.ior = evaluate_ior<SP>(sc, film.ior, wavelength);
  return r;
}

// ---- microsurface random walk (bsdf_external.hxx:12-230) ---------------------------------------------------
constexpr uint32_t kScatteringOrderMax = 16u;

struct MicroRay {
  V3 w;
  float Lambda, h, C1, G1;

  DEV void update_direction(V3 in_w, V2 alpha) {
    w = in_w;
    if (w.z > 0.9999f) {
      Lambda = 0.0f;
      return;
    }
    if (w.z < -0.9999f) {
      Lambda = -1.0f;
      return;
    }
#if defined(ETXB_PARITY) && ETXB_PARITY
    const float theta = m_acos(w.z);
    const float cosTheta = w.z;
    const float sinTheta = m_sin(theta);
    const float tanTheta = sinTheta / cosTheta;
    const float invSinTheta2 = 1.0f / (1.0f - w.z * w.z);
    const float cosPhi2 = w.x * w.x * invSinTheta2;
    const float sinPhi2 = w.y * w.y * invSinTheta2;
    const float alpha_value = sqrtf(cosPhi2 * alpha.x * alpha.x + sinPhi2 * alpha.y * alpha.y);
    const float a = 1.0f / tanTheta / alpha_value;
    Lambda = 0.5f * (-1.0f + ((a > 0) ? 1.0f : -1.0f) * sqrtf(1.0f + 1.0f / (a * a)));
#else
    // the same Smith Lambda without the trip through the angle: tan(theta) * alpha(phi) = sqrt((x ax)^2 + (y ay)^2) / z, so
    // 1 / a^2 = ((x ax)^2 + (y ay)^2) / z^2 and sign(a) = sign(z)
    const float ax = w.x * alpha.x, ay = w.y * alpha.y;
    const float inv_a2 = __fdividef(ax * ax + ay * ay, w.z * w.z);
    Lambda = 0.5f * (-1.0f + copysignf(sqrtf(1.0f + inv_a2), w.z));
#endif
  }
  DEV void update_height(float in_h) {
    h = in_h;
    C1 = tmin(1.0f, tmax(0.0f, 0.5f * (h + 1.0f)));
    if (w.z > 0.9999f)
      G1 = 1.0f;
    else if (w.z <= 0.0f)
      G1 = 0.0f;
    else
      G1 = m_pow(C1, Lambda);
  }
};
DEV MicroRay micro_ray(V3 w, V2 alpha) {
  MicroRay r;
  r.Lambda = 0.0f;
  r.h = 0.0f;
  r.C1 = 0.0f;
  r.G1 = 0.0f;
  r.update_direction(w, alpha);
  return r;
}
DEV float inv_c1(float U) { return tmax(-1.0f, tmin(1.0f, 2.0f * U - 1.0f)); }
DEV float sample_height(const MicroRay& ray, float U) {
  if (ray.w.z > 0.9999f) return kMaxFloat;
  if (ray.w.z < -0.9999f) return inv_c1(U * ray.C1);
  if (fabsf(ray.w.z) < 0.0001f) return ray.h;
  if (U > 1.0f - ray.G1) return kMaxFloat;
  float P1 = m_pow((1.0f - U), 1.0f / ray.Lambda);
  if (P1 <= 0.0f) return kMaxFloat;
  float U1 = ray.C1 / P1;
  return inv_c1(U1);
}
DEV float d_ggx(V3 wm, V2 alpha) {
  if (wm.z <= kEpsilon) return 0.0f;
  const float slope_x = -wm.x / wm.z;
  const float slope_y = -wm.y / wm.z;
  const float ax = fmaxf(kEpsilon, alpha.x * alpha.x);
  const float ay = fmaxf(kEpsilon, alpha.y * alpha.y);
  const float axy = fmaxf(kEpsilon, alpha.x * alpha.y);
  const float tmp = 1.0f + slope_x * slope_x / ax + slope_y * slope_y / ay;
  const float P22 = 1.0f / (kPi * axy * tmp * tmp);
  return P22 / (wm.z * wm.z * wm.z * wm.z);
}
// slopes of the visible normals of a unit-roughness GGX surface seen from (sin_theta_i, 0, cos_theta_i)
DEV V2 sample_p22_11_cs(float cos_theta_i, float sin_theta_i, V2 rnd) {
  V2 slope = {0.0f, 0.0f};
  const float tan_theta_i = sin_theta_i / cos_theta_i;
  const float projectedarea = 0.5f * (cos_theta_i + 1.0f);
  if (projectedarea < 0.0001f) return {0.0f, 0.0f};
  const float c = 1.0f / projectedarea;
  const float A = 2.0f * rnd.x / cos_theta_i / c - 1.0f;
  const float B = tan_theta_i;
  const float tmp = 1.0f / (A * A - 1.0f);
  const float D = sqrtf(tmax(0.0f, B * B * tmp * tmp - (A * A - B * B) * tmp));
  const float slope_x_1 = B * tmp - D;
  const float slope_x_2 = B * tmp + D;
  slope.x = (A < 0.0f || slope_x_2 > 1.0f / tan_theta_i) ? slope_x_1 : slope_x_2;
  float U2, S;
  if (rnd.y > 0.5f) {
    S = 1.0f;
    U2 = 2.0f * (rnd.y - 0.5f);
  } else {
    S = -1.0f;
    U2 = 2.0f * (0.5f - rnd.y);
  }
  const float z = (U2 * (U2 * (U2 * 0.27385f - 0.73369f) + 0.46341f)) / (U2 * (U2 * (U2 * 0.093073f + 0.309420f) - 1.000000f) + 0.597999f);
  slope.y = S * z * sqrtf(1.0f + slope.x * slope.x);
  return slope;
}
DEV V2 sample_p22_11(float theta_i, V2 rnd, V2 alpha) {
  if (theta_i < 0.0001f) {
    const float r = sqrtf(rnd.x / (1.0f - rnd.x));
    const float phi = kDoublePi * rnd.y;
    return {r * m_cos(phi), r * m_sin(phi)};
  }
  return sample_p22_11_cs(m_cos(theta_i), m_sin(theta_i), rnd);
}
// sampleVNDF / the head of samplePhaseFunction_* (bsdf_external.hxx:177-205, 239-266): a visible micro-normal for the direction wi.
// Parity build: through acos / atan2 / sin / cos like the reference.  Product build: the stretched direction's own components ARE the
// cosine and sine of both angles, no transcendental is needed.
DEV V3 visible_micronormal(V2 rnd, V3 wi, V2 alpha) {
  const V3 wi_11 = normalize(V3{alpha.x * wi.x, alpha.y * wi.y, wi.z});
#if defined(ETXB_PARITY) && ETXB_PARITY
  V2 slope_11 = sample_p22_11(m_acos(wi_11.z), rnd, alpha);
  const float phi = m_atan2(wi_11.y, wi_11.x);
  V2 slope = {m_cos(phi) * slope_11.x - m_sin(phi) * slope_11.y, m_sin(phi) * slope_11.x + m_cos(phi) * slope_11.y};
#else
  const float sin_theta = sqrtf(wi_11.x * wi_11.x + wi_11.y * wi_11.y);
  V2 slope_11;
  float cos_phi = 1.0f, sin_phi = 0.0f;
  if ((sin_theta < 0.0001f) && (wi_11.z > 0.0f)) {  // theta_i < 1e-4: the isotropic closed form
    const float r = sqrtf(rnd.x / (1.0f - rnd.x));
    float s, c;
    __sincosf(kDoublePi * rnd.y - kPi, &s, &c);
    slope_11 = {-r * c, -r * s};
  } else {
    slope_11 = sample_p22_11_cs(wi_11.z, sin_theta, rnd);
  }
  if (sin_theta > 0.0f) {
    const float inv = 1.0f / sin_theta;
    cos_phi = wi_11.x * inv;
    sin_phi = wi_11.y * inv;
  } else if (signbit(wi_11.x)) {
    cos_phi = -1.0f;  // at normal incidence the reference rotates by atan2(+-0, -0) = +-pi: a negative zero x turns the slope round
  }
  V2 slope = {cos_phi * slope_11.x - sin_phi * slope_11.y, sin_phi * slope_11.x + cos_phi * slope_11.y};
#endif
  slope.x *= alpha.x;
  slope.y *= alpha.y;
  if ((slope.x != slope.x) || !finitef(slope.x)) {
    return (wi.z > 0) ? V3{0.0f, 0.0f, 1.0f} : normalize(V3{wi.x, wi.y, 0.0f});
  }
  return normalize(V3{-slope.x, -slope.y, 1.0f});
}
// shared head of samplePhaseFunction_{conductor,dielectric} (bsdf_external.hxx:239-266, 413-441): visible micro-normal
DEV V3 sample_visible_micronormal(V2 slope_rnd, V3 wi, V2 alpha) { return visible_micronormal(slope_rnd, wi, alpha); }

template <bool SP>
DEV Spec<SP> phase_function_reflection(float wavelength, const MicroRay& ray, V3 wo, V2 alpha, const IorSample<SP>& ext_ior, const IorSample<SP>& int_ior,
  const ThinfilmEval<SP>& thinfilm) {
  if (ray.w.z > 0.9999f) return Spec<SP>::make(0.0f);
  float projectedArea = (ray.w.z < -0.9999f) ? 1.0f : ray.Lambda * ray.w.z;
  if (projectedArea < kEpsilon) return Spec<SP>::make(0.0f);
  const V3 wh = normalize(-ray.w + wo);
  if (wh.z < 0.0f) return Spec<SP>::make(0.0f);
  float w_dot_h = dot(-ray.w, wh);
  if (w_dot_h < kEpsilon) return Spec<SP>::make(0.0f);
  const Spec<SP> f = fresnel_calculate<SP>(wavelength, w_dot_h, ext_ior, int_ior, thinfilm);
  const float dg = d_ggx(wh, alpha);
  const float d = dg / (4.0f * projectedArea);
  return f * d;
}

DEV float abgam(float x) {
  const float g0 = 1.0f / 12.0f, g1 = 1.0f / 30.0f, g2 = 53.0f / 210.0f, g3 = 195.0f / 371.0f, g4 = 22999.0f / 22737.0f, g5 = 29944523.0f / 19733142.0f,
              g6 = 109535241009.0f / 48264275462.0f;
  constexpr float kHalfLogDoublePi = 0.918938518f;
  return kHalfLogDoublePi - x + (x - 0.5f) * m_log(x) + g0 / (x + g1 / (x + g2 / (x + g3 / (x + g4 / (x + g5 / (x + g6 / x))))));
}
DEV float gamma_fn(float x) { return m_exp(abgam(x + 5.0f)) / (x * (x + 1.0f) * (x + 2.0f) * (x + 3.0f) * (x + 4.0f)); }
DEV float beta_fn(float m, float n) { return gamma_fn(m) * gamma_fn(n) / gamma_fn(m + n); }

DEV V3 refract_dir(V3 wi, V3 wm, float eta) {
  const float cos_theta_i = dot(wi, wm);
  const float cos_theta_t2 = 1.0f - (1.0f - cos_theta_i * cos_theta_i) / (eta * eta);
  const float cos_theta_t = -sqrtf(tmax(0.0f, cos_theta_t2));
  return wm * (dot(wi, wm) / eta + cos_theta_t) - wi / eta;
}

template <bool SP>
DEV Spec<SP> eval_phase_function_dielectric(float wavelength, const MicroRay& ray, V3 wo, bool reflection, const IorSample<SP>& ext_ior, const IorSample<SP>& int_ior,
  const ThinfilmEval<SP>& thinfilm, V2 alpha) {
  if (ray.w.z > 0.9999f) return Spec<SP>::make(0.0f);
  if (reflection) return phase_function_reflection<SP>(wavelength, ray, wo, alpha, ext_ior, int_ior, thinfilm);
  float projectedArea = (ray.w.z < -0.9999f) ? 1.0f : ray.Lambda * ray.w.z;
  if (projectedArea < kEpsilon) return Spec<SP>::make(0.0f);
  float eta = (int_ior.eta / ext_ior.eta).monochromatic();
  V3 wh = normalize(-ray.w + wo * eta);
  wh *= (wh.z > 0) ? 1.0f : -1.0f;
  float i_dot_m = -dot(wh, ray.w);
  if (i_dot_m < 0) return Spec<SP>::make(0.0f);
  float o_dot_m = dot(wo, wh);
  float scalar = eta * eta * i_dot_m * tmax(0.0f, -o_dot_m) * d_ggx(wh, alpha) / (projectedArea * sqr(i_dot_m + eta * o_dot_m));
  Spec<SP> f = fresnel_calculate<SP>(wavelength, i_dot_m, ext_ior, int_ior, thinfilm);
  return (1.0f - f) * scalar;
}

template <bool SP>
struct DielectricPhaseSample {
  V3 w_o;
  Spec<SP> weight;
  bool reflection;
};
template <bool SP>
DEV DielectricPhaseSample<SP> sample_phase_function_dielectric(float wavelength, V2 rnd_slope, float rnd_reflection, V3 wi, V2 alpha, const IorSample<SP>& ext_ior,
  const IorSample<SP>& int_ior, const ThinfilmEval<SP>& thinfilm) {
  V3 wm = sample_visible_micronormal(rnd_slope, wi, alpha);
  float i_dot_m = dot(wi, wm);
  Spec<SP> f = fresnel_calculate<SP>(wavelength, i_dot_m, ext_ior, int_ior, thinfilm);
  float eta = (int_ior.eta / ext_ior.eta).monochromatic();
  DielectricPhaseSample<SP> r;
  r.reflection = rnd_reflection < f.monochromatic();
  r.weight = r.reflection ? f : 1.0f - f;
  r.w_o = r.reflection ? (-wi + 2.0f * wm * i_dot_m) : normalize(refract_dir(wi, wm, eta));
  return r;
}
DEV float mis_weight_dielectric(V3 wi, V3 wo, bool reflection, float eta, V2 alpha) {
  if (reflection) {
    if (wi.x == -wo.x && wi.y == -wo.y && wi.z == -wo.z) return 1.0f;
    const V3 wh = normalize(wi + wo);
    return d_ggx((wh.z > 0) ? wh : -wh, alpha);
  } else {
    const V3 wh = normalize(wi + wo * eta);
    return d_ggx((wh.z > 0) ? wh : -wh, alpha);
  }
}

// bsdf_external.hxx:466-558
template <bool SP>
DEVN Spec<SP> eval_dielectric(float wavelength, Smp& smp, V3 wi, V3 wo, bool wo_outside, V2 alpha, const IorSample<SP>& ext_ior, const IorSample<SP>& int_ior,
  const ThinfilmEval<SP>& thinfilm) {
  if ((wi.z <= 0) || (wo.z <= 0 && wo_outside) || (wo.z >= 0 && !wo_outside)) return Spec<SP>::make(0.0f);
  MicroRay ray = micro_ray(-wi, alpha);
  ray.update_height(1.0f);
  bool outside = true;
  MicroRay ray_shadowing = micro_ray(wo_outside ? wo : -wo, alpha);
  Spec<SP> singleScattering = Spec<SP>::make(0.0f);
  Spec<SP> multipleScattering = Spec<SP>::make(0.0f);
  float wi_MISweight = 0.0f;
  float eta = (int_ior.eta / ext_ior.eta).monochromatic();
  int current_scatteringOrder = 0;
  while (current_scatteringOrder < int(kScatteringOrderMax)) {
    ray.update_height(sample_height(ray, smp.next()));
    if (ray.h == kMaxFloat) break;
    current_scatteringOrder++;
    if (current_scatteringOrder == 1) {
      Spec<SP> phasefunction = eval_phase_function_dielectric<SP>(wavelength, ray, wo, wo_outside, ext_ior, int_ior, thinfilm, alpha);
      float G2_G1;
      if (wo_outside)
        G2_G1 = (1.0f + (-ray.Lambda - 1.0f)) / (1.0f + (-ray.Lambda - 1.0f) + ray_shadowing.Lambda);
      else
        G2_G1 = (1.0f + (-ray.Lambda - 1.0f)) * beta_fn(1.0f + (-ray.Lambda - 1.0f), 1.0f + ray_shadowing.Lambda);
      if (finitef(G2_G1)) {
        singleScattering = phasefunction * G2_G1;
      }
    }
    if (current_scatteringOrder > 1) {
      Spec<SP> phasefunction;
      float MIS;
      if (outside) {
        phasefunction = eval_phase_function_dielectric<SP>(wavelength, ray, wo, wo_outside, ext_ior, int_ior, thinfilm, alpha);
        MIS = wi_MISweight / (wi_MISweight + mis_weight_dielectric(-ray.w, wo, wo_outside, eta, alpha));
      } else {
        phasefunction = eval_phase_function_dielectric<SP>(wavelength, ray, -wo, !wo_outside, int_ior, ext_ior, thinfilm, alpha);
        MIS = wi_MISweight / (wi_MISweight + mis_weight_dielectric(-ray.w, -wo, !wo_outside, 1.0f / eta, alpha));
      }
      ray_shadowing.update_height((outside == wo_outside) ? ray.h : -ray.h);
      multipleScattering += phasefunction * ray_shadowing.G1 * MIS;
    }
    V2 rnd_slope = (current_scatteringOrder == 1) && smp.has_fixed() ? V2{smp.fixed_u, smp.fixed_v} : smp.next_2d();
    float rnd_reflection = (current_scatteringOrder == 1) && smp.has_fixed() ? smp.fixed_w : smp.next();
    auto next_sample = sample_phase_function_dielectric<SP>(wavelength, rnd_slope, rnd_reflection, -ray.w, alpha, (outside ? ext_ior : int_ior),
      (outside ? int_ior : ext_ior), thinfilm);
    if (next_sample.reflection) {
      ray.update_direction(next_sample.w_o, alpha);
      ray.update_height(ray.h);
    } else {
      outside = !outside;
      ray.update_direction(-next_sample.w_o, alpha);
      ray.update_height(-ray.h);
    }
    if (current_scatteringOrder == 1) wi_MISweight = mis_weight_dielectric(wi, ray.w, outside, eta, alpha);
    if ((ray.h != ray.h) || (ray.w.x != ray.w.x) || (ray.w.z <= kEpsilon)) return Spec<SP>::make(0.0f);
  }
  return 0.5f * singleScattering + multipleScattering;
}

// ---- Diffuse (bsdf_various.hxx:36-133).  diffuse_variation 0 (Lambert) stays inline; 1 (rough microsurface walk) and 2 (vMF fit)
// go through ONE out-of-line routine (defined further down) ----------------------------------------------------------
template <bool SP>
DEVN BEval<SP> diffuse_layer_variation(const DeviceScene& sc, const BData& d, V3 local_w_i, V3 local_w_o, const etxb_material& m, Smp& smp);

// DiffuseBSDF::diffuse_layer (bsdf_various.hxx:36-71) — also the base layer of PlasticBSDF::evaluate (bsdf_plastic.hxx:136)
template <bool SP>
DEV BEval<SP> diffuse_layer(const DeviceScene& sc, const BData& d, V3 local_w_i, V3 local_w_o, const etxb_material& m, Smp& smp) {
  if (m.diffuse_variation != 0u) return diffuse_layer_variation<SP>(sc, d, local_w_i, local_w_o, m, smp);
  if (local_w_o.z <= 0.0f) return beval_zero<SP>();
  Spec<SP> diffuse = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength);
  BEval<SP> e;
  e.eta = 1.0f;
  e.func = diffuse / kPi;
  e.bsdf = e.func * local_w_o.z;
  e.pdf = kInvPi * local_w_o.z;
  return e;
}
// DiffuseBSDF::sample for variations 0 and 2 (bsdf_various.hxx:73-100): cosine lobe, weight = layer.bsdf / layer.pdf
template <bool SP>
DEV BSample<SP> diffuse_sample(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  Frame frame = normal_frame(d);
  V3 local_w_i = frame.to_local(-d.w_i);
  BSample<SP> r = bsample_zero<SP>();
  r.eta = 1.0f;
  r.properties = kBsdfReflection | kBsdfDiffuse;
  V2 cos_rnd = smp.has_fixed() ? V2{smp.fixed_u, smp.fixed_v} : smp.next_2d();
  V3 local_w_o = sample_cosine_local(cos_rnd, 1.0f);
  BEval<SP> dl = diffuse_layer<SP>(sc, d, local_w_i, local_w_o, m, smp);
  r.weight = dl.pdf == 0.0f ? Spec<SP>::make(0.0f) : dl.bsdf / dl.pdf;
  r.pdf = dl.pdf;
  r.w_o = frame.from_local(local_w_o);
  return r;
}
// DiffuseBSDF::evaluate (bsdf_various.hxx:102-111), every variation
template <bool SP>
DEV BEval<SP> diffuse_evaluate(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m, Smp& smp) {
  Frame frame = normal_frame(d);
  V3 local_w_o = frame.to_local(w_o);
  if (local_w_o.z <= kEpsilon) return beval_zero<SP>();
  V3 local_w_i = frame.to_local(-d.w_i);
  return diffuse_layer<SP>(sc, d, local_w_i, local_w_o, m, smp);
}
DEV float diffuse_pdf(const BData& d, V3 w_o) {
  float n_dot_o = dot(front_facing_normal(d), w_o);
  if (n_dot_o <= kEpsilon) return 0.0f;
  return kInvPi * n_dot_o;
}

// ---- Diffuse, diffuse_variation 1: Heitz/Dupuy rough diffuse microsurface, a random walk in BOTH sample and evaluate
// (bsdf_external.hxx:177-205 sampleVNDF, :557-578 samplePhaseFunction_diffuse, :580-629 eval_diffuse, :660-693 sample_diffuse) ----
DEV V3 sample_vndf(Smp& smp, V3 wi, V2 alpha) { return visible_micronormal(smp.next_2d(), wi, alpha); }
DEV V3 sample_phase_function_diffuse(Smp& smp, V3 wm) {
  float r1 = 2.0f * smp.next() - 1.0f;
  float r2 = 2.0f * smp.next() - 1.0f;
  float phi = 0.0f;
  float r = (r1 * r1 > r2 * r2) ? r1 : r2;
  if (r1 * r1 > r2 * r2) {
    phi = (kPi / 4.0f) * (r2 / r1);
  } else if ((r1 != 0.0f) && (r2 != 0.0f)) {
    phi = (kPi / 2.0f) - (r1 / r2) * (kPi / 4.0f);
  }
  float x = r * m_cos(phi);
  float y = r * m_sin(phi);
  float z = sqrtf(tmax(0.0f, 1.0f - x * x - y * y));
  Basis basis = orthonormal_basis(wm);
  return x * basis.u + y * basis.v + z * wm;
}
template <bool SP>
DEVN Spec<SP> eval_rough_diffuse(Smp& smp, V3 wi, V3 wo, V2 alpha, Spec<SP> albedo) {
  MicroRay ray_shadowing = micro_ray(wo, alpha);
  MicroRay ray = micro_ray(-wi, alpha);
  ray.update_height(1.0f);
  Spec<SP> res = Spec<SP>::make(0.0f);
  Spec<SP> energy = Spec<SP>::make(1.0f);
  int scattering_order = 0;
  while (true) {
    ray.update_height(sample_height(ray, smp.next()));
    if (ray.h == kMaxFloat) break;
    V3 wm = sample_vndf(smp, -ray.w, alpha);
    Spec<SP> phasefunction = energy * albedo * tmax(0.0f, dot(wm, wo) * kInvPi);
    if (scattering_order == 0) {
      float G2_G1 = -ray.Lambda / (ray_shadowing.Lambda - ray.Lambda);
      if (G2_G1 > 0) res += phasefunction * G2_G1;
    } else {
      ray_shadowing.update_height(ray.h);
      res += phasefunction * ray_shadowing.G1;
    }
    ray.update_direction(sample_phase_function_diffuse(smp, wm), alpha);
    ray.update_height(ray.h);
    energy = energy * albedo;
    if ((scattering_order++ > int(kScatteringOrderMax)) || (ray.h != ray.h) || (ray.w.x != ray.w.x)) return Spec<SP>::make(0.0f);
  }
  return res;
}
template <bool SP>
DEVN V3 sample_rough_diffuse(Smp& smp, V3 wi, V2 alpha, Spec<SP> albedo, Spec<SP>& energy) {
  energy = Spec<SP>::make(1.0f);
  MicroRay ray = micro_ray(-wi, alpha);
  ray.update_height(1.0f);
  int current_scatteringOrder = 0;
  while (true) {
    ray.update_height(sample_height(ray, smp.next()));
    if (ray.h == kMaxFloat) break;
    current_scatteringOrder++;
    V3 wm = sample_vndf(smp, -ray.w, alpha);
    ray.update_direction(sample_phase_function_diffuse(smp, wm), alpha);
    ray.update_height(ray.h);
    energy = energy * albedo;
    if (current_scatteringOrder > int(kScatteringOrderMax)) {
      energy = Spec<SP>::make(0.0f);
      return V3{0.0f, 0.0f, 1.0f};
    }
  }
  return ray.w;
}
// DiffuseBSDF::sample / evaluate for diffuse_variation 1 (bsdf_various.hxx:36-112)
template <bool SP>
DEV BSample<SP> rough_diffuse_sample(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  Frame frame = normal_frame(d);
  V3 local_w_i = frame.to_local(-d.w_i);
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  BSample<SP> r = bsample_zero<SP>();
  r.eta = 1.0f;
  r.properties = kBsdfReflection | kBsdfDiffuse;
  Spec<SP> diffuse = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength);
  V3 local_w_o = sample_rough_diffuse<SP>(smp, local_w_i, roughness, diffuse, r.weight);
  r.pdf = kInvPi * local_w_o.z;
  r.w_o = frame.from_local(local_w_o);
  return r;
}
// ---- Diffuse, diffuse_variation 2: d'Eon & Weidlich, "VMF Diffuse: A Unified Rough Diffuse BRDF" — a closed-form fit, no sampler
// draws (bsdf_external.hxx:696-897; the coefficients are the paper's, the operation order is the reference's) ----
DEV float erf_buermann(float x) {  // :700-705, Buermann series
  float e = m_exp(-x * x);
  return (x >= 0.0f ? 1.0f : -1.0f) * 2.0f / kSqrtPi * sqrtf(1.0f - e) * (kSqrtPi / 2.0f + 31.0f / 200.0f * e - 341.0f / 8000.0f * e * e);
}
DEV Spec<true> spec_erf(Spec<true> x) { return {erf_buermann(x.v)}; }
DEV Spec<false> spec_erf(Spec<false> x) {  // :707-715: the RGB overload works on whole responses (float3 sign / sqrt / exp)
  Spec<false> e = spec_exp(-(x * x));
  Spec<false> sg = {x.x >= 0.0f ? 1.0f : -1.0f, x.y >= 0.0f ? 1.0f : -1.0f, x.z >= 0.0f ? 1.0f : -1.0f};
  Spec<false> om = 1.0f - e;
  Spec<false> root = {sqrtf(om.x), sqrtf(om.y), sqrtf(om.z)};
  return sg * 2.0f / kSqrtPi * root * (31.0f / 200.0f * e + kSqrtPi / 2.0f - 341.0f / 8000.0f * e * e);
}
DEV Spec<true> spec_sqrt(Spec<true> a) { return {sqrtf(a.v)}; }
DEV Spec<false> spec_sqrt(Spec<false> a) { return {sqrtf(a.x), sqrtf(a.y), sqrtf(a.z)}; }
DEV Spec<true> spec_atan(Spec<true> a) { return {m_atan(a.v)}; }
DEV Spec<false> spec_atan(Spec<false> a) { return {m_atan(a.x), m_atan(a.y), m_atan(a.z)}; }
DEV Spec<true> spec_pow(Spec<true> a, Spec<true> b) { return {m_pow(a.v, b.v)}; }
DEV Spec<false> spec_pow(Spec<false> a, Spec<false> b) { return {m_pow(a.x, b.x), m_pow(a.y, b.y), m_pow(a.z, b.z)}; }
DEV Spec<true> spec_max0(Spec<true> a) { return {fmaxf(a.v, 0.0f)}; }
DEV Spec<false> spec_max0(Spec<false> a) { return {fmaxf(a.x, 0.0f), fmaxf(a.y, 0.0f), fmaxf(a.z, 0.0f)}; }

// multiple-scattering term of the fit (:717-722)
template <bool SP>
DEV Spec<SP> vmf_fm(float ui, float uo, float r, Spec<SP> c) {
  Spec<SP> C = spec_sqrt(1.0f - c);
  Spec<SP> Ck = (1.0f - 0.5441615108674713f * C - 0.45302863761693374f * (1.0f - c)) / (1.4293127703064865f * C + 1.0f);
  Spec<SP> Ca = c / spec_pow(1.16942f * C + 1.0075f, spec_atan((0.0225272f + (-0.264641f + r) * r) * spec_erf(c)));
  return spec_max0(0.384016f * (Ca + -0.341969f) * Ca * Ck * (-0.0578978f / (0.287663f + ui * uo) + fabsf(-0.0898863f + m_tanh(r))));
}
// cross section of a Beckmann surface, expanded for small m (:724-738)
DEV float vmf_sigma_beckmann_expanded(float u, float m) {
  if (0.0f == m) return (u + fabsf(u)) / 2.0f;
  float m2 = m * m;
  if (1.0f == u) return 1.0f - 0.5f * m2;
#if !(defined(ETXB_PARITY) && ETXB_PARITY)
  // u = -1 (a sampled w_o exactly along n: the product build's m_pow rounds sqrt(u) of the largest samples up to 1) is the limit 0 of the
  // expression below, which evaluates it as inf * 0
  if (-1.0f == u) return 0.0f;
#endif
  float expansion_term = -0.25f * m2 * (u + fabsf(u));
  float u2 = u * u;
  return ((m_exp(u2 / (m2 * (-1.0f + u2))) * m * sqrtf(1.0f - u2)) / sqrtf(kPi) + u * (1.0f + erf_buermann(u / (m * sqrtf(1.0f - u2))))) / 2.0f + expansion_term;
}
DEV float vmf_coth(float x) { return (m_exp(-x) + m_exp(x)) / (-m_exp(-x) + m_exp(x)); }  // :739-741
// vMF cross section (:743-785): Legendre-style expansion in u with closed-form coefficients in m
DEVN float vmf_sigma(float u, float m) {
  if (m < 0.25f) return vmf_sigma_beckmann_expanded(u, m);
  float m2 = m * m, m4 = m2 * m2, m8 = m4 * m4;
  float u2 = u * u, u4 = u2 * u2, u6 = u2 * u4, u8 = u4 * u4, u10 = u6 * u4, u12 = u6 * u6;
  float coth2m2 = vmf_coth(2.0f / m2);
  float sinh2m2 = m_sinh(2.0f / m2);
  if (m > 0.9f) return 0.25f - 0.25f * u * (m2 - 2.0f * coth2m2) + 0.0390625f * (-1.0f + 3.0f * u2) * (4.0f + 3.0f * m4 - 6.0f * m2 * coth2m2);
  float q2 = 1.0132789611816406e-6f * (35.0f - 1260.0f * u2 + 6930.0f * u4 - 12012.0f * u6 + 6435.0f * u8) * (1.0f + coth2m2) *
             (-256.0f - 315.0f * m4 * (128.0f + 33.0f * m4 * (80.0f + 364.0f * m4 + 195.0f * m8)) +
              18.0f * m2 * (256.0f + 385.0f * m4 * (32.0f + 312.0f * m4 + 585.0f * m8)) * coth2m2) *
             sinh2m2;
  float q1 = 9.12696123123169e-8f * (-63.0f + 3465.0f * u2 - 30030.0f * u4 + 90090.0f * u6 - 109395.0f * u8 + 46189.0f * u10) * (1.0f + coth2m2) *
             (-1024.0f - 495.0f * m4 * (768.0f + 91.0f * m4 * (448.0f + 15.0f * m4 * (448.0f + 1836.0f * m4 + 969.0f * m8))) +
              110.0f * m2 * (256.0f + 117.0f * m4 * (256.0f + 21.0f * m4 * (336.0f + 85.0f * m4 * (32.0f + 57.0f * m4)))) * coth2m2) *
             sinh2m2;
  float q0 = 4.3655745685100555e-9f * (231.0f - 18018.0f * u2 + 225225.0f * u4 - 1.02102e6f * u6 + 2.078505e6f * u8 - 1.939938e6f * u10 + 676039.0f * u12) *
             (1.0f + coth2m2) *
             (-4096.0f - 3003.0f * m4 * (1024.0f + 45.0f * m4 * (2560.0f + 51.0f * m4 * (1792.0f + 285.0f * m4 * (80.0f + 308.0f * m4 + 161.0f * m8)))) +
              78.0f * m2 * (2048.0f + 385.0f * m4 * (1280.0f + 153.0f * m4 * (512.0f + 57.0f * m4 * (192.0f + 35.0f * m4 * (40.0f + 69.0f * m4))))) * coth2m2) *
             sinh2m2;
  float e2m2 = m_exp(2.0f / m2);
  return 0.25f - 0.25f * u * (m2 - 2.0f * coth2m2) + 0.0390625f * (-1.0f + 3.0f * u2) * (4.0f + 3.0f * m4 - 6.0f * m2 * coth2m2) -
         0.000732421875f * (3.0f - 30.0f * u2 + 35.0f * u4) * (16.0f + 180.0f * m4 + 105.0f * m8 - 10.0f * m2 * (8.0f + 21.0f * m4) * coth2m2) +
         0.000049591064453125f * (-5.0f + 105.0f * u2 - 315.0f * u4 + 231.0f * u6) *
           (64.0f + 105.0f * m4 * (32.0f + 180.0f * m4 + 99.0f * m8) - 42.0f * m2 * (16.0f + 240.0f * m4 + 495.0f * m8) * coth2m2) +
         (q2 / e2m2) - (q1 / e2m2) + (q0 / e2m2);
}
// vMFdiffuseBRDF (:787-894): three single/multiple-scattering orders as low-order Fourier series in the azimuth difference
template <bool SP>
DEVN Spec<SP> vmf_diffuse_brdf(V3 w_i, V3 w_o, V2 roughness, Spec<SP> albedo) {
  float r = sqrtf(roughness.x * roughness.y);
  const float r_max = 1.0f - 4.0f * kEpsilon;
  r = (r < 0.0f) ? 0.0f : (r > r_max ? r_max : r);
  if (r == 0.0f) return albedo * kInvPi;
  float cos_theta_i = w_i.z;
  float sin_theta_i = sqrtf(1.0f - cos_theta_i * cos_theta_i);
  float cos_theta_o = w_o.z;
  float sin_theta_o = sqrtf(1.0f - cos_theta_o * cos_theta_o);
  float cos_phi_diff = 0.0f;
  if (sin_theta_i > 0.0f && sin_theta_o > 0.0f) {
    auto clamp11 = [](float v) { return (v < -1.0f) ? -1.0f : (v > 1.0f ? 1.0f : v); };
    float sin_phi_i = clamp11(w_i.y / sin_theta_i);
    float cos_phi_i = clamp11(w_i.x / sin_theta_i);
    float sin_phi_o = clamp11(w_o.y / sin_theta_o);
    float cos_phi_o = clamp11(w_o.x / sin_theta_o);
    cos_phi_diff = clamp11(cos_phi_i * cos_phi_o + sin_phi_i * sin_phi_o);
  }
  float phi = m_acos(cos_phi_diff);
  float ui = w_i.z, uo = w_o.z;
  float m = -m_log(1.0f - sqrtf(r));
  float sigmai = vmf_sigma(ui, m);
  float sigmao = vmf_sigma(uo, m);
  float sigmano = vmf_sigma(-uo, m);
  float sigio = sigmai * sigmao;
  float sigdenom = uo * sigmai + ui * sigmano;
  float r2 = r * r;
  float r25 = r2 * sqrtf(r);
  float r3 = r * r2;
  float r4 = r2 * r2;
  float r45 = r4 * sqrtf(r);
  float r5 = r3 * r2;
  float ui2 = saturatef(ui * ui);
  float uo2 = saturatef(uo * uo);
  float sqrtuiuo = sqrtf((1.0f - ui2) * (1.0f - uo2));

  float C100 = 1.0f + (-0.1f * r + 0.84f * r4) / (1.0f + 9.0f * r3);
  float C101 = (0.0173f * r + 20.4f * r2 - 9.47f * r3) / (1.0f + 7.46f * r);
  float C102 = (-0.927f * r + 2.37f * r2) / (1.24f + r2);
  float C103 = (-0.110f * r - 1.54f * r2) / (1.0f - 1.05f * r + 7.1f * r2);
  float f10 = ((C100 + C101 * ui * uo + C102 * ui2 * uo2 + C103 * (ui2 + uo2)) * sigio) / sigdenom;

  float C110 = (0.54f * r - 0.182f * r3) / (1.0f + 1.32f * r2);
  float C111 = (-0.097f * r + 0.62f * r2 - 0.375f * r3) / (1.0f + 0.4f * r3);
  float C112 = 0.283f + 0.862f * r - 0.681f * r2;
  float f11 = (sqrtuiuo * (C110 + C111 * ui * uo)) * m_pow(sigio, C112) / sigdenom;

  float C120 = (2.25f * r + 5.1f * r2) / (1.0f + 9.8f * r + 32.4f * r2);
  float C121 = (-4.32f * r + 6.0f * r3) / (1.0f + 9.7f * r + 287.0f * r3);
  float f12 = ((1.0f - ui2) * (1.0f - uo2) * (C120 + C121 * uo) * (C120 + C121 * ui)) / (ui + uo);

  float C200 = (0.00056f * r + 0.226f * r2) / (1.0f + 7.07f * r2);
  float C201 = (-0.268f * r + 4.57f * r2 - 12.04f * r3) / (1.0f + 36.7f * r3);
  float C202 = (0.418f * r + 2.52f * r2 - 0.97f * r3) / (1.0f + 10.0f * r2);
  float C203 = (0.068f * r - 2.25f * r2 + 2.65f * r3) / (1.0f + 21.4f * r3);
  float C204 = (0.050f * r - 4.22f * r3) / (1.0f + 17.6f * r2 + 43.1f * r3);
  float f20 = (C200 + C201 * ui * uo + C203 * ui2 * uo2 + C202 * (ui + uo) + C204 * (ui2 + uo2)) / (ui + uo);

  float C210 = (-0.049f * r - 0.027f * r3) / (1.0f + 3.36f * r2);
  float C211 = (2.77f * r2 - 8.332f * r25 + 6.073f * r3) / (1.0f + 50.0f * r4);
  float C212 = (-0.431f * r2 - 0.295f * r3) / (1.0f + 23.9f * r3);
  float f21 = (sqrtuiuo * (C210 + C211 * ui * uo + C212 * (ui + uo))) / (ui + uo);

  float C300 = (-0.083f * r3 + 0.262f * r4) / (1.0f - 1.9f * r2 + 38.6f * r4);
  float C301 = (-0.627f * r2 + 4.95f * r25 - 2.44f * r3) / (1.0f + 31.5f * r4);
  float C302 = (0.33f * r2 + 0.31f * r25 + 1.4f * r3) / (1.0f + 20.0f * r3);
  float C303 = (-0.74f * r2 + 1.77f * r25 - 4.06f * r3) / (1.0f + 215.0f * r5);
  float C304 = (-1.026f * r3) / (1.0f + 5.81f * r2 + 13.2f * r3);
  float f30 = (C300 + C301 * ui * uo + C303 * ui2 * uo2 + C302 * (ui + uo) + C304 * (ui2 + uo2)) / (ui + uo);

  float C310 = (0.028f * r2 - 0.0132f * r3) / (1.0f + 7.46f * r2 - 3.315f * r4);
  float C311 = (-0.134f * r2 + 0.162f * r25 + 0.302f * r3) / (1.0f + 57.5f * r45);
  float C312 = (-0.119f * r2 + 0.5f * r25 - 0.207f * r3) / (1.0f + 18.7f * r3);
  float f31 = (sqrtuiuo * (C310 + C311 * ui * uo + C312 * (ui + uo))) / (ui + uo);

  Spec<SP> t0 = albedo * tmax(0.0f, f10 + f11 * m_cos(phi) * 2.0f + f12 * m_cos(2.0f * phi) * 2.0f);
  Spec<SP> t1 = albedo * albedo * tmax(0.0f, f20 + f21 * m_cos(phi) * 2.0f);
  Spec<SP> t2 = albedo * albedo * albedo * tmax(0.0f, f30 + f31 * m_cos(phi) * 2.0f);
  Spec<SP> t4 = vmf_fm<SP>(ui, uo, r, albedo);
  return kInvPi * (t0 + t1 + t2) + t4;
}

// DiffuseBSDF::diffuse_layer for variations 1 and 2 (bsdf_various.hxx:36-71)
template <bool SP>
DEVN BEval<SP> diffuse_layer_variation(const DeviceScene& sc, const BData& d, V3 local_w_i, V3 local_w_o, const etxb_material& m, Smp& smp) {
  if (local_w_o.z <= 0.0f) return beval_zero<SP>();
  Spec<SP> diffuse = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength);
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  BEval<SP> e;
  e.eta = 1.0f;
  if (m.diffuse_variation == 1u) {
    e.bsdf = eval_rough_diffuse<SP>(smp, local_w_i, local_w_o, roughness, diffuse);
    e.func = e.bsdf / local_w_o.z;
  } else {
    e.func = vmf_diffuse_brdf<SP>(local_w_i, local_w_o, roughness, diffuse);
    e.bsdf = e.func * local_w_o.z;
  }
  e.pdf = kInvPi * local_w_o.z;
  return e;
}

// ---- Dielectric (bsdf_dielectric.hxx:60-259) ---------------------------------------------------------------
DEV bool dielectric_is_delta(const DeviceScene& sc, const etxb_material& m, V2 tex) {
  V2 r = evaluate_roughness(sc, m, tex);
  return tmax(r.x, r.y) <= kDeltaAlphaTreshold;
}
template <bool SP>
DEVN float dielectric_pdf(const DeviceScene& sc, const BData& d, V3 in_w_o, const etxb_material& m, Smp& smp) {
  Frame lf = {d.tan, d.btn, d.nrm, false};
  V3 w_i = lf.to_local(-d.w_i);
  if (fabsf(w_i.z) <= kEpsilon) return 0.0f;
  V3 w_o = lf.to_local(in_w_o);
  if (fabsf(w_o.z) <= kEpsilon) return 0.0f;
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  IorSample<SP> ext_ior = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> int_ior = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  const bool outside = w_i.z > 0;
  const bool reflection = w_i.z * w_o.z > 0.0f;
  V3 wh;
  float dwh_dwo;
  if (reflection) {
    wh = normalize(w_o + w_i);
    dwh_dwo = 1.0f / (4.0f * dot(w_o, wh));
  } else {
    float eta = outside ? (int_ior.eta / ext_ior.eta).monochromatic() : (ext_ior.eta / int_ior.eta).monochromatic();
    wh = normalize(w_i + w_o * eta);
    float sqrt_denom = dot(w_i, wh) + eta * dot(w_o, wh);
    dwh_dwo = sqr(eta) * dot(w_o, wh) / sqr(sqrt_denom);
  }
  wh *= (wh.z >= 0.0f) ? 1.0f : -1.0f;
  MicroRay ray = micro_ray(w_i * (outside ? 1.0f : -1.0f), roughness);
  float dg = d_ggx(wh, roughness);
  float prob = tmax(0.0f, dot(wh, ray.w) * dg / ((1.0f + ray.Lambda) * ray.w.z));
  float f = fresnel_calculate<SP>(d.wavelength, dot(w_i, wh), outside ? ext_ior : int_ior, outside ? int_ior : ext_ior, thinfilm).monochromatic();
  prob *= reflection ? f : (1.0f - f);
  return fabsf(prob * dwh_dwo) + fabsf(w_o.z);
}
template <bool SP>
DEVN BSample<SP> dielectric_sample(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  Frame lf = {d.tan, d.btn, d.nrm, false};
  V3 w_i = lf.to_local(-d.w_i);
  bool in_outside = w_i.z > 0;
  float direction_scale = in_outside ? 1.0f : -1.0f;
  IorSample<SP> ext_ior = in_outside ? evaluate_ior<SP>(sc, m.ext_ior, d.wavelength) : evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  IorSample<SP> int_ior = in_outside ? evaluate_ior<SP>(sc, m.int_ior, d.wavelength) : evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  BSample<SP> result = bsample_zero<SP>();
  result.weight = Spec<SP>::make(1.0f);
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  MicroRay ray = micro_ray(-direction_scale * w_i, roughness);
  ray.update_height(1.0f);
  bool ray_outside = true;
  uint32_t scattering_order = 0;
  while (true) {
    float sampled_height = sample_height(ray, smp.next());
    if (sampled_height == kMaxFloat) break;
    ray.update_height(sampled_height);
    V2 rnd_slope = (scattering_order == 0) && smp.has_fixed() ? V2{smp.fixed_u, smp.fixed_v} : smp.next_2d();
    float rnd_reflection = (scattering_order == 0) && smp.has_fixed() ? smp.fixed_w : smp.next();
    auto s = sample_phase_function_dielectric<SP>(d.wavelength, rnd_slope, rnd_reflection, -ray.w, roughness, (ray_outside ? ext_ior : int_ior),
      (ray_outside ? int_ior : ext_ior), thinfilm);
    result.weight *= s.weight;
    if (s.reflection) {
      ray.update_direction(s.w_o, roughness);
      ray.update_height(ray.h);
    } else {
      ray_outside = !ray_outside;
      ray.update_direction(-s.w_o, roughness);
      ray.update_height(-ray.h);
    }
    if (scattering_order++ > kScatteringOrderMax) {
      return bsample_zero<SP>();
    }
  }
  V3 lw_o = direction_scale * (ray_outside ? ray.w : -ray.w);
  uint32_t delta_sample = dielectric_is_delta(sc, m, d.tex) ? kBsdfDelta : 0u;
  if (w_i.z * lw_o.z > 0.0f) {
    result.eta = 1.0f;
    result.weight = (result.weight / result.weight.monochromatic()) * apply_image<SP>(sc, m.reflectance, d.tex, d.wavelength);
    result.properties = kBsdfReflection | delta_sample;
    result.medium_index = d.current_medium;
  } else {
    float eta = (int_ior.eta / ext_ior.eta).monochromatic();
    float factor = sqr(1.0f / eta);
    result.eta = eta;
    result.weight = (result.weight / result.weight.monochromatic()) * apply_image<SP>(sc, m.scattering, d.tex, d.wavelength) * factor;
    result.properties = kBsdfTransmission | kBsdfMediumChanged | delta_sample;
    result.medium_index = in_outside ? m.int_medium : m.ext_medium;
  }
  result.w_o = normalize(lf.from_local(lw_o));
  result.pdf = dielectric_pdf<SP>(sc, d, result.w_o, m, smp);
  return result;
}
template <bool SP>
DEVN BEval<SP> dielectric_evaluate(const DeviceScene& sc, const BData& d, V3 in_w_o, const etxb_material& m, Smp& smp) {
  Frame lf = {d.tan, d.btn, d.nrm, false};
  V3 w_i = lf.to_local(-d.w_i);
  if (fabsf(w_i.z) <= kEpsilon) return beval_zero<SP>();
  V3 w_o = lf.to_local(in_w_o);
  if (fabsf(w_o.z) <= kEpsilon) return beval_zero<SP>();
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  IorSample<SP> ext_ior = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> int_ior = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  bool forward_path = d.path_source == kPathCamera;
  float backward_scale = fabsf(1.0f / w_i.z);
  Spec<SP> value;
  float wl = d.wavelength;
  if (w_i.z > 0) {
    if (w_o.z >= 0) {
      value = forward_path ? eval_dielectric<SP>(wl, smp, w_i, w_o, true, roughness, ext_ior, int_ior, thinfilm)
                           : eval_dielectric<SP>(wl, smp, w_o, w_i, true, roughness, ext_ior, int_ior, thinfilm) * backward_scale;
    } else {
      value = forward_path ? eval_dielectric<SP>(wl, smp, w_i, w_o, false, roughness, ext_ior, int_ior, thinfilm)
                           : eval_dielectric<SP>(wl, smp, -w_o, -w_i, false, roughness, int_ior, ext_ior, thinfilm) * backward_scale;
    }
  } else if (w_o.z <= 0) {
    value = forward_path ? eval_dielectric<SP>(wl, smp, -w_i, -w_o, true, roughness, int_ior, ext_ior, thinfilm)
                         : eval_dielectric<SP>(wl, smp, -w_o, -w_i, true, roughness, int_ior, ext_ior, thinfilm) * backward_scale;
  } else {
    value = forward_path ? eval_dielectric<SP>(wl, smp, -w_i, -w_o, false, roughness, int_ior, ext_ior, thinfilm)
                         : eval_dielectric<SP>(wl, smp, w_o, w_i, false, roughness, ext_ior, int_ior, thinfilm) * backward_scale;
  }
  if (value.is_zero()) return beval_zero<SP>();
  bool reflection = w_i.z * w_o.z > 0.0f;
  BEval<SP> e;
  e.eta = 1.0f;
  e.func = (2.0f * value) * apply_image<SP>(sc, reflection ? m.reflectance : m.scattering, d.tex, d.wavelength);
  e.bsdf = e.func * fabsf(w_o.z);
  e.pdf = dielectric_pdf<SP>(sc, d, in_w_o, m, smp);
  return e;
}

// ---- conductor pieces of the microsurface walk (bsdf_external.hxx:233-344) ------------------------------------
template <bool SP>
DEV V3 sample_phase_function_conductor(float wavelength, V2 slope_rnd, V3 wi, V2 alpha, const IorSample<SP>& ext_ior, const IorSample<SP>& int_ior,
  const ThinfilmEval<SP>& thinfilm, Spec<SP>& weight) {
  V3 wm = sample_visible_micronormal(slope_rnd, wi, alpha);
  float i_dot_m = dot(wi, wm);
  weight = fresnel_calculate<SP>(wavelength, i_dot_m, ext_ior, int_ior, thinfilm);
  return -wi + 2.0f * wm * i_dot_m;
}
DEV float mis_weight_conductor(V3 wi, V3 wo, V2 alpha) {
  if (wi.x == -wo.x && wi.y == -wo.y && wi.z == -wo.z) return 1.0f;
  const V3 wh = normalize(wi + wo);
  return d_ggx((wh.z > 0) ? wh : -wh, alpha);
}
template <bool SP>
DEVN Spec<SP> eval_conductor(float wavelength, Smp& smp, V3 wi, V3 wo, V2 alpha, const IorSample<SP>& ext_ior, const IorSample<SP>& int_ior, const ThinfilmEval<SP>& thinfilm) {
  if (wi.z <= 0 || wo.z <= 0) return Spec<SP>::make(0.0f);
  MicroRay ray = micro_ray(-wi, alpha);
  ray.update_height(1.0f);
  Spec<SP> energy = Spec<SP>::make(1.0f);
  MicroRay ray_shadowing = micro_ray(wo, alpha);
  const V3 wh = normalize(wi + wo);
  const float D = d_ggx(wh, alpha);
  const float G2 = 1.0f / (1.0f + (-ray.Lambda - 1.0f) + ray_shadowing.Lambda);
  Spec<SP> singleScattering = fresnel_calculate<SP>(wavelength, dot(ray.w, wh), ext_ior, int_ior, thinfilm) * D * G2 / (4.0f * wi.z);
  float wi_MISweight = 0.0f;
  Spec<SP> multipleScattering = Spec<SP>::make(0.0f);
  uint32_t current_scatteringOrder = 0;
  while (current_scatteringOrder < kScatteringOrderMax) {
    ray.update_height(sample_height(ray, smp.next()));
    if (ray.h == kMaxFloat) break;
    current_scatteringOrder++;
    if (current_scatteringOrder > 1) {
      Spec<SP> phasefunction = phase_function_reflection<SP>(wavelength, ray, wo, alpha, ext_ior, int_ior, thinfilm);
      ray_shadowing.update_height(ray.h);
      float shadowing = ray_shadowing.G1;
      Spec<SP> I = energy * phasefunction * shadowing;
      const float MIS = wi_MISweight / (wi_MISweight + mis_weight_conductor(-ray.w, wo, alpha));
      multipleScattering += I * MIS;
    }
    V2 slope_rnd = (current_scatteringOrder == 1) && smp.has_fixed() ? V2{smp.fixed_u, smp.fixed_v} : smp.next_2d();
    Spec<SP> weight;
    ray.update_direction(sample_phase_function_conductor<SP>(wavelength, slope_rnd, -ray.w, alpha, ext_ior, int_ior, thinfilm, weight), alpha);
    energy = energy * weight;
    ray.update_height(ray.h);
    if (current_scatteringOrder == 1) wi_MISweight = mis_weight_conductor(wi, ray.w, alpha);
    if ((ray.h != ray.h) || (ray.w.x != ray.w.x)) return Spec<SP>::make(0.0f);
  }
  return 0.5f * singleScattering + multipleScattering;
}

// ---- Conductor (bsdf_conductor.hxx) -----------------------------------------------------------------------------
DEV float conductor_pdf_local(V3 w_i, V3 w_o, V2 roughness) {
  MicroRay ray = micro_ray(w_i, roughness);
  return d_ggx(normalize(w_o + w_i), roughness) / (1.0f + ray.Lambda) / (4.0f * w_i.z) + w_o.z;
}
template <bool SP>
DEVN BSample<SP> conductor_sample(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  Frame lf = normal_frame(d);
  V3 w_i = lf.to_local(-d.w_i);
  IorSample<SP> ext_ior = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> int_ior = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  uint32_t delta_sample = dielectric_is_delta(sc, m, d.tex) ? kBsdfDelta : 0u;
  BSample<SP> result = bsample_zero<SP>();
  result.properties = kBsdfReflection | delta_sample;
  result.medium_index = d.current_medium;
  result.eta = 1.0f;
  result.weight = Spec<SP>::make(1.0f);
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  MicroRay ray = micro_ray(-w_i, roughness);
  ray.update_height(1.0f);
  uint32_t scattering_order = 0;
  while (true) {
    ray.update_height(sample_height(ray, smp.next()));
    if (ray.h == kMaxFloat) break;
    V2 slope_rnd = (scattering_order == 0) && smp.has_fixed() ? V2{smp.fixed_u, smp.fixed_v} : smp.next_2d();
    Spec<SP> weight = Spec<SP>::make(1.0f);
    ray.update_direction(sample_phase_function_conductor<SP>(d.wavelength, slope_rnd, -ray.w, roughness, ext_ior, int_ior, thinfilm, weight), roughness);
    ray.update_height(ray.h);
    result.weight *= weight;
    if ((scattering_order++ > kScatteringOrderMax) || (ray.h != ray.h) || (ray.w.x != ray.w.x)) {
      result.weight = Spec<SP>::make(0.0f);
      ray.w = V3{0, 0, 1};
      break;
    }
  }
  V3 lw_o = ray.w;
  result.weight *= apply_image<SP>(sc, m.reflectance, d.tex, d.wavelength);
  result.pdf = conductor_pdf_local(w_i, lw_o, roughness);
  result.w_o = normalize(lf.from_local(lw_o));
  return result;
}
template <bool SP>
DEVN BEval<SP> conductor_evaluate(const DeviceScene& sc, const BData& d, V3 in_w_o, const etxb_material& m, Smp& smp) {
  Frame lf = normal_frame(d);
  V3 w_o = lf.to_local(in_w_o);
  if (w_o.z <= kEpsilon) return beval_zero<SP>();
  V3 w_i = lf.to_local(-d.w_i);
  if (w_i.z <= kEpsilon) return beval_zero<SP>();
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  IorSample<SP> ext_ior = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> int_ior = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  Spec<SP> value = eval_conductor<SP>(d.wavelength, smp, w_i, w_o, roughness, ext_ior, int_ior, thinfilm);
  BEval<SP> e;
  e.eta = 1.0f;
  e.bsdf = value * apply_image<SP>(sc, m.reflectance, d.tex, d.wavelength);
  e.func = e.bsdf / w_o.z;
  e.pdf = conductor_pdf_local(w_i, w_o, roughness);
  return e;
}
DEV float conductor_pdf(const DeviceScene& sc, const BData& d, V3 in_w_o, const etxb_material& m) {
  Frame lf = normal_frame(d);
  V3 w_o = lf.to_local(in_w_o);
  if (w_o.z <= kEpsilon) return 0.0f;
  V3 w_i = lf.to_local(-d.w_i);
  if (w_i.z <= kEpsilon) return 0.0f;
  return conductor_pdf_local(w_i, w_o, evaluate_roughness(sc, m, d.tex));
}

// ---- Plastic (bsdf_plastic.hxx) + GGX NormalDistribution::sample (bsdf.hxx:125-142) --------------------------------
DEV V3 ggx_sample_normal(const Frame& frame, V2 alpha_in, Smp& smp, V3 in_w_i) {
  const float kMinAlpha = 1.0f / 256.0f;
  V2 alpha = {fmaxf(kMinAlpha, alpha_in.x), fmaxf(kMinAlpha, alpha_in.y)};
  V3 w_i = frame.to_local(-in_w_i);
  V3 v_h = normalize(V3{alpha.x * w_i.x, alpha.y * w_i.y, w_i.z});
  float v_h_len = v_h.x * v_h.x + v_h.y * v_h.y;
  V3 u = v_h_len > 0.0f ? V3{-v_h.y, v_h.x, 0.0f} / sqrtf(v_h_len) : V3{1.0f, 0.0f, 0.0f};
  V3 v = cross(v_h, u);
  float r = sqrtf(smp.next());
  float phi = kDoublePi * smp.next();
  float t1 = r * m_cos(phi);
  float t2 = r * m_sin(phi);
  float s = 0.5f * (1.0f + v_h.z);
  t2 = (1.0f - s) * sqrtf(1.0f - t1 * t1) + s * t2;
  V3 n_h = t1 * u + t2 * v + sqrtf(tmax(0.0f, 1.0f - t1 * t1 - t2 * t2)) * v_h;
  V3 local_m = normalize(V3{alpha.x * n_h.x, alpha.y * n_h.y, n_h.z});
  return frame.from_local(local_m);
}
template <bool SP>
DEVN Spec<SP> plastic_specular_func(const DeviceScene& sc, const BData& d, V3 in_w_o, const etxb_material& m, Smp& smp) {
  Frame lf = {d.tan, d.btn, d.nrm, false};
  V3 w_i = lf.to_local(-d.w_i);
  if (w_i.z <= kEpsilon) return Spec<SP>::make(0.0f);
  V3 w_o = lf.to_local(in_w_o);
  if (w_o.z <= kEpsilon) return Spec<SP>::make(0.0f);
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  IorSample<SP> ext_ior = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> int_ior = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  Spec<SP> value = eval_dielectric<SP>(d.wavelength, smp, w_i, w_o, true, roughness, ext_ior, int_ior, thinfilm);
  return 2.0f * value * apply_image<SP>(sc, m.reflectance, d.tex, d.wavelength);
}
template <bool SP>
DEVN float plastic_specular_pdf(const DeviceScene& sc, const BData& d, V3 in_w_o, const etxb_material& m, Smp& smp) {
  Frame lf = {d.tan, d.btn, d.nrm, false};
  V3 w_i = lf.to_local(-d.w_i);
  if (w_i.z <= kEpsilon) return 0.0f;
  V3 w_o = lf.to_local(in_w_o);
  if (w_o.z <= kEpsilon) return 0.0f;
  IorSample<SP> ext_ior = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> int_ior = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  V3 wh = normalize(w_o + w_i);
  float dwh_dwo = 1.0f / (4.0f * dot(w_o, wh));
  MicroRay ray = micro_ray(w_i, roughness);
  float dg = d_ggx(wh, roughness);
  float prob = tmax(0.0f, dot(wh, ray.w) * dg / ((1.0f + ray.Lambda) * ray.w.z));
  float f = fresnel_calculate<SP>(d.wavelength, dot(w_i, wh), ext_ior, int_ior, thinfilm).monochromatic();
  prob *= f;
  return fabsf(prob * dwh_dwo);
}
template <bool SP>
DEVN BEval<SP> plastic_evaluate(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m, Smp& smp) {
  Frame frame = normal_frame(d);
  V3 mh = normalize(w_o - d.w_i);
  float n_dot_o = dot(frame.nrm, w_o);
  float m_dot_o = dot(mh, w_o);
  if ((n_dot_o <= kEpsilon) || (m_dot_o <= kEpsilon)) return beval_zero<SP>();
  IorSample<SP> eta_e = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> eta_i = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  Spec<SP> fr = fresnel_calculate<SP>(d.wavelength, dot(d.w_i, mh), eta_e, eta_i, thinfilm);
  V3 local_w_o = frame.to_local(w_o);
  V3 local_w_i = frame.to_local(-d.w_i);
  BEval<SP> diff_layer = diffuse_layer<SP>(sc, d, local_w_i, local_w_o, m, smp);
  Spec<SP> spec_layer = plastic_specular_func<SP>(sc, d, w_o, m, smp);
  float spec_pdf = plastic_specular_pdf<SP>(sc, d, w_o, m, smp);
  BEval<SP> e;
  e.eta = 1.0f;
  e.func = diff_layer.func * (1.0f - fr) + spec_layer / n_dot_o;
  e.bsdf = diff_layer.func * (1.0f - fr) * n_dot_o + spec_layer;
  e.pdf = diff_layer.pdf * (1.0f - fr).monochromatic() + spec_pdf;
  return e;
}
template <bool SP>
DEVN float plastic_pdf(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m, Smp& smp) {
  Frame frame = normal_frame(d);
  V3 mh = normalize(w_o - d.w_i);
  float m_dot_o = dot(mh, w_o);
  float n_dot_o = dot(frame.nrm, w_o);
  if ((n_dot_o <= kEpsilon) || (m_dot_o <= kEpsilon)) return 0.0f;
  IorSample<SP> eta_e = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> eta_i = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  Spec<SP> fr = fresnel_calculate<SP>(d.wavelength, dot(d.w_i, mh), eta_e, eta_i, thinfilm);
  float diff_pdf = kInvPi * n_dot_o;
  float spec_pdf = plastic_specular_pdf<SP>(sc, d, w_o, m, smp);
  return diff_pdf * (1.0f - fr).monochromatic() + spec_pdf;
}
template <bool SP>
DEVN BSample<SP> plastic_sample(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  Frame frame = normal_frame(d);
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  V3 mh = ggx_sample_normal(frame, roughness, smp, d.w_i);
  IorSample<SP> ext_ior = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> int_ior = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  Spec<SP> f = fresnel_calculate<SP>(d.wavelength, dot(d.w_i, mh), ext_ior, int_ior, thinfilm);
  V3 w_i = frame.to_local(-d.w_i);
  if (w_i.z <= kEpsilon) return bsample_zero<SP>();
  V3 in_w_o = {0.0f, 0.0f, 0.0f};
  bool sample_diffuse = smp.next() > f.monochromatic();
  if (sample_diffuse == false) {
    in_w_o = reflect(d.w_i, mh);
    sample_diffuse = dot(frame.nrm, in_w_o) <= kEpsilon;
  }
  if (sample_diffuse) {
    in_w_o = frame.from_local(sample_cosine_local(smp.next_2d(), 1.0f));
  }
  BEval<SP> eval = plastic_evaluate<SP>(sc, d, in_w_o, m, smp);
  BSample<SP> r = bsample_zero<SP>();
  r.w_o = in_w_o;
  r.weight = eval.bsdf / eval.pdf;
  r.properties = kBsdfReflection | (sample_diffuse ? kBsdfDiffuse : 0u);
  r.medium_index = d.current_medium;
  r.pdf = eval.pdf;
  return r;
}

// ---- Thinfilm class (delta; bsdf_dielectric.hxx:3-58) -----------------------------------------------------------
template <bool SP>
DEV BSample<SP> thinfilm_sample(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  Frame frame = normal_frame(d);
  IorSample<SP> ext_ior = evaluate_ior<SP>(sc, m.ext_ior, d.wavelength);
  IorSample<SP> int_ior = evaluate_ior<SP>(sc, m.int_ior, d.wavelength);
  ThinfilmEval<SP> thinfilm = evaluate_thinfilm<SP>(sc, d.wavelength, m.thinfilm, d.tex, smp);
  Spec<SP> fr = fresnel_calculate<SP>(d.wavelength, dot(d.w_i, d.nrm), ext_ior, int_ior, thinfilm);
  float f = fr.monochromatic();
  BSample<SP> r = bsample_zero<SP>();
  if (smp.next() <= f) {
    r.w_o = normalize(reflect(d.w_i, frame.nrm));
    r.pdf = f;
    r.weight = apply_image<SP>(sc, m.reflectance, d.tex, d.wavelength);
    r.weight *= fr / f;
    r.properties = kBsdfDelta | kBsdfReflection;
    r.medium_index = d.current_medium;
  } else {
    r.w_o = d.w_i;
    r.pdf = 1.0f - f;
    r.weight = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength);
    r.weight *= (1.0f - fr) / (1.0f - f);
    r.properties = kBsdfDelta | kBsdfTransmission | kBsdfMediumChanged;
    r.medium_index = frame.entering ? m.int_medium : m.ext_medium;
  }
  return r;
}

// ---- Translucent (bsdf_various.hxx:135-215) ---------------------------------------------------------------------
template <bool SP>
DEV BSample<SP> translucent_sample(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  Frame frame = normal_frame(d);
  Spec<SP> tr = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength);
  Spec<SP> rf = apply_image<SP>(sc, m.reflectance, d.tex, d.wavelength);
  float tr_value = tr.monochromatic(), rf_value = rf.monochromatic();
  float total = tr_value + rf_value;
  if (total == 0.0f) return bsample_zero<SP>();
  V3 w_o = sample_cosine_around(smp.next_2d(), frame.nrm, 1.0f);
  float n_dot_o = fabsf(dot(w_o, frame.nrm));
  BSample<SP> r = bsample_zero<SP>();
  if (smp.next() < tr_value / total) {
    r.eta = 1.0f;
    r.w_o = -w_o;
    r.pdf = n_dot_o * kInvPi * (tr_value / total);
    r.properties = kBsdfDiffuse | kBsdfTransmission | kBsdfMediumChanged;
    r.medium_index = frame.entering ? m.int_medium : m.ext_medium;
    r.weight = tr;
  } else {
    r.eta = 1.0f;
    r.w_o = w_o;
    r.pdf = n_dot_o * kInvPi * (rf_value / total);
    r.properties = kBsdfDiffuse | kBsdfReflection;
    r.medium_index = d.current_medium;
    r.weight = rf;
  }
  return r;
}
template <bool SP>
DEV BEval<SP> translucent_evaluate(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m) {
  Frame frame = normal_frame(d);
  float n_dot_i = -dot(frame.nrm, d.w_i);
  float n_dot_o = dot(frame.nrm, w_o);
  bool reflection = n_dot_o * n_dot_i > 0.0f;
  Spec<SP> tr = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength);
  Spec<SP> rf = apply_image<SP>(sc, m.reflectance, d.tex, d.wavelength);
  float tr_value = tr.monochromatic(), rf_value = rf.monochromatic();
  float total = tr_value + rf_value;
  if (total == 0.0f) return beval_zero<SP>();
  float scale = (total > 1.0f) ? 1.0f / total : 1.0f;
  n_dot_o = fabsf(n_dot_o);
  BEval<SP> e;
  e.eta = 1.0f;
  e.func = (reflection ? rf : tr) * (scale * kInvPi);
  e.bsdf = e.func * n_dot_o;
  e.pdf = kInvPi * n_dot_o * (reflection ? rf_value / total : tr_value / total);
  return e;
}
template <bool SP>
DEV float translucent_pdf(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m) {
  Frame frame = normal_frame(d);
  float n_dot_i = -dot(frame.nrm, d.w_i);
  float n_dot_o = dot(frame.nrm, w_o);
  float tr_value = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength).monochromatic();
  float rf_value = apply_image<SP>(sc, m.reflectance, d.tex, d.wavelength).monochromatic();
  float total = tr_value + rf_value;
  bool reflection = n_dot_o * n_dot_i > 0.0f;
  return (total == 0.0f) ? 0.0f : kInvPi * fabsf(n_dot_o) * (reflection ? rf_value / total : tr_value / total);
}

// ---- Mirror (bsdf_various.hxx:217-262) ----------------------------------------------------------------------------
DEV bool direction_matches(V3 ideal, V3 actual) {  // math.hxx:1087-1091
  const V3 i = normalize(ideal);
  const V3 a = normalize(actual);
  return dot(i, a) > 1.0f - kInvMaxHalf;
}
template <bool SP>
DEV BSample<SP> mirror_sample(const DeviceScene& sc, const BData& d, const etxb_material& m) {
  Frame frame = normal_frame(d);
  BSample<SP> r = bsample_zero<SP>();
  r.w_o = normalize(reflect(d.w_i, frame.nrm));
  r.weight = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength);
  r.pdf = 1.0f;
  r.properties = kBsdfDelta | kBsdfReflection;
  return r;
}
template <bool SP>
DEV BEval<SP> mirror_evaluate(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m) {
  BEval<SP> e = beval_zero<SP>();
  Frame frame = normal_frame(d);
  const V3 ideal_w_o = normalize(reflect(d.w_i, frame.nrm));
  const V3 actual_w_o = normalize(w_o);
  if (direction_matches(ideal_w_o, actual_w_o)) {
    e.func = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength);
    e.bsdf = e.func;
    e.pdf = 1.0f;
  }
  return e;
}
DEV float mirror_pdf(const BData& d, V3 w_o) {
  Frame frame = normal_frame(d);
  const V3 ideal_w_o = normalize(reflect(d.w_i, frame.nrm));
  const V3 actual_w_o = normalize(w_o);
  return direction_matches(ideal_w_o, actual_w_o) ? 1.0f : 0.0f;
}

// ---- Velvet (bsdf_velvet.hxx) -------------------------------------------------------------------------------------
DEV float lambda_velvet_l(float r, float x) {
  x = fmaxf(x, 0.0f);
  float t0 = sqr(1.0f - r), t1 = (1.0f - sqr(1.0f - r));
  float a = t0 * 25.3245f + t1 * 21.5473f;
  float b = t0 * 3.32435f + t1 * 3.82987f;
  float c = t0 * 0.16801f + t1 * 0.19823f;
  float dd = t0 * -1.27393f + t1 * -1.97760f;
  float e = t0 * -4.85967f + t1 * -4.32054f;
  return a / (1.0f + b * m_pow(x, c)) + dd * x + e;
}
DEV float lambda_velvet(float r, float cos_t) {
  if (cos_t < 0.5f) return m_exp(lambda_velvet_l(r, cos_t));
  return m_exp(2.0f * lambda_velvet_l(r, 0.5f) - lambda_velvet_l(r, 1.0f - cos_t));
}
DEV float fresnel_approximate(float f0, float f90, float cos_t) { return f0 + (f90 - f0) * m_pow(fmaxf(1.0f - cos_t, 0.0f), 5.0f); }
template <bool SP>
DEV BEval<SP> velvet_evaluate(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m) {
  Frame frame = normal_frame(d);
  float n_dot_o = fmaxf(0.0f, dot(w_o, frame.nrm));
  float n_dot_i = fmaxf(0.0f, -dot(d.w_i, frame.nrm));
  if ((n_dot_o <= kEpsilon) || (n_dot_i <= kEpsilon)) return beval_zero<SP>();
  V3 mh = normalize(w_o - d.w_i);
  float m_dot_o = fmaxf(0.0f, dot(w_o, mh));
  float m_dot_i = fmaxf(0.0f, -dot(d.w_i, mh));
  if ((m_dot_o <= kEpsilon) || (m_dot_i <= kEpsilon)) return beval_zero<SP>();
  V2 roughness = evaluate_roughness(sc, m, d.tex);
  float specular_scale_base = 0.0f;
  float alpha = 0.5f * (roughness.x + roughness.y);
  if (alpha > kEpsilon) {
    float inv_alpha = 1.0f / (kEpsilon + alpha);
    float m_dot_n = dot(mh, frame.nrm);
    float sin_t = (1.0f - m_dot_n * m_dot_n);
    float dd = (2.0f + inv_alpha) * m_pow(sin_t, 0.5f * inv_alpha) / kDoublePi;
    float l_i = lambda_velvet(alpha, n_dot_i);
    float l_o = lambda_velvet(alpha, n_dot_o);
    float g = 1.0f / (1.0f + l_i + l_o);
    specular_scale_base = 0.25f * dd * g / n_dot_i;
  }
  Spec<SP> diffuse = apply_image<SP>(sc, m.scattering, d.tex, d.wavelength);
  Spec<SP> specular = apply_image<SP>(sc, m.reflectance, d.tex, d.wavelength);
  // diffuse_burley
  float f90 = 0.5f + 2.0f * alpha * m_dot_o * m_dot_o;
  float lightScatter = fresnel_approximate(1.0f, f90, n_dot_o);
  float viewScatter = fresnel_approximate(1.0f, f90, n_dot_i);
  float diffuse_scale = lightScatter * viewScatter * kInvPi;
  BEval<SP> e;
  e.eta = 1.0f;
  e.func = diffuse * diffuse_scale + specular * specular_scale_base / n_dot_o;
  e.bsdf = diffuse * diffuse_scale * n_dot_o + specular * specular_scale_base;
  e.pdf = 1.0f / kDoublePi;
  return e;
}
template <bool SP>
DEV BSample<SP> velvet_sample(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  Frame frame = normal_frame(d);
  V3 w_o = sample_cosine_around(smp.next_2d(), frame.nrm, 0.0f);
  BEval<SP> eval = velvet_evaluate<SP>(sc, d, w_o, m);
  BSample<SP> r = bsample_zero<SP>();
  r.w_o = w_o;
  r.properties = kBsdfReflection | kBsdfDiffuse;
  r.medium_index = d.current_medium;
  r.eta = 1.0f;
  r.pdf = eval.pdf;
  r.weight = eval.bsdf / eval.pdf;
  return r;
}
DEV float velvet_pdf(const BData& d) {
  Frame frame = normal_frame(d);
  if (frame.entering == false) return 0.0f;
  return 1.0f / kDoublePi;
}

// ---- Principled: stochastic pick of Conductor / Dielectric / Plastic on a modified copy of the material (bsdf_principled.hxx) ----
DEV void principled_as_conductor(const DeviceScene& sc, etxb_material& m) {
  m.int_ior.cls = kSpdClassConductor;
  m.int_ior.eta_index = sc.default_conductor_eta;
  m.int_ior.k_index = sc.default_conductor_k;
  m.scattering.image_index = kInvalidIndex;
}
DEV void principled_as_dielectric(const DeviceScene& sc, etxb_material& m) {
  m.int_ior.cls = 3u;  // SpectralDistribution::Class::Dielectric
  m.int_ior.eta_index = sc.default_dielectric_eta;
  m.int_ior.k_index = kInvalidIndex;
  m.reflectance.image_index = kInvalidIndex;
}
template <bool SP>
DEVN BSample<SP> principled_sample(const DeviceScene& sc, const BData& d, const etxb_material& in_m, Smp& smp) {
  etxb_material m = in_m;
  float metalness = evaluate_metalness(sc, m, d.tex);
  if (smp.next() < metalness) {
    principled_as_conductor(sc, m);
    return conductor_sample<SP>(sc, d, m, smp);
  }
  principled_as_dielectric(sc, m);
  if (smp.next() < m.transmission.value[0]) return dielectric_sample<SP>(sc, d, m, smp);
  return plastic_sample<SP>(sc, d, m, smp);
}
template <bool SP>
DEVN BEval<SP> principled_evaluate(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& in_m, Smp& smp) {
  etxb_material m = in_m;
  float metalness = evaluate_metalness(sc, m, d.tex);
  if (smp.next() < metalness) {
    principled_as_conductor(sc, m);
    return conductor_evaluate<SP>(sc, d, w_o, m, smp);
  }
  principled_as_dielectric(sc, m);
  if (smp.next() < m.transmission.value[0]) return dielectric_evaluate<SP>(sc, d, w_o, m, smp);
  return plastic_evaluate<SP>(sc, d, w_o, m, smp);
}
template <bool SP>
DEVN float principled_pdf(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& in_m, Smp& smp) {
  etxb_material m = in_m;
  float metalness = evaluate_metalness(sc, m, d.tex);
  if (smp.next() < metalness) {
    principled_as_conductor(sc, m);
    return conductor_pdf(sc, d, w_o, m);
  }
  principled_as_dielectric(sc, m);
  if (smp.next() < m.transmission.value[0]) return dielectric_pdf<SP>(sc, d, w_o, m, smp);
  return plastic_pdf<SP>(sc, d, w_o, m, smp);
}

// ---- dispatch (scene_bsdf.hxx:56-90) -----------------------------------------------------------------------
// Classes / variants not implemented on the device are rejected by etxb_upload_scene (ETXB_ERR_UNSUPPORTED).
// The Lambert case is inlined at every call site; all other classes go through ONE out-of-line copy of the switch per kernel
// module (the microfacet random walks are large: inlining them at each of the ~10 call sites of a bounce kernel multiplies code
// size, instruction-cache misses and compile time for no gain).
template <bool SP>
DEVG_BSDF BSample<SP> bsdf_sample_generic(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  switch (m.cls) {
    case ETXB_MAT_DIFFUSE:  // diffuse_variation 1 walks the microsurface, 2 samples the cosine lobe like 0 (which the caller handles inline)
      return (m.diffuse_variation == 1u) ? rough_diffuse_sample<SP>(sc, d, m, smp) : diffuse_sample<SP>(sc, d, m, smp);
    case ETXB_MAT_TRANSLUCENT: return translucent_sample<SP>(sc, d, m, smp);
    case ETXB_MAT_PLASTIC: return plastic_sample<SP>(sc, d, m, smp);
    case ETXB_MAT_CONDUCTOR: return conductor_sample<SP>(sc, d, m, smp);
    case ETXB_MAT_DIELECTRIC: return dielectric_sample<SP>(sc, d, m, smp);
    case ETXB_MAT_THINFILM: return thinfilm_sample<SP>(sc, d, m, smp);
    case ETXB_MAT_MIRROR: return mirror_sample<SP>(sc, d, m);
    case ETXB_MAT_VELVET: return velvet_sample<SP>(sc, d, m, smp);
    case ETXB_MAT_PRINCIPLED: return principled_sample<SP>(sc, d, m, smp);
    case ETXB_MAT_BOUNDARY: {  // BoundaryBSDF::sample (bsdf_various.hxx:266-277)
      BSample<SP> r = bsample_zero<SP>();
      r.w_o = d.w_i;
      r.pdf = 1.0f;
      r.weight = Spec<SP>::make(1.0f);
      r.properties = kBsdfTransmission | kBsdfMediumChanged;
      r.medium_index = (dot(d.nrm, d.w_i) < 0.0f) ? m.int_medium : m.ext_medium;
      return r;
    }
    default: {  // VoidBSDF::sample (bsdf_various.hxx:5-15)
      BSample<SP> r = bsample_zero<SP>();
      r.w_o = d.w_i;
      r.properties = kBsdfDelta;
      r.medium_index = d.current_medium;
      return r;
    }
  }
}
template <bool SP>
DEV BSample<SP> bsdf_sample(const DeviceScene& sc, const BData& d, const etxb_material& m, Smp& smp) {
  if ((m.cls == ETXB_MAT_DIFFUSE) && (m.diffuse_variation == 0u)) return diffuse_sample<SP>(sc, d, m, smp);
  return bsdf_sample_generic<SP>(sc, d, m, smp);
}
template <bool SP>
DEVG_BSDF BEval<SP> bsdf_evaluate_generic(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m, Smp& smp) {
  switch (m.cls) {
    case ETXB_MAT_DIFFUSE: return diffuse_evaluate<SP>(sc, d, w_o, m, smp);
    case ETXB_MAT_TRANSLUCENT: return translucent_evaluate<SP>(sc, d, w_o, m);
    case ETXB_MAT_PLASTIC: return plastic_evaluate<SP>(sc, d, w_o, m, smp);
    case ETXB_MAT_CONDUCTOR: return conductor_evaluate<SP>(sc, d, w_o, m, smp);
    case ETXB_MAT_DIELECTRIC: return dielectric_evaluate<SP>(sc, d, w_o, m, smp);
    case ETXB_MAT_MIRROR: return mirror_evaluate<SP>(sc, d, w_o, m);
    case ETXB_MAT_VELVET: return velvet_evaluate<SP>(sc, d, w_o, m);
    case ETXB_MAT_PRINCIPLED: return principled_evaluate<SP>(sc, d, w_o, m, smp);
    default: return beval_zero<SP>();  // Thinfilm, Boundary, Void evaluate to zero
  }
}
template <bool SP>
DEV BEval<SP> bsdf_evaluate(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m, Smp& smp) {
  if ((m.cls == ETXB_MAT_DIFFUSE) && (m.diffuse_variation == 0u)) return diffuse_evaluate<SP>(sc, d, w_o, m, smp);
  return bsdf_evaluate_generic<SP>(sc, d, w_o, m, smp);
}
template <bool SP>
DEVG_BSDF float bsdf_pdf_generic(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m, Smp& smp) {
  switch (m.cls) {
    case ETXB_MAT_DIFFUSE: return diffuse_pdf(d, w_o);
    case ETXB_MAT_TRANSLUCENT: return translucent_pdf<SP>(sc, d, w_o, m);
    case ETXB_MAT_PLASTIC: return plastic_pdf<SP>(sc, d, w_o, m, smp);
    case ETXB_MAT_CONDUCTOR: return conductor_pdf(sc, d, w_o, m);
    case ETXB_MAT_DIELECTRIC: return dielectric_pdf<SP>(sc, d, w_o, m, smp);
    case ETXB_MAT_MIRROR: return mirror_pdf(d, w_o);
    case ETXB_MAT_VELVET: return velvet_pdf(d);
    case ETXB_MAT_PRINCIPLED: return principled_pdf<SP>(sc, d, w_o, m, smp);
    default: return 0.0f;
  }
}
template <bool SP>
DEV float bsdf_pdf(const DeviceScene& sc, const BData& d, V3 w_o, const etxb_material& m, Smp& smp) {
  if (m.cls == ETXB_MAT_DIFFUSE) return diffuse_pdf(d, w_o);
  return bsdf_pdf_generic<SP>(sc, d, w_o, m, smp);
}
template <bool SP>
DEV float bsdf_reverse_pdf(const DeviceScene& sc, const BData& in_d, V3 in_w_o, const etxb_material& m, Smp& smp) {
  V3 w_o = -in_d.w_i;
  BData d = in_d;
  d.w_i = -in_w_o;
  return bsdf_pdf<SP>(sc, d, w_o, m, smp);
}

}  // namespace etxb
