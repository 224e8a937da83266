// kernels_view.cuh — the viewer's output views and the film's error against a reference image (included once, by module.cu, after
// kernels_denoise.cuh).  DESIGN §14.
//
//   k_film_tonemap       the LDR export's frame (app.cxx:268-282): the tone curve below, 8 bits by truncation, alpha 255
//   k_film_view          the viewer's fragment shader (render.cxx:252-388) per pixel: one of six OutputViews, float4 or the window's RGBA8
//   k_film_error_blocks  first pass of the error reduction: one float64 record per block of kErrorChunk pixels
//   k_film_error_final   second pass: one block folds the block records in a fixed order
//
// The layer and the reference are read at the same storage index, as the shader's Load(coord) reads both textures at one coordinate.
#pragma once

namespace etxb {

// The tone curve of the export and of the view: one definition, so etxb_read_film_ldr keeps its bytes.  CUDA's expf / powf in both builds.
// The shader's pow(abs(v), ...) drops its abs here: the branch is only taken for v > 0.0031308 (or NaN, which stays NaN).
DEV float tone_curve(float v, float exposure) { return 1.0f - expf(-exposure * v); }
DEV float linear_to_gamma(float v) { return (v <= 0.0031308f) ? (12.92f * v) : (1.055f * powf(v, 1.0f / 2.4f) - 0.055f); }

__global__ void __launch_bounds__(256) k_film_tonemap(const float4* layer, uint32_t* out_rgba8, uint32_t count, float exposure) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float4 v = layer[i];
  float c[3] = {v.x, v.y, v.z};
  uint32_t packed = 0xff000000u;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    float g = linear_to_gamma(tone_curve(c[k], exposure));
    g = (g > 0.0f) ? fminf(g, 1.0f) : 0.0f;
    packed |= uint32_t(255.0f * g) << (8 * k);
  }
  out_rgba8[i] = packed;
}

// OutputView (raytracer/options.hxx:9-18) and ViewOptions (:40-45)
constexpr uint32_t kViewResult = 0u, kViewAlpha = 1u, kViewOriginal = 2u, kViewReference = 3u, kViewRelative = 4u, kViewAbsolute = 5u;
constexpr uint32_t kViewToneMapping = 1u, kViewSRGB = 2u, kViewSkipColorConversion = 4u;
constexpr float kViewThreshold = 1.0f / 8192.0f;

// dot(v.xyz, (0.2627, 0.6780, 0.0593)) in float32, left to right, never contracted: the same value in both builds
DEV float view_lum(float4 v) { return __fadd_rn(__fadd_rn(__fmul_rn(v.x, 0.2627f), __fmul_rn(v.y, 0.6780f)), __fmul_rn(v.z, 0.0593f)); }

DEV float4 view_tonemap(float4 v, uint32_t options, float exposure) {
  if (options & kViewToneMapping) v = make_float4(tone_curve(v.x, exposure), tone_curve(v.y, exposure), tone_curve(v.z, exposure), tone_curve(v.w, exposure));
  if (options & kViewSRGB) v = make_float4(linear_to_gamma(v.x), linear_to_gamma(v.y), linear_to_gamma(v.z), v.w);
  return v;
}

DEV bool any_nan(float4 v) { return isnan(v.x) || isnan(v.y) || isnan(v.z) || isnan(v.w); }
DEV bool any_inf(float4 v) { return isinf(v.x) || isinf(v.y) || isinf(v.z) || isinf(v.w); }

// fragment_main (render.cxx:332-386) at one pixel; `ref` is read only by the views that use it
DEV float4 film_view_pixel(const float4* layer, const float4* ref, uint32_t i, uint32_t view, uint32_t options, float exposure) {
  const float4 c = layer[i];
  if (view == kViewAlpha) return make_float4(exposure * c.w, exposure * c.w, exposure * c.w, exposure * c.w);
  if (options & kViewSkipColorConversion) return make_float4(exposure * c.x, exposure * c.y, exposure * c.z, exposure * c.w);
  // validate(): the markers, else max(0, c) returned as it is (not tone-mapped) wherever it differs from c
  if (any_nan(c)) return make_float4(123456.0f, 0.0f, 123456.0f, 1.0f);
  if (any_inf(c)) return make_float4(0.0f, 123456.0f, 123456.0f, 1.0f);
  if ((c.x < 0.0f) || (c.y < 0.0f) || (c.z < 0.0f) || (c.w < 0.0f))
    return make_float4(fmaxf(0.0f, c.x), fmaxf(0.0f, c.y), fmaxf(0.0f, c.z), fmaxf(0.0f, c.w));
  switch (view) {
    case kViewResult:
      return view_tonemap(c, options, exposure);
    case kViewOriginal:
      return make_float4(exposure * c.x, exposure * c.y, exposure * c.z, exposure * c.w);
    case kViewReference:
      return view_tonemap(ref[i], options, exposure);
    default: {
      const float r_lum = view_lum(ref[i]), c_lum = view_lum(c);
      const float above = fmaxf(0.0f, r_lum - c_lum), below = fmaxf(0.0f, c_lum - r_lum);
      if (view == kViewRelative) return make_float4(exposure * above, exposure * below, 0.0f, 0.0f);
      return make_float4((above > kViewThreshold) ? 1.0f : 0.0f, (below > kViewThreshold) ? 1.0f : 0.0f, 0.0f, 0.0f);
    }
  }
}

// what an 8-bit UNORM render target stores: clamp to [0, 1] (NaN -> 0), floor(255 x + 0.5), never contracted
DEV uint32_t unorm8(float x) { return uint32_t(floorf(__fadd_rn(__fmul_rn(fminf(fmaxf(x, 0.0f), 1.0f), 255.0f), 0.5f))); }

// out_f or out_rgba8 (the other is null)
__global__ void __launch_bounds__(256) k_film_view(const float4* layer, const float4* ref, uint32_t count, uint32_t view, uint32_t options, float exposure,
                                                   float4* out_f, uint32_t* out_rgba8) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float4 v = film_view_pixel(layer, ref, i, view, options, exposure);
  if (out_f) out_f[i] = v;
  else out_rgba8[i] = unorm8(v.x) | (unorm8(v.y) << 8u) | (unorm8(v.z) << 16u) | (unorm8(v.w) << 24u);
}

// ---- the error reduction ----------------------------------------------------------------------------------------------------------------
// Block b of kErrorThreads threads takes pixels [b kErrorChunk, (b + 1) kErrorChunk); thread t adds pixels b kErrorChunk + t + k kErrorThreads in
// order of k; the block folds its threads by halving; the final block folds the block records t, t + kErrorThreads, ... per thread, then by
// halving.  Every step depends on the pixel count alone, so the result is a function of the two images.
constexpr uint32_t kErrorThreads = 256u, kErrorChunk = 16u * kErrorThreads;

struct ErrorSums {
  double se, rel, abs_lum, lum, ref_lum;                        // mean_rgb: `se` holds the reference's r + g + b
  unsigned long long finite, nonfinite, negative, above, below;
};

DEV void error_add(ErrorSums& a, const ErrorSums& b) {
  a.se += b.se, a.rel += b.rel, a.abs_lum += b.abs_lum, a.lum += b.lum, a.ref_lum += b.ref_lum;
  a.finite += b.finite, a.nonfinite += b.nonfinite, a.negative += b.negative, a.above += b.above, a.below += b.below;
}

DEV double lum64(float4 v) { return double(v.x) * 0.2627 + double(v.y) * 0.6780 + double(v.z) * 0.0593; }

// MeanOnly: the reference's mean over every pixel and channel (the ε of rel_mse), taken once when the reference is set
template <bool MeanOnly>
DEV void error_pixel(ErrorSums& s, const float4* layer, const float4* ref, uint32_t i, double eps) {
  const float4 r = ref[i];
  if (MeanOnly) {
    s.se += double(r.x) + double(r.y) + double(r.z);
    return;
  }
  const float4 c = layer[i];
  if (!isfinite(c.x) || !isfinite(c.y) || !isfinite(c.z)) {
    s.nonfinite += 1u;
    return;
  }
  s.finite += 1u;
  s.negative += ((c.x < 0.0f) || (c.y < 0.0f) || (c.z < 0.0f)) ? 1u : 0u;
  const float cv[3] = {c.x, c.y, c.z}, rv[3] = {r.x, r.y, r.z};
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double d = double(cv[k]) - double(rv[k]), d2 = d * d;
    s.se += d2;
    s.rel += d2 / (double(rv[k]) * double(rv[k]) + eps);
  }
  const float r_lum = view_lum(r), c_lum = view_lum(c);
  s.above += (fmaxf(0.0f, r_lum - c_lum) > kViewThreshold) ? 1u : 0u;
  s.below += (fmaxf(0.0f, c_lum - r_lum) > kViewThreshold) ? 1u : 0u;
  const double cl = lum64(c), rl = lum64(r);
  s.abs_lum += fabs(cl - rl);
  s.lum += cl;
  s.ref_lum += rl;
}

DEV void error_fold(ErrorSums* sh, ErrorSums s) {
  const uint32_t t = threadIdx.x;
  sh[t] = s;
  __syncthreads();
  for (uint32_t h = kErrorThreads / 2u; h > 0u; h >>= 1u) {
    if (t < h) error_add(sh[t], sh[t + h]);
    __syncthreads();
  }
}

template <bool MeanOnly>
__global__ void __launch_bounds__(kErrorThreads) k_film_error_blocks(const float4* layer, const float4* ref, uint32_t count, double eps, ErrorSums* blocks) {
  __shared__ ErrorSums sh[kErrorThreads];
  ErrorSums s = {};
  const uint32_t begin = blockIdx.x * kErrorChunk, end = umin(count, begin + kErrorChunk);
  for (uint32_t i = begin + threadIdx.x; i < end; i += kErrorThreads) error_pixel<MeanOnly>(s, layer, ref, i, eps);
  error_fold(sh, s);
  if (threadIdx.x == 0u) blocks[blockIdx.x] = sh[0];
}

__global__ void __launch_bounds__(kErrorThreads) k_film_error_final(const ErrorSums* blocks, uint32_t block_count, ErrorSums* out) {
  __shared__ ErrorSums sh[kErrorThreads];
  ErrorSums s = {};
  for (uint32_t b = threadIdx.x; b < block_count; b += kErrorThreads) error_add(s, blocks[b]);
  error_fold(sh, s);
  if (threadIdx.x == 0u) *out = sh[0];
}

}  // namespace etxb
