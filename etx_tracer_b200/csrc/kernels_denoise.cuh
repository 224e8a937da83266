// kernels_denoise.cuh — Film::denoise on the device (included once, by module.cu, after kernels_pt.cuh).  DESIGN §13.
//
// The reference hands three film layers to OpenImageDenoise (film.cxx:420-423), a trained network whose weights this project does not have.
// In its place: non-local means on the colour with a dual-buffer variance estimate (Rousselle, Knaus, Zwicker 2012), combined with feature
// weights on the normal and albedo guides by the minimum of the weights (Rousselle, Manzi, Zwicker 2013); one fixed filter, no selection.
// tests/denoise_model.py is the float64 statement of the same filter, constants included.
//
//   k_denoise_variance  per pixel: the variance of the running mean from the two half buffers, the colour with non-finite pixels zeroed
//   k_denoise_smooth    3 x 3 box of the variance, clamped at the film edge
//   k_denoise_nlm       one 16 x 16 tile of output pixels per block, the colour and variance of its (16 + 2 (r + f))^2 halo in shared memory;
//                       per window offset: the per-pixel distance term over the tile + f, a separable (2f + 1)^2 box sum, the weight, the sums
//
// Every buffer is in the film's storage order (y-flipped rows): the filter is symmetric under a mirror, so the order does not change it.
#pragma once

namespace etxb {

constexpr int kDenoiseR = 10;        // window radius r
constexpr int kDenoiseF = 3;         // patch radius f
constexpr float kDenoiseKc = 0.45f;  // colour: k_c
constexpr float kDenoiseAlpha = 1.0f;
constexpr float kDenoiseEps = 1e-10f;
constexpr float kDenoiseKf = 0.6f;   // features: k_f
constexpr float kDenoiseTau = 1e-3f;
constexpr int kDenoiseTile = 16;
constexpr int kDenoiseHalo = kDenoiseR + kDenoiseF;
constexpr int kDenoiseExt = kDenoiseTile + 2 * kDenoiseHalo;  // halo side: colour and variance of these pixels sit in shared memory
constexpr int kDenoisePatch = kDenoiseTile + 2 * kDenoiseF;   // side of the per-offset distance term

struct DenoiseInputs {
  const float4* color;      // the layer to filter (Result or Camera)
  const float4* camera;     // F: the camera layer, running mean of n samples
  const float4* half;       // H: CameraAdaptive, the mean of the even-indexed samples
  const uint32_t* counts;   // per-pixel sample count (path tracer's InternalData, bits 0-29), or null: `count` everywhere
  uint32_t count;
  const float4* normals;    // guides, or null (no feature weight)
  const float4* albedo;
  uint32_t width, height;
};

DEV bool finite3(float4 v) { return isfinite(v.x) && isfinite(v.y) && isfinite(v.z); }
DEV float4 finite_or_zero(float4 v) { return make_float4(isfinite(v.x) ? v.x : 0.0f, isfinite(v.y) ? v.y : 0.0f, isfinite(v.z) ? v.z : 0.0f, 0.0f); }
DEV float denoise_exp(float x) {
#if defined(ETXB_PARITY) && ETXB_PARITY
  return expf(x);
#else
  return __expf(x);
#endif
}

// Var(F) = (H - O)^2 h (n - h) / n^2 with h = ceil(n / 2) and O = (n F - h H) / (n - h), the mean of the odd-indexed samples.  `u` is the colour
// with .w = 1 where the pixel takes part (colour and variance finite) and 0 where it is copied through; *not_ready is set where n < 2.
__global__ void __launch_bounds__(256) k_denoise_variance(const __grid_constant__ DenoiseInputs in, float4* u, float4* var, uint32_t* not_ready) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= in.width * in.height) return;
  const uint32_t n = in.counts ? (in.counts[i] & 0x3fffffffu) : in.count;
  if (n < 2u) {
    *not_ready = 1u;
    return;
  }
  const uint32_t h = (n + 1u) / 2u;
  const float fn = float(n), fh = float(h), fm = float(n - h), scale = fh * fm / (fn * fn);
  const float4 F = in.camera[i], H = in.half[i], c = in.color[i];
  const float ox = (fn * F.x - fh * H.x) / fm, oy = (fn * F.y - fh * H.y) / fm, oz = (fn * F.z - fh * H.z) / fm;
  const float4 v = make_float4((H.x - ox) * (H.x - ox) * scale, (H.y - oy) * (H.y - oy) * scale, (H.z - oz) * (H.z - oz) * scale, 0.0f);
  const bool ok = finite3(c) && finite3(v);
  u[i] = ok ? make_float4(c.x, c.y, c.z, 1.0f) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  var[i] = ok ? v : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}

__global__ void __launch_bounds__(256) k_denoise_smooth(const float4* var, float4* out, uint32_t width, uint32_t height) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= width * height) return;
  const int x = int(i % width), y = int(i / width);
  float sx = 0.0f, sy = 0.0f, sz = 0.0f;
  for (int dy = -1; dy <= 1; ++dy) {
    const int yy = min(max(y + dy, 0), int(height) - 1);
    for (int dx = -1; dx <= 1; ++dx) {
      const float4 v = var[min(max(x + dx, 0), int(width) - 1) + yy * int(width)];
      sx += v.x;
      sy += v.y;
      sz += v.z;
    }
  }
  out[i] = make_float4(sx / 9.0f, sy / 9.0f, sz / 9.0f, 0.0f);
}

// 1 / (k_f^2 max(tau, |grad g(p)|^2)) with central differences clamped at the film edge; 0 without the guide (its weight is then 1)
DEV float guide_inv_scale(const float4* g, int x, int y, int w, int h) {
  if (!g) return 0.0f;
  const float4 l = finite_or_zero(g[max(x - 1, 0) + y * w]), r = finite_or_zero(g[min(x + 1, w - 1) + y * w]);
  const float4 d = finite_or_zero(g[x + max(y - 1, 0) * w]), u = finite_or_zero(g[x + min(y + 1, h - 1) * w]);
  const float gx0 = 0.5f * (r.x - l.x), gx1 = 0.5f * (r.y - l.y), gx2 = 0.5f * (r.z - l.z);
  const float gy0 = 0.5f * (u.x - d.x), gy1 = 0.5f * (u.y - d.y), gy2 = 0.5f * (u.z - d.z);
  const float g2 = gx0 * gx0 + gx1 * gx1 + gx2 * gx2 + gy0 * gy0 + gy1 * gy1 + gy2 * gy2;
  return 1.0f / (kDenoiseKf * kDenoiseKf * fmaxf(kDenoiseTau, g2));
}
DEV float guide_distance(const float4* g, float4 gp, uint32_t q) {
  const float4 gq = finite_or_zero(g[q]);
  const float a = gp.x - gq.x, b = gp.y - gq.y, c = gp.z - gq.z;
  return a * a + b * b + c * c;
}

__global__ void __launch_bounds__(kDenoiseTile * kDenoiseTile) k_denoise_nlm(const __grid_constant__ DenoiseInputs in, const float4* u, const float4* var, float4* out) {
  __shared__ float s_u[3][kDenoiseExt * kDenoiseExt];
  __shared__ float s_v[3][kDenoiseExt * kDenoiseExt];
  __shared__ uint8_t s_ok[kDenoiseExt * kDenoiseExt];
  __shared__ float s_d[kDenoisePatch * kDenoisePatch];   // distance term at the tile's pixels + f, for the current offset
  __shared__ float s_row[kDenoisePatch * kDenoiseTile];  // its sums along x
  const int w = int(in.width), h = int(in.height);
  const int ox = int(blockIdx.x) * kDenoiseTile, oy = int(blockIdx.y) * kDenoiseTile;
  const int tid = int(threadIdx.x), tx = tid % kDenoiseTile, ty = tid / kDenoiseTile;
  constexpr int kThreads = kDenoiseTile * kDenoiseTile;
  for (int k = tid; k < kDenoiseExt * kDenoiseExt; k += kThreads) {
    const int gx = min(max(ox - kDenoiseHalo + k % kDenoiseExt, 0), w - 1), gy = min(max(oy - kDenoiseHalo + k / kDenoiseExt, 0), h - 1);
    const float4 c = u[gx + gy * w], v = var[gx + gy * w];
    s_u[0][k] = c.x;
    s_u[1][k] = c.y;
    s_u[2][k] = c.z;
    s_v[0][k] = v.x;
    s_v[1][k] = v.y;
    s_v[2][k] = v.z;
    s_ok[k] = (c.w != 0.0f) ? 1u : 0u;
  }
  const int px = ox + tx, py = oy + ty;
  const bool inside = (px < w) && (py < h);
  const int cx = min(px, w - 1), cy = min(py, h - 1);
  const uint32_t pi = uint32_t(cx + cy * w);
  float inv_n = 0.0f, inv_a = 0.0f;
  float4 gn = {}, ga = {};
  if (in.normals) {
    inv_n = guide_inv_scale(in.normals, cx, cy, w, h);
    gn = finite_or_zero(in.normals[pi]);
  }
  if (in.albedo) {
    inv_a = guide_inv_scale(in.albedo, cx, cy, w, h);
    ga = finite_or_zero(in.albedo[pi]);
  }
  __syncthreads();
  constexpr float kColorScale = kDenoiseKc * kDenoiseKc;
  constexpr float kMeanScale = 1.0f / float(3 * (2 * kDenoiseF + 1) * (2 * kDenoiseF + 1));
  float sw = 0.0f, s0 = 0.0f, s1 = 0.0f, s2 = 0.0f;
  for (int dy = -kDenoiseR; dy <= kDenoiseR; ++dy) {
    for (int dx = -kDenoiseR; dx <= kDenoiseR; ++dx) {
      // the distance term at s = (tile pixel + o), against s + (dx, dy); both read at their clamped film positions (the halo was loaded clamped)
      for (int k = tid; k < kDenoisePatch * kDenoisePatch; k += kThreads) {
        const int a = (k / kDenoisePatch + kDenoiseR) * kDenoiseExt + (k % kDenoisePatch + kDenoiseR), b = a + dy * kDenoiseExt + dx;
        float d = 0.0f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float va = s_v[c][a], vb = s_v[c][b], e = s_u[c][a] - s_u[c][b];
          d += (e * e - kDenoiseAlpha * (va + fminf(va, vb))) / (kDenoiseEps + kColorScale * (va + vb));
        }
        s_d[k] = d;
      }
      __syncthreads();
      for (int k = tid; k < kDenoisePatch * kDenoiseTile; k += kThreads) {
        const int r = k / kDenoiseTile, c = k % kDenoiseTile;
        float s = 0.0f;
#pragma unroll
        for (int j = 0; j < 2 * kDenoiseF + 1; ++j) s += s_d[r * kDenoisePatch + c + j];
        s_row[k] = s;
      }
      __syncthreads();
      const int qx = px + dx, qy = py + dy;
      const int qk = (ty + kDenoiseHalo + dy) * kDenoiseExt + (tx + kDenoiseHalo + dx);
      if (inside && (qx >= 0) && (qx < w) && (qy >= 0) && (qy < h) && s_ok[qk]) {
        float dc = 0.0f;
#pragma unroll
        for (int j = 0; j < 2 * kDenoiseF + 1; ++j) dc += s_row[(ty + j) * kDenoiseTile + tx];
        float d = fmaxf(0.0f, dc * kMeanScale);
        const uint32_t q = uint32_t(qx + qy * w);
        if (in.normals) d = fmaxf(d, guide_distance(in.normals, gn, q) * inv_n);
        if (in.albedo) d = fmaxf(d, guide_distance(in.albedo, ga, q) * inv_a);
        const float wq = denoise_exp(-d);  // min over the three weights = exp(-max of the three distances)
        sw += wq;
        s0 += wq * s_u[0][qk];
        s1 += wq * s_u[1][qk];
        s2 += wq * s_u[2][qk];
      }
      __syncthreads();
    }
  }
  if (!inside) return;
  const int pk = (ty + kDenoiseHalo) * kDenoiseExt + (tx + kDenoiseHalo);
  if (!s_ok[pk]) {
    out[pi] = in.color[pi];  // non-finite colour or variance: copied through
    return;
  }
  out[pi] = make_float4(s0 / sw, s1 / sw, s2 / sw, 1.0f);
}

// CameraAdaptive under the VCM (film.cxx:173-230, the every-other-sample mean the reference keeps for every integrator): launched after the
// camera pass on iterations whose sample index is even — the odd ones leave the layer as it is.  Film pixel i reads its block's path as
// k_film_fill_blocks does (at pixel size 1 the path of pixel i is its own).
__global__ void __launch_bounds__(256) k_film_adaptive_vcm(const __grid_constant__ LaunchParams p, float4* adaptive) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const FilmBuffers& film = p.film;
  if (i >= film.width * film.height) return;
  const uint32_t px = i % film.width, py = film.height - 1u - i / film.width;
  const uint32_t path = (px / film.pixel_size) + (py / film.pixel_size) * film.dims_x;
  if (!pixel_owned(p, path)) return;
  const float4 cv = p.camera_value[path];
  V3 v = {cv.x, cv.y, cv.z};
  if (p.camera_sample_index != 0u) {
    const double ds = double(p.camera_sample_index);
    const float t = float(ds / (ds + 2.0));
    const float4 v_old = adaptive[i];
    v = {lerpf(v.x, v_old.x, t), lerpf(v.y, v_old.y, t), lerpf(v.z, v_old.z, t)};
  }
  adaptive[i] = make_float4(v.x, v.y, v.z, 1.0f);
}

}  // namespace etxb
