// portable_math.h — deterministic float transcendentals shared by host and device.
//
// Why this exists: parity between the CUDA path and the CPU oracle is bit-exact only if every
// float operation is the same on both sides.  +,-,*,/ and sqrt are IEEE-754 on x86-64 (SSE) and
// on sm_90a as long as FMA contraction is off (gcc -ffp-contract=off, nvcc -fmad=false), but libm
// (glibc) and CUDA's math library round sinf/cosf/powf/... differently.  The functions below are
// computed in double precision from +,-,*,/ and bit casts only, so the *same source* gives the *same
// bits* under g++ and nvcc.  They are used
//   * by the parity build of the CUDA module (-DETXB_PARITY=1): the device code calls pm_*;
//   * by the oracle (oracle/libm_override.cxx), which re-exports them under the libm names so the
//     reference's headers (which call sinf/powf/... ) bind to them.
// The product ("fast") build does not use this file's transcendentals: it calls CUDA's own.
//
// Accuracy: every function is accurate to well below 1 float ulp (double intermediate, then one
// rounding), special cases follow C99 Annex F for the cases that can occur on the path.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PM_FN __host__ __device__ __forceinline__
#else
#define PM_FN inline
#endif

namespace pm {

PM_FN double bits_to_double(uint64_t u) {
  union { uint64_t u; double d; } c;
  c.u = u;
  return c.d;
}
PM_FN uint64_t double_to_bits(double d) {
  union { uint64_t u; double d; } c;
  c.d = d;
  return c.u;
}
PM_FN float bits_to_float(uint32_t u) {
  union { uint32_t u; float f; } c;
  c.u = u;
  return c.f;
}
PM_FN uint32_t float_to_bits(float f) {
  union { uint32_t u; float f; } c;
  c.f = f;
  return c.u;
}

PM_FN bool is_nan(double x) { return x != x; }
PM_FN bool is_nanf(float x) { return x != x; }
PM_FN double inf_d() { return bits_to_double(0x7ff0000000000000ull); }
PM_FN double nan_d() { return bits_to_double(0x7ff8000000000000ull); }
PM_FN double abs_d(double x) { return bits_to_double(double_to_bits(x) & 0x7fffffffffffffffull); }
PM_FN bool sign_d(double x) { return (double_to_bits(x) >> 63) != 0; }
PM_FN bool is_inf(double x) { return abs_d(x) == inf_d(); }

// The coarse preview's pixel offset inside an s x s block for path `index` of `iteration` (include/etx_b200.h, etxb_set_film_pixel_size): the
// reference draws it from rand(); here x is the first 32-bit value of a hash of (index, iteration) and y the second, each % s, so that an
// iteration stays a function of its index.  Shared like the transcendentals: the device and the oracle call this one definition.  The
// mixer is Wellons' "lowbias32".
PM_FN uint32_t preview_hash(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}
PM_FN void preview_offset(uint32_t index, uint32_t iteration, uint32_t size, uint32_t& dx, uint32_t& dy) {
  const uint32_t first = preview_hash(index ^ preview_hash(iteration ^ 0x9e3779b9u));
  const uint32_t second = preview_hash(first ^ 0x85ebca6bu);
  dx = first % size;
  dy = second % size;
}

// 2^k for k in [-1022, 1023]
PM_FN double pow2i(int k) { return bits_to_double(uint64_t(k + 1023) << 52); }

// ---- exp -------------------------------------------------------------------------------------------
PM_FN double exp_d(double x) {
  if (is_nan(x)) return x;
  if (x > 709.0) return inf_d();
  if (x < -745.0) return 0.0;
  const double kInvLn2 = 1.4426950408889634074;
  const double kLn2Hi = 6.93147180369123816490e-01;
  const double kLn2Lo = 1.90821492927058770002e-10;
  double kf = x * kInvLn2;
  int k = int(kf + (kf >= 0.0 ? 0.5 : -0.5));
  double r = (x - double(k) * kLn2Hi) - double(k) * kLn2Lo;
  // Taylor to r^13, |r| <= 0.3466
  double p = 1.0 / 6227020800.0;
  p = p * r + 1.0 / 479001600.0;
  p = p * r + 1.0 / 39916800.0;
  p = p * r + 1.0 / 3628800.0;
  p = p * r + 1.0 / 362880.0;
  p = p * r + 1.0 / 40320.0;
  p = p * r + 1.0 / 5040.0;
  p = p * r + 1.0 / 720.0;
  p = p * r + 1.0 / 120.0;
  p = p * r + 1.0 / 24.0;
  p = p * r + 1.0 / 6.0;
  p = p * r + 0.5;
  p = p * r + 1.0;
  p = p * r + 1.0;
  // scale by 2^k in two steps so that k may leave the normal exponent range
  int k1 = k / 2;
  int k2 = k - k1;
  return (p * pow2i(k1)) * pow2i(k2);
}

// ---- log -------------------------------------------------------------------------------------------
PM_FN double log_d(double x) {
  if (is_nan(x)) return x;
  if (x < 0.0) return nan_d();
  if (x == 0.0) return -inf_d();
  if (is_inf(x)) return x;
  uint64_t b = double_to_bits(x);
  int e = int(b >> 52);
  if (e == 0) {  // subnormal: renormalise
    x = x * 18014398509481984.0;  // 2^54
    b = double_to_bits(x);
    e = int(b >> 52) - 54;
  }
  e -= 1023;
  double m = bits_to_double((b & 0x000fffffffffffffull) | 0x3ff0000000000000ull);  // [1,2)
  if (m > 1.4142135623730951) {
    m = m * 0.5;
    e += 1;
  }
  double f = (m - 1.0) / (m + 1.0);
  double f2 = f * f;
  double s = 1.0 / 25.0;
  s = s * f2 + 1.0 / 23.0;
  s = s * f2 + 1.0 / 21.0;
  s = s * f2 + 1.0 / 19.0;
  s = s * f2 + 1.0 / 17.0;
  s = s * f2 + 1.0 / 15.0;
  s = s * f2 + 1.0 / 13.0;
  s = s * f2 + 1.0 / 11.0;
  s = s * f2 + 1.0 / 9.0;
  s = s * f2 + 1.0 / 7.0;
  s = s * f2 + 1.0 / 5.0;
  s = s * f2 + 1.0 / 3.0;
  s = s * f2 + 1.0;
  const double kLn2Hi = 6.93147180369123816490e-01;
  const double kLn2Lo = 1.90821492927058770002e-10;
  double de = double(e);
  return de * kLn2Hi + (de * kLn2Lo + 2.0 * f * s);
}

// ---- sin / cos -------------------------------------------------------------------------------------
PM_FN void sincos_reduce(double x, double& r, int& q) {
  const double kTwoOverPi = 0.63661977236758134308;
  const double kPio2Hi = 1.57079632673412561417e+00;
  const double kPio2Lo = 6.07710050650619224932e-11;
  const double kPio2Lo2 = 2.02226624879595063154e-21;
  double kf = x * kTwoOverPi;
  double kr = kf + (kf >= 0.0 ? 0.5 : -0.5);
  // |x| is a float-range angle; beyond 2^31 quadrants precision is gone anyway
  if (kr > 2147483000.0) kr = 2147483000.0;
  if (kr < -2147483000.0) kr = -2147483000.0;
  int k = int(kr);
  double dk = double(k);
  r = ((x - dk * kPio2Hi) - dk * kPio2Lo) - dk * kPio2Lo2;
  q = k & 3;
}
PM_FN double sin_poly(double r) {
  double r2 = r * r;
  double p = -1.0 / 355687428096000.0;  // 17!
  p = p * r2 + 1.0 / 1307674368000.0;   // 15!
  p = p * r2 - 1.0 / 6227020800.0;      // 13!
  p = p * r2 + 1.0 / 39916800.0;        // 11!
  p = p * r2 - 1.0 / 362880.0;          // 9!
  p = p * r2 + 1.0 / 5040.0;            // 7!
  p = p * r2 - 1.0 / 120.0;             // 5!
  p = p * r2 + 1.0 / 6.0;               // -(3!) sign folded below
  return r - r * r2 * p;
}
PM_FN double cos_poly(double r) {
  double r2 = r * r;
  double p = 1.0 / 6402373705728000.0;  // 18!
  p = p * r2 - 1.0 / 20922789888000.0;  // 16!
  p = p * r2 + 1.0 / 87178291200.0;     // 14!
  p = p * r2 - 1.0 / 479001600.0;       // 12!
  p = p * r2 + 1.0 / 3628800.0;         // 10!
  p = p * r2 - 1.0 / 40320.0;           // 8!
  p = p * r2 + 1.0 / 720.0;             // 6!
  p = p * r2 - 1.0 / 24.0;              // 4!
  p = p * r2 + 0.5;
  return 1.0 - r2 * p;
}
PM_FN double sin_d(double x) {
  if (is_nan(x) || is_inf(x)) return nan_d();
  double r;
  int q;
  sincos_reduce(x, r, q);
  switch (q) {
    case 0: return sin_poly(r);
    case 1: return cos_poly(r);
    case 2: return -sin_poly(r);
    default: return -cos_poly(r);
  }
}
PM_FN double cos_d(double x) {
  if (is_nan(x) || is_inf(x)) return nan_d();
  double r;
  int q;
  sincos_reduce(x, r, q);
  switch (q) {
    case 0: return cos_poly(r);
    case 1: return -sin_poly(r);
    case 2: return -cos_poly(r);
    default: return sin_poly(r);
  }
}

// ---- atan family -----------------------------------------------------------------------------------
PM_FN double sqrt_d(double x) {
#if defined(__CUDA_ARCH__)
  return __dsqrt_rn(x);
#else
  return __builtin_sqrt(x);
#endif
}
PM_FN double atan_pos(double x) {  // x >= 0, finite or inf
  const double kPio2 = 1.57079632679489661923;
  const double kPio4 = 0.78539816339744830962;
  if (is_inf(x)) return kPio2;
  bool inv = x > 1.0;
  if (inv) x = 1.0 / x;
  double base = 0.0;
  if (x > 0.41421356237309503) {
    x = (x - 1.0) / (x + 1.0);
    base = kPio4;
  }
  double x2 = x * x;
  double s = 1.0 / 47.0;
  s = 1.0 / 45.0 - s * x2;
  s = 1.0 / 43.0 - s * x2;
  s = 1.0 / 41.0 - s * x2;
  s = 1.0 / 39.0 - s * x2;
  s = 1.0 / 37.0 - s * x2;
  s = 1.0 / 35.0 - s * x2;
  s = 1.0 / 33.0 - s * x2;
  s = 1.0 / 31.0 - s * x2;
  s = 1.0 / 29.0 - s * x2;
  s = 1.0 / 27.0 - s * x2;
  s = 1.0 / 25.0 - s * x2;
  s = 1.0 / 23.0 - s * x2;
  s = 1.0 / 21.0 - s * x2;
  s = 1.0 / 19.0 - s * x2;
  s = 1.0 / 17.0 - s * x2;
  s = 1.0 / 15.0 - s * x2;
  s = 1.0 / 13.0 - s * x2;
  s = 1.0 / 11.0 - s * x2;
  s = 1.0 / 9.0 - s * x2;
  s = 1.0 / 7.0 - s * x2;
  s = 1.0 / 5.0 - s * x2;
  s = 1.0 / 3.0 - s * x2;
  s = 1.0 - s * x2;
  double a = base + x * s;
  return inv ? (kPio2 - a) : a;
}
PM_FN double atan_d(double x) {
  if (is_nan(x)) return x;
  return sign_d(x) ? -atan_pos(-x) : atan_pos(x);
}
PM_FN double atan2_d(double y, double x) {
  const double kPi = 3.14159265358979323846;
  const double kPio2 = 1.57079632679489661923;
  if (is_nan(x) || is_nan(y)) return nan_d();
  bool ys = sign_d(y), xs = sign_d(x);
  if (y == 0.0) {
    double r = xs ? kPi : 0.0;
    return ys ? -r : r;
  }
  if (x == 0.0) return ys ? -kPio2 : kPio2;
  if (is_inf(x) && is_inf(y)) {
    double r = xs ? 3.0 * kPi / 4.0 : kPi / 4.0;
    return ys ? -r : r;
  }
  double a = atan_pos(abs_d(y) / abs_d(x));
  if (xs) a = kPi - a;
  return ys ? -a : a;
}

// ---- float front ends ------------------------------------------------------------------------------
PM_FN float expf_(float x) { return float(exp_d(double(x))); }
PM_FN float logf_(float x) { return float(log_d(double(x))); }
PM_FN float sinf_(float x) { return float(sin_d(double(x))); }
PM_FN float cosf_(float x) { return float(cos_d(double(x))); }
PM_FN float tanf_(float x) { return float(sin_d(double(x)) / cos_d(double(x))); }
PM_FN float atanf_(float x) { return float(atan_d(double(x))); }
PM_FN float atan2f_(float y, float x) { return float(atan2_d(double(y), double(x))); }
PM_FN float acosf_(float x) {
  double d = double(x);
  if (is_nan(d)) return x;
  if (d > 1.0 || d < -1.0) return float(nan_d());
  return float(atan2_d(sqrt_d((1.0 - d) * (1.0 + d)), d));
}
PM_FN float asinf_(float x) {
  double d = double(x);
  if (is_nan(d)) return x;
  if (d > 1.0 || d < -1.0) return float(nan_d());
  return float(atan2_d(d, sqrt_d((1.0 - d) * (1.0 + d))));
}
PM_FN float coshf_(float x) {
  double e = exp_d(abs_d(double(x)));
  return float(0.5 * (e + 1.0 / e));
}
PM_FN float sinhf_(float x) {
  double d = double(x);
  double a = abs_d(d);
  double r;
  if (a < 0.125) {
    double a2 = a * a;
    r = a * (1.0 + a2 * (1.0 / 6.0 + a2 * (1.0 / 120.0 + a2 * (1.0 / 5040.0 + a2 * (1.0 / 362880.0)))));
  } else {
    double e = exp_d(a);
    r = 0.5 * (e - 1.0 / e);
  }
  return float(sign_d(d) ? -r : r);
}
PM_FN float tanhf_(float x) {
  double d = double(x);
  if (is_nan(d)) return x;
  double a = abs_d(d);
  double r;
  if (a < 0.125) {
    double a2 = a * a;
    r = a * (1.0 + a2 * (-1.0 / 3.0 + a2 * (2.0 / 15.0 + a2 * (-17.0 / 315.0 + a2 * (62.0 / 2835.0 + a2 * (-1382.0 / 155925.0))))));
  } else if (a > 20.0) {
    r = 1.0;
  } else {
    double e = exp_d(2.0 * a);
    r = (e - 1.0) / (e + 1.0);
  }
  return float(sign_d(d) ? -r : r);
}
PM_FN float atanhf_(float x) {
  double d = double(x);
  if (is_nan(d)) return x;
  if (d > 1.0 || d < -1.0) return float(nan_d());
  return float(0.5 * log_d((1.0 + d) / (1.0 - d)));
}

PM_FN bool is_odd_integerf(float y) {
  // |y| < 2^24 and integral and odd
  float a = y < 0.0f ? -y : y;
  if (a >= 16777216.0f) return false;
  int i = int(a);
  return (float(i) == a) && (i & 1);
}
PM_FN bool is_integerf(float y) {
  float a = y < 0.0f ? -y : y;
  if (a >= 8388608.0f) return true;
  return float(int(a)) == a;
}
PM_FN float powf_(float x, float y) {
  const float kInf = bits_to_float(0x7f800000u);
  if (y == 0.0f) return 1.0f;
  if (x == 1.0f) return 1.0f;
  if (is_nanf(x) || is_nanf(y)) return bits_to_float(0x7fc00000u);
  float ax = x < 0.0f ? -x : x;
  bool xneg = (float_to_bits(x) >> 31) != 0;
  if (y == kInf) return (ax > 1.0f) ? kInf : ((ax == 1.0f) ? 1.0f : 0.0f);
  if (y == -kInf) return (ax > 1.0f) ? 0.0f : ((ax == 1.0f) ? 1.0f : kInf);
  if (ax == 0.0f) {
    bool odd = is_odd_integerf(y);
    if (y > 0.0f) return (odd && xneg) ? -0.0f : 0.0f;
    return (odd && xneg) ? -kInf : kInf;
  }
  if (ax == kInf) {
    bool odd = is_odd_integerf(y);
    if (y > 0.0f) return (odd && xneg) ? -kInf : kInf;
    return (odd && xneg) ? -0.0f : 0.0f;
  }
  if (xneg && !is_integerf(y)) return bits_to_float(0x7fc00000u);
  double r = exp_d(double(y) * log_d(double(ax)));
  if (xneg && is_odd_integerf(y)) r = -r;
  return float(r);
}

// ---- complex<float> helpers (results as re, im) ----------------------------------------------------
PM_FN void csqrtf_(float a, float b, float& re, float& im) {
  if (a == 0.0f && b == 0.0f) {
    re = 0.0f;
    im = b;
    return;
  }
  double da = double(a), db = double(b);
  double h = sqrt_d(da * da + db * db);
  double t = sqrt_d(0.5 * (abs_d(da) + h));
  if (da >= 0.0) {
    re = float(t);
    im = float(db / (2.0 * t));
  } else {
    double r = abs_d(db) / (2.0 * t);
    re = float(r);
    im = float(sign_d(db) ? -t : t);
  }
}
PM_FN void cexpf_(float a, float b, float& re, float& im) {
  double e = exp_d(double(a));
  if (b == 0.0f) {
    re = float(e);
    im = b;
    return;
  }
  re = float(e * cos_d(double(b)));
  im = float(e * sin_d(double(b)));
}
PM_FN float cabsf_(float a, float b) {
  double da = double(a), db = double(b);
  return float(sqrt_d(da * da + db * db));
}
// libgcc's __divsc3 computes float complex division in double and rounds once (gcc >= 10 on x86-64).
PM_FN void cdivf_(float a, float b, float c, float d, float& re, float& im) {
  double aa = a, bb = b, cc = c, dd = d;
  double denom = (cc * cc) + (dd * dd);
  re = float(((aa * cc) + (bb * dd)) / denom);
  im = float(((bb * cc) - (aa * dd)) / denom);
}

}  // namespace pm
