// Complex arithmetic helpers and register-resident radix-2/4/8/16 butterflies.
// Everything is templated on the real type T (double for the fp64 engine, float
// for the fp32 engine) and on SIGN (+1 inverse transform e^{+2 pi i ...}, -1
// forward).  No shared or global memory is touched here.
#pragma once
#include <cuda_runtime.h>

#ifndef HD
#ifdef CWTB_HOST_EMU
#define HD inline  // tests-only CPU emulation build: no device code at all
#define HD_NOINLINE inline
#else
#define HD __host__ __device__ __forceinline__
// a function whose code one kernel runs from several call sites: kept out of line so the kernel's
// code stays small enough for the instruction cache
#define HD_NOINLINE __host__ __device__ __noinline__
#endif
#endif

namespace cwtb {

template <typename T> struct Vec2;
template <> struct Vec2<double> { using type = double2; };
template <> struct Vec2<float> { using type = float2; };
template <typename T> using cx = typename Vec2<T>::type;

template <typename T> HD cx<T> mk(T a, T b) {
  cx<T> r; r.x = a; r.y = b; return r;
}
template <typename V> HD V cadd(V a, V b) { a.x += b.x; a.y += b.y; return a; }
template <typename V> HD V csub(V a, V b) { a.x -= b.x; a.y -= b.y; return a; }
template <typename V> HD V cmul(V a, V b) {
  V r;
  r.x = a.x * b.x - a.y * b.y;
  r.y = a.x * b.y + a.y * b.x;
  return r;
}
template <typename V> HD V cconj(V a) { a.y = -a.y; return a; }
// multiply by SIGN * i
template <int SIGN, typename V> HD V mul_si(V a) {
  V r;
  if (SIGN > 0) { r.x = -a.y; r.y = a.x; } else { r.x = a.y; r.y = -a.x; }
  return r;
}
template <typename V, typename T> HD V cscale(V a, T s) { a.x *= s; a.y *= s; return a; }

// sin(pi x), cos(pi x)
HD void sincospi_hd(double x, double *s, double *c) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  sincospi(x, s, c);
#else
  ::sincos(3.14159265358979323846 * x, s, c);
#endif
}

// sin(x), cos(x) in double
HD void sincos_hd(double x, double *s, double *c) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  sincos(x, s, c);
#else
  ::sincos(x, s, c);
#endif
}

// re^2 + im^2 with every operation rounded (no fused multiply-add): the value numpy's
// `re**2 + im**2` has, so that thresholds on it select the same points
HD double norm2_rn(double re, double im) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  return __dadd_rn(__dmul_rn(re, re), __dmul_rn(im, im));
#else
  return re * re + im * im;
#endif
}

// s + w x with each operation rounded (no fused multiply-add): a sum of such steps in a fixed order
// is one fixed sequence of correctly rounded operations, on the device and on the host alike
HD double add_mul_rn(double s, double w, double x) {
#if defined(__CUDA_ARCH__) && !defined(CWTB_HOST_EMU)
  return __dadd_rn(s, __dmul_rn(w, x));
#else
  return s + w * x;
#endif
}

// ---- DFT_R in registers: x[c] <- sum_i x[i] e^{SIGN 2 pi i * i*c/R}, natural order ----
template <int SIGN, typename V> HD void dft2(V &a, V &b) {
  V t = csub(a, b);
  a = cadd(a, b);
  b = t;
}

template <int SIGN, typename V>
HD void dft4(V &x0, V &x1, V &x2, V &x3) {
  V t0 = cadd(x0, x2), t1 = csub(x0, x2);
  V t2 = cadd(x1, x3), t3 = mul_si<SIGN>(csub(x1, x3));
  x0 = cadd(t0, t2);
  x2 = csub(t0, t2);
  x1 = cadd(t1, t3);
  x3 = csub(t1, t3);
}

// a * e^{SIGN i pi/4} and a * e^{SIGN 3 i pi/4}
template <int SIGN, typename T, typename V> HD V mul_w8_1(V a) {
  const T h = (T)0.70710678118654752440;
  V r;
  if (SIGN > 0) { r.x = (a.x - a.y) * h; r.y = (a.x + a.y) * h; }
  else          { r.x = (a.x + a.y) * h; r.y = (a.y - a.x) * h; }
  return r;
}
template <int SIGN, typename T, typename V> HD V mul_w8_3(V a) {
  const T h = (T)0.70710678118654752440;
  V r;  // e^{SIGN 3 i pi/4} = (-1 + SIGN i)/sqrt2
  if (SIGN > 0) { r.x = (-a.x - a.y) * h; r.y = (a.x - a.y) * h; }
  else          { r.x = (a.y - a.x) * h; r.y = (-a.x - a.y) * h; }
  return r;
}

template <int SIGN, typename T, typename V> HD void dft8(V *x) {
  // decimation in time: evens / odds
  V e0 = x[0], e1 = x[2], e2 = x[4], e3 = x[6];
  V o0 = x[1], o1 = x[3], o2 = x[5], o3 = x[7];
  dft4<SIGN>(e0, e1, e2, e3);
  dft4<SIGN>(o0, o1, o2, o3);
  o1 = mul_w8_1<SIGN, T>(o1);
  o2 = mul_si<SIGN>(o2);
  o3 = mul_w8_3<SIGN, T>(o3);
  x[0] = cadd(e0, o0); x[4] = csub(e0, o0);
  x[1] = cadd(e1, o1); x[5] = csub(e1, o1);
  x[2] = cadd(e2, o2); x[6] = csub(e2, o2);
  x[3] = cadd(e3, o3); x[7] = csub(e3, o3);
}

template <int SIGN, typename T, typename V> HD void dft16(V *x) {
  V e[8], o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { e[i] = x[2 * i]; o[i] = x[2 * i + 1]; }
  dft8<SIGN, T>(e);
  dft8<SIGN, T>(o);
  // w16^c = e^{SIGN i pi c/8}
  const T c1 = (T)0.92387953251128675613, s1 = (T)0.38268343236508977173;
  V w;
  w.x = c1; w.y = SIGN * s1;  o[1] = cmul(o[1], w);
  o[2] = mul_w8_1<SIGN, T>(o[2]);
  w.x = s1; w.y = SIGN * c1;  o[3] = cmul(o[3], w);
  o[4] = mul_si<SIGN>(o[4]);
  w.x = -s1; w.y = SIGN * c1; o[5] = cmul(o[5], w);
  o[6] = mul_w8_3<SIGN, T>(o[6]);
  w.x = -c1; w.y = SIGN * s1; o[7] = cmul(o[7], w);
#pragma unroll
  for (int i = 0; i < 8; ++i) { x[i] = cadd(e[i], o[i]); x[i + 8] = csub(e[i], o[i]); }
}

// radix-32: two radix-16 halves (even / odd inputs) + w32^c twiddles
template <int SIGN, typename T, typename V> HD void dft32(V *x) {
  V e[16], o[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) { e[i] = x[2 * i]; o[i] = x[2 * i + 1]; }
  dft16<SIGN, T>(e);
  dft16<SIGN, T>(o);
  // cos(k pi/16), sin(k pi/16), k = 1..7
  const T c1 = (T)0.98078528040323044913, s1 = (T)0.19509032201612826785;
  const T c2 = (T)0.92387953251128675613, s2 = (T)0.38268343236508977173;
  const T c3 = (T)0.83146961230254523708, s3 = (T)0.55557023301960222474;
  const T c5 = s3, s5 = c3, c6 = s2, s6 = c2, c7 = s1, s7 = c1;
  V w;
#define CWTB_TW32(k, cr, sr) w.x = (cr); w.y = SIGN * (sr); o[k] = cmul(o[k], w);
  CWTB_TW32(1, c1, s1)
  CWTB_TW32(2, c2, s2)
  CWTB_TW32(3, c3, s3)
  o[4] = mul_w8_1<SIGN, T>(o[4]);
  CWTB_TW32(5, c5, s5)
  CWTB_TW32(6, c6, s6)
  CWTB_TW32(7, c7, s7)
  o[8] = mul_si<SIGN>(o[8]);
  CWTB_TW32(9, -s1, c1)
  CWTB_TW32(10, -s2, c2)
  CWTB_TW32(11, -s3, c3)
  o[12] = mul_w8_3<SIGN, T>(o[12]);
  CWTB_TW32(13, -c3, s3)
  CWTB_TW32(14, -c2, s2)
  CWTB_TW32(15, -c1, s1)
#undef CWTB_TW32
#pragma unroll
  for (int i = 0; i < 16; ++i) { x[i] = cadd(e[i], o[i]); x[i + 16] = csub(e[i], o[i]); }
}

template <int R, int SIGN, typename T, typename V> HD void dftR(V *x) {
  if (R == 2) dft2<SIGN>(x[0], x[1]);
  else if (R == 4) dft4<SIGN>(x[0], x[1], x[2], x[3]);
  else if (R == 8) dft8<SIGN, T>(x);
  else if (R == 16) dft16<SIGN, T>(x);
  else if (R == 32) dft32<SIGN, T>(x);
}

}  // namespace cwtb
