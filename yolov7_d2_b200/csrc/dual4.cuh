// Forward-mode differentiation with a 4-wide dual number: value + partial derivatives w.r.t. one (cx, cy, w, h) box.  Box-loss kernels
// written with it follow the reference formula line by line and get the gradient of exactly that arithmetic.  Sub-gradients of min / max /
// clamp match torch: ties between the two arguments split 0.5 / 0.5, and a clamp passes the gradient at its bound.
#pragma once

namespace {

struct D4 {
  float v, g[4];
};
__device__ __forceinline__ D4 cst(float v) { return D4{v, {0.f, 0.f, 0.f, 0.f}}; }
__device__ __forceinline__ D4 var(float v, int i) {
  D4 r = cst(v);
  r.g[i] = 1.f;
  return r;
}
__device__ __forceinline__ D4 operator+(const D4& a, const D4& b) { return D4{a.v + b.v, {a.g[0] + b.g[0], a.g[1] + b.g[1], a.g[2] + b.g[2], a.g[3] + b.g[3]}}; }
__device__ __forceinline__ D4 operator-(const D4& a, const D4& b) { return D4{a.v - b.v, {a.g[0] - b.g[0], a.g[1] - b.g[1], a.g[2] - b.g[2], a.g[3] - b.g[3]}}; }
__device__ __forceinline__ D4 operator*(const D4& a, const D4& b) {
  return D4{a.v * b.v, {a.g[0] * b.v + a.v * b.g[0], a.g[1] * b.v + a.v * b.g[1], a.g[2] * b.v + a.v * b.g[2], a.g[3] * b.v + a.v * b.g[3]}};
}
__device__ __forceinline__ D4 operator/(const D4& a, const D4& b) {
  const float q = a.v / b.v, ib = 1.f / b.v;
  return D4{q, {(a.g[0] - q * b.g[0]) * ib, (a.g[1] - q * b.g[1]) * ib, (a.g[2] - q * b.g[2]) * ib, (a.g[3] - q * b.g[3]) * ib}};
}
__device__ __forceinline__ D4 operator+(const D4& a, float b) { D4 r = a; r.v += b; return r; }
__device__ __forceinline__ D4 operator-(const D4& a, float b) { D4 r = a; r.v -= b; return r; }
__device__ __forceinline__ D4 operator*(const D4& a, float b) { return D4{a.v * b, {a.g[0] * b, a.g[1] * b, a.g[2] * b, a.g[3] * b}}; }
__device__ __forceinline__ D4 operator-(float a, const D4& b) { return D4{a - b.v, {-b.g[0], -b.g[1], -b.g[2], -b.g[3]}}; }
__device__ __forceinline__ D4 mix(const D4& a, const D4& b, float wa) {  // wa*a + (1-wa)*b on the derivatives
  const float wb = 1.f - wa;
  return D4{wa >= 0.5f ? a.v : b.v, {wa * a.g[0] + wb * b.g[0], wa * a.g[1] + wb * b.g[1], wa * a.g[2] + wb * b.g[2], wa * a.g[3] + wb * b.g[3]}};
}
__device__ __forceinline__ D4 dmax(const D4& a, const D4& b) { return a.v > b.v ? a : (a.v < b.v ? b : mix(a, b, 0.5f)); }
__device__ __forceinline__ D4 dmin(const D4& a, const D4& b) { return a.v < b.v ? a : (a.v > b.v ? b : mix(a, b, 0.5f)); }
__device__ __forceinline__ D4 clamp_min(const D4& a, float lo) { return a.v >= lo ? a : cst(lo); }  // torch.clamp: gradient 1 at the bound
__device__ __forceinline__ D4 clamp(const D4& a, float lo, float hi) { return (a.v >= lo && a.v <= hi) ? a : cst(a.v < lo ? lo : hi); }
__device__ __forceinline__ D4 datan(const D4& a) {
  const float d = 1.f / (1.f + a.v * a.v);
  return D4{atanf(a.v), {a.g[0] * d, a.g[1] * d, a.g[2] * d, a.g[3] * d}};
}

}  // namespace
