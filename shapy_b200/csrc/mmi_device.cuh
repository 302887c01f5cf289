// Device-side triangle/triangle predicates with the exact semantics of the reference operator
// mesh-mesh-intersection/src/mesh_mesh_intersect_cuda_op.cu (quirks included; SURVEY.md 8c):
//   CMP 91-92, SatCrossEdge 151-169, point_to_barycentric 186-200, ray_triangle_intersect 202-232,
//   isect_interval 234-253, TriangleTriangleIsectSepAxis 270-341, checkOverlap 362-373,
//   find_triangle_triangle_intersection_points 375-518.
// Templated on the scalar type T (float or double) as the reference is.  Its double instantiation still
// passes values through float-only functions, and so does this one, at exactly the same points:
//   - CMP converts the difference and the operands to float (fabsf / fmaxf) against FLT_EPSILON: cmp0();
//   - isect_interval folds the projections with fminf / fmaxf, so each interval is float-rounded before the
//     overlap test: axis_separates();
//   - everything else (cross products, projections, AABBs, the ray test, barycentrics) stays in T.
// For T = float the conversions are no-ops.
// Translation units including this header are compiled with -fmad=false so that the results are identical
// to the plain-C oracles (oracle/mmi_oracle.c for float, oracle/mmi_oracle_scalar.c built as double).
#pragma once
#include <cfloat>
#include <cuda_runtime.h>

namespace shapy {
namespace mmi {

template <typename T> struct Vec3;
template <> struct Vec3<float> { using type = float3; };
template <> struct Vec3<double> { using type = double3; };
template <typename T> using vec3 = typename Vec3<T>::type;

template <typename T>
struct TriT {
  vec3<T> v0, v1, v2;
};
using Tri = TriT<float>;

template <typename V> __device__ __forceinline__ V sub3(V a, V b) { return V{a.x - b.x, a.y - b.y, a.z - b.z}; }
template <typename V> __device__ __forceinline__ V add3(V a, V b) { return V{a.x + b.x, a.y + b.y, a.z + b.z}; }
template <typename S, typename V> __device__ __forceinline__ V mul3(S s, V a) { return V{a.x * s, a.y * s, a.z * s}; }
template <typename V> __device__ __forceinline__ auto dot3(V a, V b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename V> __device__ __forceinline__ V cross3(V a, V b) {
  return V{a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
__device__ __forceinline__ float min_(float a, float b) { return fminf(a, b); }
__device__ __forceinline__ float max_(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ double min_(double a, double b) { return fmin(a, b); }
__device__ __forceinline__ double max_(double a, double b) { return fmax(a, b); }

// CMP(x, 0): fabsf / fmaxf take float, so a double x is rounded to float first.
template <typename T> __device__ __forceinline__ bool cmp0(T x) {
  const float f = (float)x;
  return fabsf(f) <= FLT_EPSILON * fmaxf(1.0f, fabsf(f));
}

template <typename V> __device__ __forceinline__ V sat_cross_edge(V a, V b, V c, V d) {
  V ab = sub3(b, a), cd = sub3(d, c);
  V result = cross3(ab, cd);
  if (!cmp0(dot3(ab, cd))) return result;
  V axis = cross3(ab, sub3(c, a));
  result = cross3(ab, axis);
  if (!cmp0(dot3(result, result))) return result;
  return V{0, 0, 0};
}

// isect_interval: the projections are exact in T, the fminf / fmaxf folding rounds them to float.
template <typename T>
__device__ __forceinline__ bool axis_separates(vec3<T> ax, const TriT<T> &t1, const TriT<T> &t2) {
  float p = (float)dot3(ax, t1.v0), l1 = p, h1 = p;
  p = (float)dot3(ax, t1.v1); l1 = fminf(l1, p); h1 = fmaxf(h1, p);
  p = (float)dot3(ax, t1.v2); l1 = fminf(l1, p); h1 = fmaxf(h1, p);
  p = (float)dot3(ax, t2.v0);
  float l2 = p, h2 = p;
  p = (float)dot3(ax, t2.v1); l2 = fminf(l2, p); h2 = fmaxf(h2, p);
  p = (float)dot3(ax, t2.v2); l2 = fminf(l2, p); h2 = fmaxf(h2, p);
  bool overlap = (l1 <= h2) && (l2 <= h1);
  return !overlap && !cmp0(dot3(ax, ax));
}

template <typename T>
__device__ inline bool sat11(const TriT<T> &t1, const TriT<T> &t2) {
  if (axis_separates<T>(sat_cross_edge(t1.v0, t1.v1, t1.v1, t1.v2), t1, t2)) return false;
  if (axis_separates<T>(sat_cross_edge(t2.v0, t2.v1, t2.v1, t2.v2), t1, t2)) return false;
  const vec3<T> a0[3] = {t1.v0, t1.v1, t1.v2}, a1[3] = {t1.v1, t1.v2, t1.v0};
  const vec3<T> b0[3] = {t2.v0, t2.v1, t2.v2}, b1[3] = {t2.v1, t2.v2, t2.v0};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j)
      if (axis_separates<T>(sat_cross_edge(a0[i], a1[i], b0[j], b1[j]), t1, t2)) return false;
  return true;
}

// EPSILON (1e-4) is a double literal: the |det| test is in double for both scalar types.
template <typename T, typename V>
__device__ __forceinline__ bool ray_tri(V orig, V dir, V v0, V v1, V v2, T &t, V &p) {
  V v0v1 = sub3(v1, v0), v0v2 = sub3(v2, v0);
  V pvec = cross3(dir, v0v2);
  T det = dot3(v0v1, pvec);
  if (fabs((double)det) < 1e-4) return false;
  T inv = 1 / det;
  V tvec = sub3(orig, v0);
  T u = dot3(tvec, pvec) * inv;
  if (u < 0 || u > 1) return false;
  V qvec = cross3(tvec, v0v1);
  T v = dot3(dir, qvec) * inv;
  if (v < 0 || u + v > 1) return false;
  t = dot3(v0v2, qvec) * inv;
  p = add3(mul3(t, dir), orig);
  return true;
}

template <typename V> __device__ __forceinline__ V to_bary(V p, V a, V b, V c) {
  using T = decltype(p.x);
  V v0 = sub3(b, a), v1 = sub3(c, a), v2 = sub3(p, a);
  T d00 = dot3(v0, v0), d01 = dot3(v0, v1), d11 = dot3(v1, v1), d20 = dot3(v2, v0), d21 = dot3(v2, v1);
  T denom = d00 * d11 - d01 * d01;
  T y = (d11 * d20 - d01 * d21) / denom;
  T z = (d00 * d21 - d01 * d20) / denom;
  return V{(T)(1.0 - y - z), y, z};
}

// Returns true when a first intersection point exists; bc1/bc2 written only then.
template <typename T>
__device__ inline bool isect_points(const TriT<T> &Q, const TriT<T> &T_, vec3<T> &bc1, vec3<T> &bc2) {
  using V = vec3<T>;
  const V qe[3] = {sub3(Q.v1, Q.v0), sub3(Q.v2, Q.v1), sub3(Q.v0, Q.v2)};
  const V qo[3] = {Q.v0, Q.v1, Q.v2};
  const V te[3] = {sub3(T_.v1, T_.v0), sub3(T_.v2, T_.v1), sub3(T_.v0, T_.v2)};
  const V to[3] = {T_.v0, T_.v1, T_.v2};
  const T t_max = sizeof(T) == 4 ? (T)FLT_MAX : (T)DBL_MAX;
  T tmin = t_max;
  bool found_first = false, found_second = false;
  V ip = V{0, 0, 0}, ip1 = ip, ip2 = ip;
  T t = 0;  // uninitialised in the reference; 0 / NaN give identical results
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    bool hit = ray_tri(qo[i], qe[i], T_.v0, T_.v1, T_.v2, t, ip);
    if (t > 1 || t < 0) continue;
    if (hit && !found_first) { ip1 = ip; found_first = true; tmin = t; }
    T s = (T)((double)t + 1e-4);
    hit = ray_tri(add3(qo[i], mul3(s, qe[i])), qe[i], T_.v1, T_.v1, T_.v2, t, ip2);  // degenerate: never hits
    if (t > 1 || t < 0) continue;
    if (hit && found_first && t > tmin && !found_second) { ip2 = ip; found_second = true; }
  }
  if (found_first) bc1 = to_bary(ip1, T_.v0, T_.v1, T_.v2);
  if (found_second) { bc2 = to_bary(ip2, T_.v0, T_.v1, T_.v2); return true; }
  tmin = t_max;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    bool hit = ray_tri(to[i], te[i], Q.v0, Q.v1, Q.v2, t, ip);
    if (t > 1 || t < 0) continue;
    if (hit && !found_first) { ip1 = ip; tmin = t; found_first = true; }
    T s = (T)((double)t + 1e-4);
    hit = ray_tri(add3(to[i], mul3(s, te[i])), te[i], Q.v0, Q.v1, Q.v2, t, ip);
    if (t > 1 || t < 0) continue;
    if (hit && found_first && t > tmin && !found_second) { ip2 = ip; found_second = true; }
  }
  if (found_first) bc1 = to_bary(ip1, T_.v0, T_.v1, T_.v2);
  if (found_second) { bc2 = to_bary(ip2, T_.v0, T_.v1, T_.v2); return true; }
  if (found_first) bc2 = bc1;
  return found_first;
}

template <typename T>
struct BoxT {
  vec3<T> lo, hi;
};
using Box = BoxT<float>;
template <typename T> __device__ __forceinline__ BoxT<T> tri_box(const TriT<T> &t) {
  BoxT<T> b;
  b.lo = vec3<T>{min_(t.v0.x, min_(t.v1.x, t.v2.x)), min_(t.v0.y, min_(t.v1.y, t.v2.y)),
                 min_(t.v0.z, min_(t.v1.z, t.v2.z))};
  b.hi = vec3<T>{max_(t.v0.x, max_(t.v1.x, t.v2.x)), max_(t.v0.y, max_(t.v1.y, t.v2.y)),
                 max_(t.v0.z, max_(t.v1.z, t.v2.z))};
  return b;
}
template <typename T> __device__ __forceinline__ bool box_overlap(const BoxT<T> &a, const BoxT<T> &b) {
  return (a.lo.x <= b.hi.x) && (a.hi.x >= b.lo.x) && (a.lo.y <= b.hi.y) && (a.hi.y >= b.lo.y) &&
         (a.lo.z <= b.hi.z) && (a.hi.z >= b.lo.z);
}

// Float bounds of a T interval that contain it: the identity for float, outward rounding for double.
__device__ __forceinline__ float lo_f32(float x) { return x; }
__device__ __forceinline__ float hi_f32(float x) { return x; }
__device__ __forceinline__ float lo_f32(double x) { return __double2float_rd(x); }
__device__ __forceinline__ float hi_f32(double x) { return __double2float_ru(x); }
template <typename T> __device__ __forceinline__ Box box_f32(const BoxT<T> &b) {
  Box r;
  r.lo = make_float3(lo_f32(b.lo.x), lo_f32(b.lo.y), lo_f32(b.lo.z));
  r.hi = make_float3(hi_f32(b.hi.x), hi_f32(b.hi.y), hi_f32(b.hi.z));
  return r;
}

}  // namespace mmi
}  // namespace shapy
