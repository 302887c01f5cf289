// The point terms of the conical distance-field penetration loss and their reverse-mode derivatives, templated on the
// scalar type: float in the loss kernels (penetration.cu), double in the penetration rows of the scan LM step (fit.cu).
// See penetration.cu for the definition of the loss.
#pragma once
#include <cuda_runtime.h>

namespace shapy {

struct PenParams {
  float sigma, linear_max;
  bool penalize_outside;
};

namespace pen {

template <typename T> struct V3 { T x, y, z; };
template <typename T> __device__ __forceinline__ V3<T> v3(T x, T y, T z) { return V3<T>{x, y, z}; }
template <typename T> __device__ __forceinline__ V3<T> ld(const float *p) { return V3<T>{(T)p[0], (T)p[1], (T)p[2]}; }
template <typename T> __device__ __forceinline__ V3<T> operator+(V3<T> a, V3<T> b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <typename T> __device__ __forceinline__ V3<T> operator-(V3<T> a, V3<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <typename T> __device__ __forceinline__ V3<T> operator*(T s, V3<T> a) { return {s * a.x, s * a.y, s * a.z}; }
template <typename T> __device__ __forceinline__ T dot(V3<T> a, V3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <typename T> __device__ __forceinline__ V3<T> cross(V3<T> a, V3<T> b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}

template <typename T> struct Cone {
  V3<T> x[3];
  V3<T> alpha, beta, N, s, t, y, c, n;
  T la, lb, lab, nN, r, k;
};

// loss.py calc_circumcircle and the unit normal of the triangle (x0, x1, x2)
template <typename T> __device__ __forceinline__ Cone<T> make_cone(V3<T> x0, V3<T> x1, V3<T> x2) {
  Cone<T> q;
  q.x[0] = x0; q.x[1] = x1; q.x[2] = x2;
  q.N = cross(x1 - x0, x2 - x0);
  q.alpha = x0 - x2;
  q.beta = x1 - x2;
  q.nN = sqrt(dot(q.N, q.N));
  q.la = sqrt(dot(q.alpha, q.alpha));
  q.lb = sqrt(dot(q.beta, q.beta));
  const V3<T> ab = q.alpha - q.beta;
  q.lab = sqrt(dot(ab, ab));
  q.r = q.lab / ((T)2 * q.nN) * q.la * q.lb;
  q.s = dot(q.alpha, q.alpha) * q.beta - dot(q.beta, q.beta) * q.alpha;
  q.t = cross(q.alpha, q.beta);
  q.y = cross(q.s, q.t);
  q.k = (T)2 * dot(q.N, q.N);
  q.c = ((T)1 / q.k) * q.y + x2;
  q.n = ((T)1 / q.nN) * q.N;
  return q;
}

// repulsion_intensity and its derivative
template <typename T> __device__ __forceinline__ T psi_of(T x, const PenParams &pp, T &dpsi) {
  const T s = pp.sigma;
  const bool lin = x <= -s && x > -(T)pp.linear_max;
  const bool quad = x > -s && (pp.penalize_outside ? x < s : x < (T)0);
  const T qa = -((T)1 - (T)2 * s) / ((T)4 * s * s);
  dpsi = (lin ? (T)-1 : (T)0) + (quad ? (T)2 * qa * x - (T)1 / ((T)2 * s) : (T)0);
  return (lin ? -x + (T)1 - s : (T)0) +
         (quad ? qa * x * x - (T)1 / ((T)2 * s) * x + (T)0.25 * ((T)3 - (T)2 * s) : (T)0);
}

template <typename T> struct PointTerms {
  V3<T> d, w;
  T x, m, D, a, psi, dpsi, u, mask, phi1, phi;
};

// phi = ([a < 1] ((1 - a) psi(x))^2)^2 of point p in cone q
template <typename T> __device__ __forceinline__ PointTerms<T> point_terms(V3<T> p, const Cone<T> &q, const PenParams &pp) {
  PointTerms<T> e;
  const T sigma = pp.sigma;
  e.d = p - q.c;
  e.x = dot(e.d, q.n);
  e.w = e.d - e.x * q.n;
  e.m = sqrt(dot(e.w, e.w));
  e.D = -q.r / sigma * e.x + q.r + (T)1e-6;
  e.a = e.m / e.D;
  e.psi = psi_of(e.x, pp, e.dpsi);
  e.u = ((T)1 - e.a) * e.psi;
  e.mask = e.a < (T)1 ? (T)1 : (T)0;
  e.phi1 = e.mask * (e.u * e.u);
  e.phi = e.phi1 * e.phi1;
  return e;
}

// Gradient of gphi * phi at point p in cone q (e its point_terms): adds to gp and to the cone's (gc, gn, gr).
template <typename T>
__device__ __forceinline__ void point_backward(V3<T> p, const Cone<T> &q, const PointTerms<T> &e, const PenParams &pp,
                                               T gphi, V3<T> &gp, V3<T> &gc, V3<T> &gn, T &gr) {
  const T sigma = pp.sigma;
  const T G = gphi * (T)2 * e.phi1 * e.mask * (T)2 * e.u;  // d(gphi phi)/du
  if (G == (T)0) return;                                   // a NaN G goes on, as the reference's does
  const T ga = -e.psi * G;
  T gx = ((T)1 - e.a) * e.dpsi * G;
  const T gm = ga / e.D, gD = -ga * e.a / e.D;
  gr += gD * ((T)1 - e.x / sigma);
  gx += gD * (-q.r / sigma);
  const V3<T> gw = e.m > (T)0 ? (gm / e.m) * e.w : v3<T>(0, 0, 0);
  gx -= dot(gw, q.n);
  gn = gn + (-e.x) * gw + gx * e.d;
  const V3<T> gd = gw + gx * q.n;
  gp = gp + gd;
  gc = gc - gd;
}

// The cone's (gc, gn, gr) back to its three vertices, added to gx[3].
template <typename T>
__device__ __forceinline__ void cone_backward(const Cone<T> &q, V3<T> gc, V3<T> gn, T gr, V3<T> gx[3]) {
  V3<T> gN = ((T)1 / q.nN) * (gn - dot(q.n, gn) * q.n);
  // r = lab / (2 nN) la lb
  const V3<T> ab = q.alpha - q.beta;
  const V3<T> gab = (gr * q.r / (q.lab * q.lab)) * ab;
  V3<T> galpha = gab + (gr * q.r / (q.la * q.la)) * q.alpha;
  V3<T> gbeta = (gr * q.r / (q.lb * q.lb)) * q.beta - gab;
  gN = gN - (gr * q.r / (q.nN * q.nN)) * q.N;
  // c = x2 + y / k, y = s x t, k = 2 N.N
  gx[2] = gx[2] + gc;
  const V3<T> gy = ((T)1 / q.k) * gc;
  const T gk = -dot(gc, q.y) / (q.k * q.k);
  gN = gN + ((T)4 * gk) * q.N;
  const V3<T> gs = cross(q.t, gy), gt = cross(gy, q.s);
  // s = |alpha|^2 beta - |beta|^2 alpha
  gbeta = gbeta + dot(q.alpha, q.alpha) * gs - ((T)2 * dot(q.alpha, gs)) * q.beta;
  galpha = galpha - dot(q.beta, q.beta) * gs + ((T)2 * dot(q.beta, gs)) * q.alpha;
  // t = alpha x beta
  galpha = galpha + cross(q.beta, gt);
  gbeta = gbeta + cross(gt, q.alpha);
  // N = (x1 - x0) x (x2 - x0)
  const V3<T> ge0 = cross(q.x[2] - q.x[0], gN), ge1 = cross(gN, q.x[1] - q.x[0]);
  gx[0] = gx[0] - ge0 - ge1 + galpha;
  gx[1] = gx[1] + ge0 + gbeta;
  gx[2] = gx[2] + ge1 - galpha - gbeta;
}

// Face indices of a pair row: false for a row whose first index is < 0 or with an index outside [0, F).
__device__ __forceinline__ bool pair_faces(const int *pairs, const int *faces, int F, int r[3], int i[3]) {
  const int fr = pairs[0], fi = pairs[1];
  if (fr < 0 || fr >= F || fi < 0 || fi >= F) return false;
  for (int k = 0; k < 3; ++k) { r[k] = faces[3 * fr + k]; i[k] = faces[3 * fi + k]; }
  return true;
}

}  // namespace pen
}  // namespace shapy
