/* TEST INFRASTRUCTURE ONLY -- the plain-C restatement of the reference's mesh-mesh intersection operator
 * (oracle/mmi_oracle.c: the same functions, line for line, quirks and deviations included; see its header for the
 * op.cu line map), written once for a scalar type `real` so that it covers the reference's two instantiations
 * (AT_DISPATCH_FLOATING_TYPES, op.cu:996):
 *   -DMMI_DOUBLE   double: oracle/_build/libmmi_oracle_f64.so, the oracle of shapy_mmi_forward_f64;
 *   (default)      float:  oracle/_build/libmmi_oracle_scalar_f32.so, checked byte for byte against the pinned
 *                  float oracle (tests/test_mmi_f64_cpu.py), which shows the two sources compute the same thing.
 * The double instantiation rounds to float where op.cu's does, because fabsf / fmaxf / fminf take float:
 *   CMP (91-92): the difference and the operands are converted to float, against FLT_EPSILON;
 *   isect_interval (234-253): the projections are folded with fminf / fmaxf, so every interval is float;
 * everything else (AABBs and the inclusive leaf test, the ray test with |det| < 1e-4 and t + 1e-4 in double,
 * barycentrics with 1.0 - y - z, tmin = DBL_MAX) stays double.  For float those conversions are no-ops.
 *
 * Slot ORDER differs from the reference (all AABB-overlapping pairs in increasing target index); the slot SET and
 * the per-slot barycentrics are what is compared.  A collision with no ray hit keeps zero barycentrics.
 *
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC [-DMMI_DOUBLE] (see oracle/mmi_oracle_f64.py).
 */
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#define EPSILON 1e-4

#ifdef MMI_DOUBLE
typedef double real;
#define REAL_MAX DBL_MAX
#define RMIN fmin
#define RMAX fmax
#else
typedef float real;
#define REAL_MAX FLT_MAX
#define RMIN fminf
#define RMAX fmaxf
#endif

typedef struct { real x, y, z; } v3;
typedef struct { v3 v0, v1, v2; } tri_t;

static inline v3 sub(v3 a, v3 b) { v3 r = {a.x - b.x, a.y - b.y, a.z - b.z}; return r; }
static inline v3 add(v3 a, v3 b) { v3 r = {a.x + b.x, a.y + b.y, a.z + b.z}; return r; }
static inline v3 scale(real s, v3 a) { v3 r = {a.x * s, a.y * s, a.z * s}; return r; }
static inline real dot(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static inline v3 cross(v3 a, v3 b) {
  v3 r = {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
  return r;
}
static inline int CMP(real x, real y) {
  return fabsf((float)(x - y)) <= FLT_EPSILON * fmaxf(1.0f, fmaxf(fabsf((float)x), fabsf((float)y)));
}

static v3 sat_cross_edge(v3 a, v3 b, v3 c, v3 d) {
  v3 ab = sub(b, a), cd = sub(d, c);
  v3 result = cross(ab, cd);
  if (!CMP(dot(ab, cd), 0.0f)) return result;
  v3 axis = cross(ab, sub(c, a));
  result = cross(ab, axis);
  if (!CMP(dot(result, result), 0.0f)) return result;
  v3 z = {0.f, 0.f, 0.f};
  return z;
}

static inline void interval(v3 ax, const tri_t *t, float *lo, float *hi) {
  float p = (float)dot(ax, t->v0);
  *lo = p; *hi = p;
  p = (float)dot(ax, t->v1); *lo = fminf(*lo, p); *hi = fmaxf(*hi, p);
  p = (float)dot(ax, t->v2); *lo = fminf(*lo, p); *hi = fmaxf(*hi, p);
}

static int sat11(const tri_t *t1, const tri_t *t2) {
  v3 axes[11];
  axes[0] = sat_cross_edge(t1->v0, t1->v1, t1->v1, t1->v2);
  axes[1] = sat_cross_edge(t2->v0, t2->v1, t2->v1, t2->v2);
  const v3 *a[3][2] = {{&t1->v0, &t1->v1}, {&t1->v1, &t1->v2}, {&t1->v2, &t1->v0}};
  const v3 *b[3][2] = {{&t2->v0, &t2->v1}, {&t2->v1, &t2->v2}, {&t2->v2, &t2->v0}};
  int n = 2;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) axes[n++] = sat_cross_edge(*a[i][0], *a[i][1], *b[j][0], *b[j][1]);
  for (int i = 0; i < 11; ++i) {
    float l1, h1, l2, h2;
    interval(axes[i], t1, &l1, &h1);
    interval(axes[i], t2, &l2, &h2);
    int overlap = (l1 <= h2) && (l2 <= h1);
    if (!overlap && !CMP(dot(axes[i], axes[i]), 0.0f)) return 0;
  }
  return 1;
}

static int ray_tri(v3 orig, v3 dir, v3 v0, v3 v1, v3 v2, real *t, v3 *p) {
  v3 v0v1 = sub(v1, v0), v0v2 = sub(v2, v0);
  v3 pvec = cross(dir, v0v2);
  real det = dot(v0v1, pvec);
  if (fabs((double)det) < EPSILON) return 0;
  real inv = 1 / det;
  v3 tvec = sub(orig, v0);
  real u = dot(tvec, pvec) * inv;
  if (u < 0 || u > 1) return 0;
  v3 qvec = cross(tvec, v0v1);
  real v = dot(dir, qvec) * inv;
  if (v < 0 || u + v > 1) return 0;
  *t = dot(v0v2, qvec) * inv;
  *p = add(scale(*t, dir), orig);
  return 1;
}

static void to_bary(v3 p, v3 a, v3 b, v3 c, real *out) {
  v3 v0 = sub(b, a), v1 = sub(c, a), v2 = sub(p, a);
  real d00 = dot(v0, v0), d01 = dot(v0, v1), d11 = dot(v1, v1), d20 = dot(v2, v0), d21 = dot(v2, v1);
  real denom = d00 * d11 - d01 * d01;
  real y = (d11 * d20 - d01 * d21) / denom;
  real z = (d00 * d21 - d01 * d20) / denom;
  out[1] = y; out[2] = z;
  out[0] = (real)(1.0 - y - z);
}

/* returns 1 if a first point was found; bc1/bc2 (3 reals each) written only then */
static int isect_points(const tri_t *Q, const tri_t *T, real *bc1, real *bc2) {
  v3 qe[3] = {sub(Q->v1, Q->v0), sub(Q->v2, Q->v1), sub(Q->v0, Q->v2)};
  v3 qo[3] = {Q->v0, Q->v1, Q->v2};
  v3 te[3] = {sub(T->v1, T->v0), sub(T->v2, T->v1), sub(T->v0, T->v2)};
  v3 to[3] = {T->v0, T->v1, T->v2};
  real tmin = REAL_MAX;
  int found_first = 0, found_second = 0;
  v3 ip = {0, 0, 0}, ip1 = {0, 0, 0}, ip2 = {0, 0, 0};
  real t = 0; /* uninitialised in the reference; 0 and NaN give identical results */
  for (int i = 0; i < 3; ++i) {
    int hit = ray_tri(qo[i], qe[i], T->v0, T->v1, T->v2, &t, &ip);
    if (t > 1 || t < 0) continue;
    if (hit && !found_first) { ip1 = ip; found_first = 1; tmin = t; }
    /* op.cu:431-434: degenerate triangle (v1, v1, v2) => det == 0 => never hits */
    real s = (real)((double)t + EPSILON);
    hit = ray_tri(add(qo[i], scale(s, qe[i])), qe[i], T->v1, T->v1, T->v2, &t, &ip2);
    if (t > 1 || t < 0) continue;
    if (hit && found_first && t > tmin && !found_second) { ip2 = ip; found_second = 1; }
  }
  if (found_first) to_bary(ip1, T->v0, T->v1, T->v2, bc1);
  if (found_second) { to_bary(ip2, T->v0, T->v1, T->v2, bc2); return 1; }
  tmin = REAL_MAX;
  for (int i = 0; i < 3; ++i) {
    int hit = ray_tri(to[i], te[i], Q->v0, Q->v1, Q->v2, &t, &ip);
    if (t > 1 || t < 0) continue;
    if (hit && !found_first) { ip1 = ip; tmin = t; found_first = 1; }
    real s = (real)((double)t + EPSILON);
    hit = ray_tri(add(to[i], scale(s, te[i])), te[i], Q->v0, Q->v1, Q->v2, &t, &ip);
    if (t > 1 || t < 0) continue;
    if (hit && found_first && t > tmin && !found_second) { ip2 = ip; found_second = 1; }
  }
  if (found_first) to_bary(ip1, T->v0, T->v1, T->v2, bc1);
  if (found_second) { to_bary(ip2, T->v0, T->v1, T->v2, bc2); return 1; }
  if (found_first) { bc2[0] = bc1[0]; bc2[1] = bc1[1]; bc2[2] = bc1[2]; }
  return found_first;
}

static inline void bbox(const tri_t *t, real *mn, real *mx) {
  mn[0] = RMIN(t->v0.x, RMIN(t->v1.x, t->v2.x)); mx[0] = RMAX(t->v0.x, RMAX(t->v1.x, t->v2.x));
  mn[1] = RMIN(t->v0.y, RMIN(t->v1.y, t->v2.y)); mx[1] = RMAX(t->v0.y, RMAX(t->v1.y, t->v2.y));
  mn[2] = RMIN(t->v0.z, RMIN(t->v1.z, t->v2.z)); mx[2] = RMAX(t->v0.z, RMAX(t->v1.z, t->v2.z));
}

/* One body.  faces_out[Q*M] must be pre-filled with -1, bcs_out[Q*M*2*3] with 0.
 * Returns the largest per-query collision count (may exceed M: extra ones are dropped,
 * where the reference would write out of bounds). */
int mmi_oracle_scalar_forward(const real *query, const real *target, int Q, int F, int M, int64_t *faces_out,
                       real *bcs_out) {
  const tri_t *q = (const tri_t *)query;
  const tri_t *tg = (const tri_t *)target;
  int worst = 0;
  for (int qi = 0; qi < Q; ++qi) {
    real qmn[3], qmx[3];
    bbox(&q[qi], qmn, qmx);
    int n = 0;
    for (int f = 0; f < F; ++f) {
      real mn[3], mx[3];
      bbox(&tg[f], mn, mx);
      if (!((qmn[0] <= mx[0]) && (qmx[0] >= mn[0]) && (qmn[1] <= mx[1]) && (qmx[1] >= mn[1]) &&
            (qmn[2] <= mx[2]) && (qmx[2] >= mn[2])))
        continue;
      if (!sat11(&q[qi], &tg[f])) continue;
      if (n < M) {
        faces_out[(int64_t)qi * M + n] = f;
        real *b = bcs_out + ((int64_t)qi * M + n) * 6;
        isect_points(&q[qi], &tg[f], b, b + 3);
      }
      ++n;
    }
    if (n > worst) worst = n;
  }
  return worst;
}
