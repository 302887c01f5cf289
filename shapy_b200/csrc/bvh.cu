// Batched LBVH mesh-mesh intersection: drop-in for mesh_mesh_intersect_cuda.mesh_to_mesh_forward
// (reference mesh-mesh-intersection/src/mesh_mesh_intersect.cpp:36-64 and
//  src/mesh_mesh_intersect_cuda_op.cu:969-1079), all bodies of the batch in the same launches, on the
// caller's stream, no host synchronisation, no allocation.
//
//   bvh_prepare_kernel   per body: triangle AABBs -> scene AABB -> 30-bit Morton code of each centroid
//                        (op.cu:140-149, 613-668), then an in-shared-memory bitonic sort of the
//                        (code, triangle id) pairs (replaces thrust::sort_by_key, op.cu:911)
//   bvh_topology_kernel  Karras-2012 radix tree, one thread per internal node (op.cu:670-765)
//   bvh_refit_kernel     bottom-up AABB refit with visit counters (op.cu:767-821)
//   bvh_query_kernel     ONE WARP PER QUERY TRIANGLE: a shared-memory node stack is drained 32 nodes at
//                        a time (each lane tests one node's two children, inclusive AABB test
//                        op.cu:362-373), overlapping internal children are pushed back and overlapping
//                        leaves queued with __ballot_sync compaction; queued leaves are then tested 32
//                        at a time with the reference's exact predicates (mmi_device.cuh) and hits are
//                        written to warp-aggregated slots.  The reference uses one THREAD per query
//                        triangle (2 active threads on the SHAPY path).
// Nodes are 32 bytes (AABB + 2 child links) instead of the reference's 72-byte pointer-based node.
// The prepare and query kernels are templated on the scalar type of the triangles (float or double, the
// reference's AT_DISPATCH_FLOATING_TYPES).  Node and leaf boxes stay float in both: for double triangles they are
// rounded outward, so the tree only prunes pairs whose double AABBs are disjoint, and the narrow phase repeats the
// reference's inclusive leaf test on the exact double AABBs before the SAT.
// Slot order within a query is unspecified (the reference's is traversal order); a collision without a
// ray hit keeps zero barycentrics (see DESIGN.md).  More than `max_collisions` hits per query are dropped
// (the reference writes out of bounds).  Compiled with -fmad=false.
#include "common.cuh"
#include "mmi_device.cuh"

namespace shapy {

struct __align__(16) BvhNode {
  float lo[3], hi[3];
  int left, right;  // >= 0: internal node index, < 0: leaf ~index (position in sorted order)
};

struct BvhWs {
  unsigned *codes;   // [B][F]
  int *ids;          // [B][F] sorted triangle ids
  BvhNode *nodes;    // [B][F-1] internal
  float *leaf_box;   // [B][F][6] in sorted order
  int *parent;       // [B][2F-1]: internal i -> parent[i], leaf j -> parent[F-1+j]
  int *counters;     // [B][F-1]
};

static size_t ws_layout(int B, int F, BvhWs *w, char *base) {
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += align_up(bytes, 256); return base ? base + o : nullptr; };
  char *p;
  p = take((size_t)B * F * 4); if (w) w->codes = (unsigned *)p;
  p = take((size_t)B * F * 4); if (w) w->ids = (int *)p;
  p = take((size_t)B * (F - 1) * sizeof(BvhNode)); if (w) w->nodes = (BvhNode *)p;
  p = take((size_t)B * F * 6 * 4); if (w) w->leaf_box = (float *)p;
  p = take((size_t)B * (2 * F - 1) * 4); if (w) w->parent = (int *)p;
  p = take((size_t)B * (F - 1) * 4); if (w) w->counters = (int *)p;
  return off;
}

template <typename T>
__device__ __forceinline__ mmi::TriT<T> ld_tri(const T *p) {
  mmi::TriT<T> t;
  t.v0 = mmi::vec3<T>{p[0], p[1], p[2]};
  t.v1 = mmi::vec3<T>{p[3], p[4], p[5]};
  t.v2 = mmi::vec3<T>{p[6], p[7], p[8]};
  return t;
}

__device__ __forceinline__ unsigned expand_bits(unsigned v) {
  v = (v * 0x00010001u) & 0xFF0000FFu;
  v = (v * 0x00000101u) & 0x0F00F00Fu;
  v = (v * 0x00000011u) & 0xC30C30C3u;
  v = (v * 0x00000005u) & 0x49249249u;
  return v;
}
__device__ __forceinline__ unsigned morton3d(float x, float y, float z) {
  x = fminf(fmaxf(x * 1024.0f, 0.0f), 1023.0f);
  y = fminf(fmaxf(y * 1024.0f, 0.0f), 1023.0f);
  z = fminf(fmaxf(z * 1024.0f, 0.0f), 1023.0f);
  return expand_bits((unsigned)x) * 4 + expand_bits((unsigned)y) * 2 + expand_bits((unsigned)z);
}

// One CTA per body.  Dynamic smem: codes[npow2] (u32) + ids[npow2] (u16/u32 depending on F).  The scene box and
// the centroids are computed in T; the normalised centroid is rounded to float for the Morton code, which only
// shapes the tree.
template <typename T, typename IdT>
__global__ void __launch_bounds__(1024) bvh_prepare_kernel(const T *__restrict__ target, int F, int npow2, BvhWs w) {
  extern __shared__ __align__(16) unsigned char sm[];
  unsigned *codes = reinterpret_cast<unsigned *>(sm);
  IdT *ids = reinterpret_cast<IdT *>(sm + (size_t)npow2 * 4);
  __shared__ T red[6][32];
  __shared__ T scene[6];
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const T *tb = target + (size_t)b * F * 9;
  const T big = sizeof(T) == 4 ? (T)FLT_MAX : (T)DBL_MAX;
  T lo[3] = {big, big, big}, hi[3] = {-big, -big, -big};
  for (int f = t; f < F; f += blockDim.x) {
    mmi::BoxT<T> bx = mmi::tri_box(ld_tri(tb + (size_t)f * 9));
    lo[0] = mmi::min_(lo[0], bx.lo.x); lo[1] = mmi::min_(lo[1], bx.lo.y); lo[2] = mmi::min_(lo[2], bx.lo.z);
    hi[0] = mmi::max_(hi[0], bx.hi.x); hi[1] = mmi::max_(hi[1], bx.hi.y); hi[2] = mmi::max_(hi[2], bx.hi.z);
  }
  for (int o = 16; o; o >>= 1)
    for (int c = 0; c < 3; ++c) {
      lo[c] = mmi::min_(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o));
      hi[c] = mmi::max_(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o));
    }
  if (lane == 0) for (int c = 0; c < 3; ++c) { red[c][warp] = lo[c]; red[3 + c][warp] = hi[c]; }
  __syncthreads();
  if (t < 6) {
    T v = red[t][0];
    for (int i = 1; i < (int)(blockDim.x >> 5); ++i) v = t < 3 ? mmi::min_(v, red[t][i]) : mmi::max_(v, red[t][i]);
    scene[t] = v;
  }
  __syncthreads();
  for (int f = t; f < npow2; f += blockDim.x) {
    unsigned code = 0xFFFFFFFFu;
    if (f < F) {
      mmi::TriT<T> tr = ld_tri(tb + (size_t)f * 9);
      T cx = (tr.v0.x + tr.v1.x + tr.v2.x) / (T)3, cy = (tr.v0.y + tr.v1.y + tr.v2.y) / (T)3,
        cz = (tr.v0.z + tr.v1.z + tr.v2.z) / (T)3;
      code = morton3d((float)((cx - scene[0]) / (scene[3] - scene[0])), (float)((cy - scene[1]) / (scene[4] - scene[1])),
                      (float)((cz - scene[2]) / (scene[5] - scene[2])));
    }
    codes[f] = code;
    ids[f] = (IdT)f;
  }
  __syncthreads();
  // bitonic sort on (code, id); padding keys are 0xFFFFFFFF with ids >= F so they end up last
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < npow2; i += blockDim.x) {
        int ixj = i ^ j;
        if (ixj > i) {
          unsigned ca = codes[i], cb = codes[ixj];
          IdT ia = ids[i], ib = ids[ixj];
          bool a_gt_b = ca > cb || (ca == cb && ia > ib);
          bool up = (i & k) == 0;
          if (a_gt_b == up) { codes[i] = cb; codes[ixj] = ca; ids[i] = ib; ids[ixj] = ia; }
        }
      }
      __syncthreads();
    }
  }
  for (int f = t; f < F; f += blockDim.x) {
    int id = (int)ids[f];
    w.codes[(size_t)b * F + f] = codes[f];
    w.ids[(size_t)b * F + f] = id;
    mmi::Box bx = mmi::box_f32(mmi::tri_box(ld_tri(tb + (size_t)id * 9)));
    float *lb = w.leaf_box + ((size_t)b * F + f) * 6;
    lb[0] = bx.lo.x; lb[1] = bx.lo.y; lb[2] = bx.lo.z; lb[3] = bx.hi.x; lb[4] = bx.hi.y; lb[5] = bx.hi.z;
  }
  for (int i = t; i < F - 1; i += blockDim.x) w.counters[(size_t)b * (F - 1) + i] = 0;
}

__device__ __forceinline__ int lcp(const unsigned *codes, const int *ids, int F, int i, int j) {
  if (i < 0 || i > F - 1 || j < 0 || j > F - 1) return -1;
  unsigned a = codes[i], c = codes[j];
  if (a == c) return __clz(a ^ c) + __clz(ids[i] ^ ids[j]);
  return __clz(a ^ c);
}

__global__ void bvh_topology_kernel(int F, BvhWs w) {
  const int b = blockIdx.y;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= F - 1) return;
  const unsigned *codes = w.codes + (size_t)b * F;
  const int *ids = w.ids + (size_t)b * F;
  int *parent = w.parent + (size_t)b * (2 * F - 1);
  BvhNode *nodes = w.nodes + (size_t)b * (F - 1);
  int d_next = lcp(codes, ids, F, idx, idx + 1), d_last = lcp(codes, ids, F, idx, idx - 1);
  int dir = d_next - d_last >= 0 ? 1 : -1;
  int d_min = lcp(codes, ids, F, idx, idx - dir);
  int lmax = 2;
  while (lcp(codes, ids, F, idx, idx + lmax * dir) > d_min) lmax *= 2;
  int l = 0;
  for (int t = lmax >> 1; t >= 1; t >>= 1)
    if (lcp(codes, ids, F, idx, idx + (l + t) * dir) > d_min) l += t;
  const int j = idx + l * dir;
  const int d_node = lcp(codes, ids, F, idx, j);
  // split position: largest s with lcp(idx, idx + s*dir) > d_node.  (The reference's search loop,
  // op.cu:735-744, re-tests its first step and then walks in unit steps; it lands on the same s.)
  int s = 0, t = l;
  do {
    t = (t + 1) >> 1;
    if (lcp(codes, ids, F, idx, idx + (s + t) * dir) > d_node) s += t;
  } while (t > 1);
  int split = idx + s * dir + min(dir, 0);
  int left, right;
  if (min(idx, j) == split) { left = ~split; parent[F - 1 + split] = idx; }
  else { left = split; parent[split] = idx; }
  if (max(idx, j) == split + 1) { right = ~(split + 1); parent[F - 1 + split + 1] = idx; }
  else { right = split + 1; parent[split + 1] = idx; }
  nodes[idx].left = left;
  nodes[idx].right = right;
  if (idx == 0) parent[0] = -1;
}

__device__ __forceinline__ void child_box(const BvhWs &w, size_t b, int F, int link, float *o) {
  if (link < 0) {
    const float *lb = w.leaf_box + (b * F + (size_t)(~link)) * 6;
    for (int c = 0; c < 6; ++c) o[c] = lb[c];
  } else {
    const volatile BvhNode *n = w.nodes + b * (F - 1) + link;
    o[0] = n->lo[0]; o[1] = n->lo[1]; o[2] = n->lo[2]; o[3] = n->hi[0]; o[4] = n->hi[1]; o[5] = n->hi[2];
  }
}

__global__ void bvh_refit_kernel(int F, BvhWs w) {
  const int b = blockIdx.y;
  const int leaf = blockIdx.x * blockDim.x + threadIdx.x;
  if (leaf >= F) return;
  const int *parent = w.parent + (size_t)b * (2 * F - 1);
  int *counters = w.counters + (size_t)b * (F - 1);
  BvhNode *nodes = w.nodes + (size_t)b * (F - 1);
  int cur = parent[F - 1 + leaf];
  while (cur >= 0) {
    if (atomicAdd(counters + cur, 1) == 0) return;  // first visitor stops, second one has both children
    __threadfence();
    float a[6], c[6];
    child_box(w, b, F, nodes[cur].left, a);
    child_box(w, b, F, nodes[cur].right, c);
    for (int k = 0; k < 3; ++k) { nodes[cur].lo[k] = fminf(a[k], c[k]); nodes[cur].hi[k] = fmaxf(a[3 + k], c[3 + k]); }
    __threadfence();
    cur = parent[cur];
  }
}

constexpr int kStackCap = 1024;  // per warp
constexpr int kQueueCap = 96;

__device__ __forceinline__ bool overlap6(const mmi::Box &q, const float *bx) {
  return (q.lo.x <= bx[3]) && (q.hi.x >= bx[0]) && (q.lo.y <= bx[4]) && (q.hi.y >= bx[1]) && (q.lo.z <= bx[5]) &&
         (q.hi.z >= bx[2]);
}

// 4 warps per CTA, one query triangle per warp.
template <typename T>
__global__ void __launch_bounds__(128) bvh_query_kernel(const T *__restrict__ query, const T *__restrict__ target,
                                                        int Q, int F, int M, BvhWs w, long long *faces_out,
                                                        T *bcs_out) {
  __shared__ int stack[4][kStackCap];
  __shared__ int queue[4][kQueueCap];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned lt_mask = (1u << lane) - 1;
  const int b = blockIdx.y;
  const int qi = blockIdx.x * 4 + warp;
  if (qi >= Q) return;
  const mmi::TriT<T> qt = ld_tri(query + ((size_t)b * Q + qi) * 9);
  const mmi::BoxT<T> qbox = mmi::tri_box(qt);
  const mmi::Box qb = mmi::box_f32(qbox);
  const T *tb = target + (size_t)b * F * 9;
  const int *ids = w.ids + (size_t)b * F;
  const BvhNode *nodes = w.nodes + (size_t)b * (F - 1);
  long long *fo = faces_out + ((size_t)b * Q + qi) * M;
  T *bo = bcs_out + ((size_t)b * Q + qi) * M * 6;
  int *st = stack[warp], *qu = queue[warp];
  int sp = 0, qn = 0, nhit = 0;
  if (F == 1) {  // a single leaf, no internal node
    if (lane == 0) qu[0] = 0;
    qn = 1;
  } else {
    if (lane == 0) st[0] = 0;
    sp = 1;
  }
  __syncwarp();
  while (sp > 0 || qn > 0) {
    if (qn >= 32 || sp == 0) {
      // ---- narrow phase: 32 queued leaves, one per lane, exact reference predicates
      const int n = min(qn, 32);
      const int cand = lane < n ? qu[qn - n + lane] : -1;
      __syncwarp();
      qn -= n;
      bool hit = false;
      mmi::vec3<T> b1{0, 0, 0}, b2 = b1;
      int tid = -1;
      if (cand >= 0) {
        tid = ids[cand];
        const mmi::TriT<T> tt = ld_tri(tb + (size_t)tid * 9);
        // float leaf boxes are the exact AABBs; double ones were rounded outward, so repeat the exact test
        if constexpr (sizeof(T) == 4) hit = mmi::sat11(qt, tt);
        else hit = mmi::box_overlap(qbox, mmi::tri_box(tt)) && mmi::sat11(qt, tt);
        if (hit) mmi::isect_points(qt, tt, b1, b2);
      }
      const unsigned mh = __ballot_sync(0xffffffffu, hit);
      if (hit) {
        const int slot = nhit + __popc(mh & lt_mask);
        if (slot < M) {
          fo[slot] = tid;
          T *o = bo + (size_t)slot * 6;
          o[0] = b1.x; o[1] = b1.y; o[2] = b1.z; o[3] = b2.x; o[4] = b2.y; o[5] = b2.z;
        }
      }
      nhit += __popc(mh);
      continue;
    }
    // ---- broad phase: pop up to 32 internal nodes (1 when the stack is nearly full: depth-first, so it
    //      can only grow by the tree depth), test both children of each against the query AABB
    const int take = sp > kStackCap - 128 ? 1 : min(sp, 32);
    const int node = lane < take ? st[sp - take + lane] : -1;
    __syncwarp();
    sp -= take;
    int link[2] = {0, 0};
    bool ov[2] = {false, false};
    if (node >= 0) {
      link[0] = nodes[node].left; link[1] = nodes[node].right;
      float bx[6];
      child_box(w, (size_t)b, F, link[0], bx); ov[0] = overlap6(qb, bx);
      child_box(w, (size_t)b, F, link[1], bx); ov[1] = overlap6(qb, bx);
    }
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const bool push = ov[c] && link[c] >= 0;
      const unsigned mp = __ballot_sync(0xffffffffu, push);
      if (push) st[sp + __popc(mp & lt_mask)] = link[c];
      sp += __popc(mp);
      const bool leaf = ov[c] && link[c] < 0;
      const unsigned ml = __ballot_sync(0xffffffffu, leaf);
      if (leaf) qu[qn + __popc(ml & lt_mask)] = ~link[c];
      qn += __popc(ml);
    }
    __syncwarp();
  }
}

__global__ void fill_i64_kernel(long long *p, size_t n, long long v) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

}  // namespace shapy

using namespace shapy;

extern "C" size_t shapy_mmi_workspace_bytes(int B, int Q, int F) {
  (void)Q;
  if (B <= 0 || F <= 0) return 0;
  return ws_layout(B, F, nullptr, nullptr) + 256;
}

// The workspace holds float boxes and int links whatever the triangles' scalar type.
extern "C" size_t shapy_mmi_workspace_bytes_f64(int B, int Q, int F) { return shapy_mmi_workspace_bytes(B, Q, F); }

template <typename T>
static int mmi_forward(const char *name, const T *query, const T *target, int B, int Q, int F, int M,
                       int64_t *collision_faces, T *collision_bcs, void *workspace, size_t workspace_bytes,
                       void *stream) {
  SHAPY_REQUIRE(query && target && collision_faces && collision_bcs, "%s: null argument", name);
  SHAPY_REQUIRE(B > 0 && Q > 0 && F > 0 && M > 0, "%s: bad sizes", name);
  SHAPY_REQUIRE(workspace && workspace_bytes >= shapy_mmi_workspace_bytes(B, Q, F), "%s: workspace too small", name);
  cudaStream_t st = (cudaStream_t)stream;
  int npow2 = 1;
  while (npow2 < F) npow2 <<= 1;
  if (npow2 > 32768) {
    set_error("%s: %d target triangles exceed the 32768 supported by the shared-memory sort", name, F);
    return SHAPY_ERR_UNSUPPORTED;
  }
  BvhWs w;
  char *base = (char *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  ws_layout(B, F, &w, base);
  const size_t n_slots = (size_t)B * Q * M;
  fill_i64_kernel<<<(unsigned)((n_slots + 255) / 256), 256, 0, st>>>((long long *)collision_faces, n_slots, -1);
  SHAPY_LAUNCH_CHECK();
  SHAPY_CUDA_TRY(cudaMemsetAsync(collision_bcs, 0, n_slots * 6 * sizeof(T), st));
  const size_t smem = (size_t)npow2 * 4 + (size_t)npow2 * 2;
  static std::atomic<unsigned long long> attr_done{0};
  SHAPY_CUDA_TRY(set_max_dynamic_smem(bvh_prepare_kernel<T, unsigned short>, 200 * 1024, attr_done));
  bvh_prepare_kernel<T, unsigned short><<<B, 1024, smem, st>>>(target, F, npow2, w);
  SHAPY_LAUNCH_CHECK();
  if (F > 1) {
    dim3 g1(ceil_div(F - 1, 128), B);
    bvh_topology_kernel<<<g1, 128, 0, st>>>(F, w);
    SHAPY_LAUNCH_CHECK();
    dim3 g2(ceil_div(F, 128), B);
    bvh_refit_kernel<<<g2, 128, 0, st>>>(F, w);
    SHAPY_LAUNCH_CHECK();
  }
  dim3 g3(ceil_div(Q, 4), B);
  bvh_query_kernel<T><<<g3, 128, 0, st>>>(query, target, Q, F, M, w, (long long *)collision_faces, collision_bcs);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_mmi_forward(const float *query, const float *target, int B, int Q, int F, int M,
                                 int64_t *collision_faces, float *collision_bcs, void *workspace,
                                 size_t workspace_bytes, void *stream) {
  return mmi_forward("shapy_mmi_forward", query, target, B, Q, F, M, collision_faces, collision_bcs, workspace,
                     workspace_bytes, stream);
}

extern "C" int shapy_mmi_forward_f64(const double *query, const double *target, int B, int Q, int F, int M,
                                     int64_t *collision_faces, double *collision_bcs, void *workspace,
                                     size_t workspace_bytes, void *stream) {
  return mmi_forward("shapy_mmi_forward_f64", query, target, B, Q, F, M, collision_faces, collision_bcs, workspace,
                     workspace_bytes, stream);
}
