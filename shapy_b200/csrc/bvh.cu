// Batched LBVH mesh-mesh intersection: drop-in for mesh_mesh_intersect_cuda.mesh_to_mesh_forward
// (reference mesh-mesh-intersection/src/mesh_mesh_intersect.cpp:36-64 and
//  src/mesh_mesh_intersect_cuda_op.cu:969-1079), all bodies of the batch in the same launches, on the
// caller's stream, no host synchronisation, no allocation.  The same tree serves the scan queries at the end of the
// file (closest points on posed meshes, nearest scan points, and the scan distance's backward).
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

// ================================================================================================ scans
// Closest points of scan points on a batch of posed meshes, the nearest scan point of each model vertex, and the
// backward of the scan -> model squared distance.  Both queries run on the LBVH above (bvh_prepare_kernel,
// bvh_topology_kernel, bvh_refit_kernel), built over a float triangle soup in the workspace: the posed triangles
// gathered from (vertices, faces), or the scan points as degenerate triangles (p, p, p).
//
//   scan_mesh_soup_kernel / scan_point_soup_kernel   the primitives of each body, [B][P][9]
//   scan_leaf_boxes_kernel    refit only: the leaf boxes of a tree built by an earlier call, from the new soup
//   scan_query_kernel<kPts>   ONE THREAD PER QUERY, nearer child first, a 64-entry (node, box distance) stack
//   scan_backward_kernel      ONE CTA PER BODY: bitonic sort of the (face, point) pairs in shared memory, then one
//                             thread per vertex gathers over its incident faces (CSR order) and their points (index
//                             order)
//
// The result is a function of the primitives and the queries only, not of the tree: a box is pruned only when its
// computed squared distance exceeds prune_bound of the current best, which is proved below to exceed the box distance
// of every primitive whose computed squared distance is <= best, and a candidate wins on a strictly smaller squared
// distance or on an equal one with a smaller primitive index.  So every primitive that could win is evaluated, and the
// winner is the lexicographic minimum of (float squared distance, index) over all of them, whatever the tree's shape
// (tests/bvh_f32_oracle.py restates it).
namespace shapy {

constexpr int kScanMaxPrims = 32768;  // the shared-memory sorts of bvh_prepare_kernel and scan_backward_kernel
// A root-to-leaf path splits at strictly increasing prefix lengths of the (30-bit Morton code, 15-bit id) key, so
// the tree is at most 45 internal nodes deep and the stack never holds more than 45 entries.
constexpr int kScanStack = 64;

struct ScanWs {
  float *soup;  // [B][P][9]
  BvhWs bvh;
};

static size_t scan_ws_layout(int B, int P, ScanWs *w, char *base) {
  const size_t soup = align_up((size_t)B * P * 9 * 4, 256);
  if (w) w->soup = (float *)base;
  return soup + ws_layout(B, P, w ? &w->bvh : nullptr, base ? base + soup : nullptr);
}

__global__ void scan_mesh_soup_kernel(const float *__restrict__ vertices, const int *__restrict__ faces, int V, int F,
                                      size_t n, float *__restrict__ soup) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // corner of [B][F][3]
  if (i >= n) return;
  const size_t bf = i / 3;
  const int b = (int)(bf / F), f = (int)(bf % F), k = (int)(i % 3);
  const float *s = vertices + ((size_t)b * V + faces[f * 3 + k]) * 3;
  float *d = soup + i * 3;
  d[0] = s[0]; d[1] = s[1]; d[2] = s[2];
}

// a point with weight <= 0 is never read: it goes in at the origin and the query skips it
__global__ void scan_point_soup_kernel(const float *__restrict__ points, const float *__restrict__ weights, size_t n,
                                       float *__restrict__ soup) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const bool keep = !weights || weights[i] > 0.f;
  const float x = keep ? points[i * 3] : 0.f, y = keep ? points[i * 3 + 1] : 0.f, z = keep ? points[i * 3 + 2] : 0.f;
  float *d = soup + i * 9;
  for (int c = 0; c < 3; ++c) { d[3 * c] = x; d[3 * c + 1] = y; d[3 * c + 2] = z; }
}

__global__ void scan_leaf_boxes_kernel(const float *__restrict__ soup, int P, BvhWs w) {
  const int b = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P) return;
  const int id = w.ids[(size_t)b * P + j];
  const mmi::Box bx = mmi::box_f32(mmi::tri_box(ld_tri(soup + ((size_t)b * P + id) * 9)));
  float *lb = w.leaf_box + ((size_t)b * P + j) * 6;
  lb[0] = bx.lo.x; lb[1] = bx.lo.y; lb[2] = bx.lo.z; lb[3] = bx.hi.x; lb[4] = bx.hi.y; lb[5] = bx.hi.z;
  if (j < P - 1) w.counters[(size_t)b * (P - 1) + j] = 0;
}

__device__ __forceinline__ float3 sub3(float3 a, float3 b) { return make_float3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// The Voronoi-region test of a non-degenerate triangle (a, b, c): the closest point of p is a + v ab + w ac.  Returns
// false when the interior's denominator is not positive (a triangle too thin for the test) or rounding put p's
// projection outside the triangle, true otherwise; then v, w >= 0 and v + w <= 1 + 4u.
__device__ __forceinline__ bool tri_region(float3 ab, float3 ac, float3 ap, float3 bp, float3 cp, float &v, float &w) {
  const float d1 = dot3(ab, ap), d2 = dot3(ac, ap);
  if (d1 <= 0.f && d2 <= 0.f) { v = 0.f; w = 0.f; return true; }  // vertex a
  const float d3 = dot3(ab, bp), d4 = dot3(ac, bp);
  if (d3 >= 0.f && d4 <= d3) { v = 1.f; w = 0.f; return true; }  // vertex b
  const float d5 = dot3(ab, cp), d6 = dot3(ac, cp);
  if (d6 >= 0.f && d5 <= d6) { v = 0.f; w = 1.f; return true; }  // vertex c
  const float vc = d1 * d4 - d3 * d2;
  if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) { v = d1 - d3 > 0.f ? d1 / (d1 - d3) : 0.f; w = 0.f; return true; }  // ab
  const float vb = d5 * d2 - d1 * d6;
  if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) { v = 0.f; w = d2 - d6 > 0.f ? d2 / (d2 - d6) : 0.f; return true; }  // ac
  const float va = d3 * d6 - d5 * d4;
  const float e1 = d4 - d3, e2 = d5 - d6;
  if (va <= 0.f && e1 >= 0.f && e2 >= 0.f) {  // bc
    w = e1 + e2 > 0.f ? e1 / (e1 + e2) : 0.f;
    v = 1.f - w;
    return true;
  }
  const float den = va + vb + vc;  // interior
  // Rounding can reach here with p's projection outside the triangle (a negative va, vb or vc near a region's
  // border); the edges then give the closest point, so (v, w) stays in the triangle (see prune_bound).
  if (!(den > 0.f && va >= 0.f && vb >= 0.f && vc >= 0.f)) return false;
  v = vb / den;
  w = vc / den;
  return true;
}

__device__ __forceinline__ float seg_t(float3 ap, float3 ab) {
  const float l2 = dot3(ab, ab);
  return l2 > 0.f ? fminf(fmaxf(dot3(ap, ab) / l2, 0.f), 1.f) : 0.f;
}

__device__ __forceinline__ float tri_d2(float3 ab, float3 ac, float3 ap, float v, float w) {
  const float3 d = make_float3(ap.x - (ab.x * v + ac.x * w), ap.y - (ab.y * v + ac.y * w), ap.z - (ab.z * v + ac.z * w));
  return dot3(d, d);
}

// Exact closest point of p on the triangle (a, b, c): squared distance, barycentrics (1 - v - w, v, w).  A zero-area
// (or too thin) triangle is the nearest of its edges ab, ac, bc, the first of them on a tie.
__device__ __forceinline__ float point_triangle(float3 p, float3 a, float3 b, float3 c, float &v, float &w) {
  const float3 ab = sub3(b, a), ac = sub3(c, a), ap = sub3(p, a);
  const float3 n = make_float3(ab.y * ac.z - ab.z * ac.y, ab.z * ac.x - ab.x * ac.z, ab.x * ac.y - ab.y * ac.x);
  if (dot3(n, n) > 0.f && tri_region(ab, ac, ap, sub3(p, b), sub3(p, c), v, w)) return tri_d2(ab, ac, ap, v, w);
  const float t0 = seg_t(ap, ab), t1 = seg_t(ap, ac), t2 = seg_t(sub3(p, b), sub3(c, b));
  float bv = t0, bw = 0.f, best = tri_d2(ab, ac, ap, t0, 0.f);
  const float e1 = tri_d2(ab, ac, ap, 0.f, t1);
  if (e1 < best) { best = e1; bv = 0.f; bw = t1; }
  const float e2 = tri_d2(ab, ac, ap, 1.f - t2, t2);
  if (e2 < best) { best = e2; bv = 1.f - t2; bw = t2; }
  v = bv;
  w = bw;
  return best;
}

__device__ __forceinline__ float box_d2(float3 p, const float *bx) {
  const float dx = fmaxf(fmaxf(bx[0] - p.x, p.x - bx[3]), 0.f);
  const float dy = fmaxf(fmaxf(bx[1] - p.y, p.y - bx[4]), 0.f);
  const float dz = fmaxf(fmaxf(bx[2] - p.z, p.z - bx[5]), 0.f);
  return dx * dx + dy * dy + dz * dz;
}

// the box of a child link of a finished tree (the refit's volatile reads are not needed once it has ended)
__device__ __forceinline__ float scan_child_box_d2(const BvhNode *nodes, const float *leaf_box, int link, float3 p) {
  const float *s = link < 0 ? leaf_box + (size_t)(~link) * 6 : nodes[link].lo;
  float bx[6];
  for (int c = 0; c < 6; ++c) bx[c] = __ldg(s + c);
  return box_d2(p, bx);
}

// The largest box distance that can still hold a primitive as near as `best`.
//
// Points: box_d2 of a point's leaf box is the same operations as its d2, so it rounds to the same value, and a node's
// box contains its children's, so its box_d2 is no larger (every operation of box_d2 is monotone).  Any bound >= best
// is exact; the relative one below keeps the points query's bits.
__device__ __forceinline__ float relative_prune_bound(float best) { return best + best * 1e-5f + 1e-12f; }

// Triangles: prune_bound(best, M) = (sqrt(best) + k u M)^2, u = 2^-24, k = 64, M the largest coordinate magnitude of
// the query and the body's scene box (the root's box), so that every coordinate of p, a, b, c is <= M.  Claim: for
// every leaf, with d2 = point_triangle(p, a, b, c) and b2 = box_d2(p, leaf box) as computed,
// b2 <= prune_bound(d2, M).  Both sides are monotone in their argument (node boxes contain leaf boxes; sqrtf, + and *
// round monotonically), so a leaf as near as `best`, and every node above it, is visited.  Proof, to first order in u
// (the k chosen leaves the O(u^2) terms far below the margin), with |x| the Euclidean norm:
//  1. tri_region and the edge fallback return v, w >= 0, v + w <= 1 + 4u.  So X = a + (b - a) v + (c - a) w lies
//     within 4u |b - a, c - a| <= 4u 2 sqrt(3) M < 14u M of the triangle, whose points lie in the leaf box:
//     D := the exact distance of p to the box <= |p - X| + 14u M.
//  2. tri_d2's vector differs from p - X, per coordinate, by the rounding of ap (2u M), of ab and ac times v, w
//     (2u M (v + w)), of the products and their sum (2 2u M (v + w)) and of the difference (u |d|): in norm by at
//     most sqrt(3) 8u M + u |d| < 14u M + u |d|.  dot3 of a vector rounds its square down by at most (1 - u)^3.
//     So s := sqrt(d2) >= (1 - 2.5u) |p - X| - 14u M.
//  3. box_d2 rounds each of its 3 + 3 + 2 operations up by at most (1 + u): sqrt(b2) <= (1 + 2.5u) D.
//  4. Then sqrt(b2) <= (1 + 5u) s + 28u M + 5u (14u M), and s <= |p - X| <= 2 sqrt(3) M (1 + 4u): 5u s <= 18u M,
//     so sqrt(b2) <= s + 46u M.
//  5. The bound as computed, fl(fl(fl(sqrt(d2)) + M ku)^2), is >= (s + 64u M)^2 (1 - u)^5: sqrtf and the add each
//     round r down by at most (1 - u), squared, and the square rounds once more.  That is >= (s + 46u M)^2, as
//     2.5u (s + 64u M) <= 18u M for s <= 7.2 M - 64u M, and s <= 3.5 M.  (M ku is exact: ku = 2^-18.)
// The bound is a function of the query and its body only, so results stay independent of the batch.
constexpr float kPruneSlack = 0x1p-18f;  // k u
__device__ __forceinline__ float prune_bound(float best, float M) {
  const float r = sqrtf(best) + M * kPruneSlack;
  return r * r;
}

// One thread per query point q of body blockIdx.y against the P primitives of that body's tree.  kPts: the
// primitives are points (soup (p, p, p)), d2 = |q - p|^2 and a primitive with prim_w <= 0 is skipped; otherwise they
// are triangles and a query with q_w <= 0 is not read (out -1, zero barycentrics and distance).
template <bool kPts>
__global__ void __launch_bounds__(128) scan_query_kernel(const float *__restrict__ queries, const float *__restrict__ q_w,
                                                         int Q, const float *__restrict__ soup,
                                                         const float *__restrict__ prim_w, int P, BvhWs w,
                                                         int *__restrict__ idx_out, float *__restrict__ bary_out,
                                                         float *__restrict__ d2_out) {
  const int b = blockIdx.y;
  const int qi = blockIdx.x * blockDim.x + threadIdx.x;
  if (qi >= Q) return;
  const size_t o = (size_t)b * Q + qi;
  float best = INFINITY, lim = INFINITY, bv = 0.f, bw = 0.f;  // lim: the prune bound of best
  int best_id = -1;
  if (kPts || !q_w || q_w[o] > 0.f) {
    const float3 q = make_float3(queries[o * 3], queries[o * 3 + 1], queries[o * 3 + 2]);
    const float *sb = soup + (size_t)b * P * 9;
    const int *ids = w.ids + (size_t)b * P;
    const BvhNode *nodes = w.nodes + (size_t)b * (P - 1);
    const float *leaf_box = w.leaf_box + (size_t)b * P * 6;
    float M = fmaxf(fmaxf(fabsf(q.x), fabsf(q.y)), fabsf(q.z));
    if (!kPts) {
      const float *root = P == 1 ? leaf_box : nodes[0].lo;
      for (int c = 0; c < 6; ++c) M = fmaxf(M, fabsf(__ldg(root + c)));
    }
    auto leaf = [&](int j) {
      const int id = __ldg(ids + j);
      const float *t = sb + (size_t)id * 9;
      float d2, v = 0.f, ww = 0.f;
      if constexpr (kPts) {
        if (prim_w && !(prim_w[(size_t)b * P + id] > 0.f)) return;
        const float3 d = sub3(q, make_float3(t[0], t[1], t[2]));
        d2 = dot3(d, d);
      } else {
        d2 = point_triangle(q, make_float3(t[0], t[1], t[2]), make_float3(t[3], t[4], t[5]),
                            make_float3(t[6], t[7], t[8]), v, ww);
      }
      if (d2 < best || (d2 == best && id < best_id)) {
        best = d2; best_id = id; bv = v; bw = ww;
        lim = kPts ? relative_prune_bound(best) : prune_bound(best, M);
      }
    };
    if (P == 1) {
      leaf(0);
    } else {
      int st_node[kScanStack];
      float st_d[kScanStack];
      int sp = 0, node = 0;
      while (true) {
        const int link[2] = {__ldg(&nodes[node].left), __ldg(&nodes[node].right)};
        const float d[2] = {scan_child_box_d2(nodes, leaf_box, link[0], q), scan_child_box_d2(nodes, leaf_box, link[1], q)};
        for (int c = 0; c < 2; ++c)
          if (link[c] < 0 && d[c] <= lim) leaf(~link[c]);
        const bool go0 = link[0] >= 0 && d[0] <= lim, go1 = link[1] >= 0 && d[1] <= lim;
        if (go0 && go1) {
          const int near = d[1] < d[0] ? 1 : 0;
          st_node[sp] = link[1 - near];
          st_d[sp] = d[1 - near];
          ++sp;
          node = link[near];
        } else if (go0 || go1) {
          node = link[go0 ? 0 : 1];
        } else {
          node = -1;
          while (sp > 0) {
            --sp;
            if (st_d[sp] <= lim) { node = st_node[sp]; break; }
          }
          if (node < 0) break;
        }
      }
    }
  }
  idx_out[o] = best_id;
  d2_out[o] = best_id >= 0 ? best : 0.f;
  if (!kPts) {
    const bool hit = best_id >= 0;
    bary_out[o * 3] = hit ? 1.f - bv - bw : 0.f;
    bary_out[o * 3 + 1] = hit ? bv : 0.f;
    bary_out[o * 3 + 2] = hit ? bw : 0.f;
  }
}

// One CTA per body.  Dynamic smem: keys[npow2] (face, u32) + ids[npow2] (point, u16).  A point with a face outside
// [0, F) (weight <= 0: -1) sorts last with key 0xFFFFFFFF and adds nothing.
__global__ void __launch_bounds__(1024) scan_backward_kernel(
    const float *__restrict__ vertices, const int *__restrict__ faces, const int *__restrict__ inc_ptr,
    const int *__restrict__ inc, int V, int F, const float *__restrict__ points, int N, int npow2,
    const int *__restrict__ face_idx, const float *__restrict__ bary, const float *__restrict__ grad,
    float *__restrict__ grad_v) {
  extern __shared__ __align__(16) unsigned char sm[];
  unsigned *keys = reinterpret_cast<unsigned *>(sm);
  unsigned short *ids = reinterpret_cast<unsigned short *>(sm + (size_t)npow2 * 4);
  const int b = blockIdx.x, t = threadIdx.x;
  for (int i = t; i < npow2; i += blockDim.x) {
    const int f = i < N ? face_idx[(size_t)b * N + i] : -1;
    keys[i] = f >= 0 && f < F ? (unsigned)f : 0xFFFFFFFFu;
    ids[i] = (unsigned short)i;
  }
  __syncthreads();
  for (int k = 2; k <= npow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = t; i < npow2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned ca = keys[i], cb = keys[ixj];
          const unsigned short ia = ids[i], ib = ids[ixj];
          const bool a_gt_b = ca > cb || (ca == cb && ia > ib);
          if (a_gt_b == ((i & k) == 0)) { keys[i] = cb; keys[ixj] = ca; ids[i] = ib; ids[ixj] = ia; }
        }
      }
      __syncthreads();
    }
  }
  const float *vb = vertices + (size_t)b * V * 3;
  const float *pb = points + (size_t)b * N * 3;
  const float *cb = bary + (size_t)b * N * 3;
  const float *gb = grad + (size_t)b * N;
  for (int v = t; v < V; v += blockDim.x) {
    float g[3] = {0.f, 0.f, 0.f};
    for (int e = inc_ptr[v]; e < inc_ptr[v + 1]; ++e) {
      const int f = inc[e] / 3, corner = inc[e] - 3 * f;
      int lo = 0, hi = npow2;  // first key >= f
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < (unsigned)f) lo = mid + 1; else hi = mid;
      }
      if (lo == npow2 || keys[lo] != (unsigned)f) continue;
      const float *x0 = vb + (size_t)faces[f * 3] * 3, *x1 = vb + (size_t)faces[f * 3 + 1] * 3,
                  *x2 = vb + (size_t)faces[f * 3 + 2] * 3;
      for (int i = lo; i < npow2 && keys[i] == (unsigned)f; ++i) {
        const int p = ids[i];
        const float *l = cb + (size_t)p * 3;
        const float s = 2.f * gb[p] * l[corner];
        for (int c = 0; c < 3; ++c) g[c] += s * ((l[0] * x0[c] + l[1] * x1[c] + l[2] * x2[c]) - pb[(size_t)p * 3 + c]);
      }
    }
    float *o = grad_v + ((size_t)b * V + v) * 3;
    o[0] = g[0]; o[1] = g[1]; o[2] = g[2];
  }
}

static int npow2_of(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

// Builds the tree over w.soup (P primitives per body), or with refit only recomputes its boxes.
static int scan_tree(const ScanWs &w, int B, int P, bool refit, cudaStream_t st) {
  if (refit) {
    scan_leaf_boxes_kernel<<<dim3(ceil_div(P, 128), B), 128, 0, st>>>(w.soup, P, w.bvh);
    SHAPY_LAUNCH_CHECK();
  } else {
    const int npow2 = npow2_of(P);
    static std::atomic<unsigned long long> attr_done{0};
    SHAPY_CUDA_TRY(set_max_dynamic_smem(bvh_prepare_kernel<float, unsigned short>, 200 * 1024, attr_done));
    bvh_prepare_kernel<float, unsigned short><<<B, 1024, (size_t)npow2 * 6, st>>>(w.soup, P, npow2, w.bvh);
    SHAPY_LAUNCH_CHECK();
    if (P > 1) {
      bvh_topology_kernel<<<dim3(ceil_div(P - 1, 128), B), 128, 0, st>>>(P, w.bvh);
      SHAPY_LAUNCH_CHECK();
    }
  }
  if (P > 1) {
    bvh_refit_kernel<<<dim3(ceil_div(P, 128), B), 128, 0, st>>>(P, w.bvh);
    SHAPY_LAUNCH_CHECK();
  }
  return SHAPY_OK;
}

static int scan_limit(const char *name, const char *what, int n) {
  if (n <= kScanMaxPrims) return SHAPY_OK;
  set_error("%s: %d %s per body exceed the %d supported (the tree and the backward sort them in shared memory)", name,
            n, what, kScanMaxPrims);
  return SHAPY_ERR_UNSUPPORTED;
}

static char *scan_base(void *workspace) { return (char *)(((uintptr_t)workspace + 255) & ~(uintptr_t)255); }

}  // namespace shapy

extern "C" size_t shapy_closest_points_workspace_bytes(int B, int F) {
  if (B <= 0 || F <= 0) return 0;
  return scan_ws_layout(B, F, nullptr, nullptr) + 256;
}

extern "C" int shapy_closest_points(const float *vertices, const int32_t *faces, int B, int V, int F,
                                    const float *points, int N, const float *weights, int refit, int32_t *face_idx,
                                    float *bary, float *sq_dist, void *workspace, size_t workspace_bytes,
                                    void *stream) {
  const char *name = "shapy_closest_points";
  SHAPY_REQUIRE(B >= 0 && N >= 0 && V > 0 && F > 0, "%s: bad sizes", name);
  if (int rc = scan_limit(name, "faces", F)) return rc;
  if (int rc = scan_limit(name, "points", N)) return rc;
  if (B == 0 || N == 0) return SHAPY_OK;
  SHAPY_REQUIRE(vertices && faces && points && face_idx && bary && sq_dist, "%s: null argument", name);
  SHAPY_REQUIRE(workspace && workspace_bytes >= shapy_closest_points_workspace_bytes(B, F), "%s: workspace too small",
                name);
  cudaStream_t st = (cudaStream_t)stream;
  ScanWs w;
  scan_ws_layout(B, F, &w, scan_base(workspace));
  const size_t n = (size_t)B * F * 3;
  scan_mesh_soup_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(vertices, faces, V, F, n, w.soup);
  SHAPY_LAUNCH_CHECK();
  if (int rc = scan_tree(w, B, F, refit != 0, st)) return rc;
  scan_query_kernel<false><<<dim3(ceil_div(N, 128), B), 128, 0, st>>>(points, weights, N, w.soup, nullptr, F, w.bvh,
                                                                       face_idx, bary, sq_dist);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" size_t shapy_nearest_points_workspace_bytes(int B, int N) { return shapy_closest_points_workspace_bytes(B, N); }

extern "C" int shapy_nearest_points(const float *queries, int B, int Q, const float *points, int N,
                                    const float *weights, int32_t *idx, float *sq_dist, void *workspace,
                                    size_t workspace_bytes, void *stream) {
  const char *name = "shapy_nearest_points";
  SHAPY_REQUIRE(B >= 0 && Q >= 0 && N > 0, "%s: bad sizes", name);
  if (int rc = scan_limit(name, "points", N)) return rc;
  if (B == 0 || Q == 0) return SHAPY_OK;
  SHAPY_REQUIRE(queries && points && idx && sq_dist, "%s: null argument", name);
  SHAPY_REQUIRE(workspace && workspace_bytes >= shapy_nearest_points_workspace_bytes(B, N), "%s: workspace too small",
                name);
  cudaStream_t st = (cudaStream_t)stream;
  ScanWs w;
  scan_ws_layout(B, N, &w, scan_base(workspace));
  const size_t n = (size_t)B * N;
  scan_point_soup_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(points, weights, n, w.soup);
  SHAPY_LAUNCH_CHECK();
  if (int rc = scan_tree(w, B, N, false, st)) return rc;
  scan_query_kernel<true><<<dim3(ceil_div(Q, 128), B), 128, 0, st>>>(queries, nullptr, Q, w.soup, weights, N, w.bvh,
                                                                      idx, nullptr, sq_dist);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

extern "C" int shapy_closest_points_backward(const float *vertices, const int32_t *faces, const int32_t *inc_ptr,
                                             const int32_t *inc, int B, int V, int F, const float *points, int N,
                                             const int32_t *face_idx, const float *bary, const float *grad_sq_dist,
                                             float *grad_vertices, void *stream) {
  const char *name = "shapy_closest_points_backward";
  SHAPY_REQUIRE(B >= 0 && N >= 0 && V > 0 && F > 0, "%s: bad sizes", name);
  if (int rc = scan_limit(name, "faces", F)) return rc;
  if (int rc = scan_limit(name, "points", N)) return rc;
  if (B == 0) return SHAPY_OK;
  SHAPY_REQUIRE(vertices && faces && inc_ptr && inc && grad_vertices, "%s: null argument", name);
  cudaStream_t st = (cudaStream_t)stream;
  if (N == 0) {
    SHAPY_CUDA_TRY(cudaMemsetAsync(grad_vertices, 0, (size_t)B * V * 3 * sizeof(float), st));
    return SHAPY_OK;
  }
  SHAPY_REQUIRE(points && face_idx && bary && grad_sq_dist, "%s: null argument", name);
  const int npow2 = npow2_of(N);
  static std::atomic<unsigned long long> attr_done{0};
  SHAPY_CUDA_TRY(set_max_dynamic_smem(scan_backward_kernel, 200 * 1024, attr_done));
  scan_backward_kernel<<<B, 1024, (size_t)npow2 * 6, st>>>(vertices, faces, inc_ptr, inc, V, F, points, N, npow2,
                                                           face_idx, bary, grad_sq_dist, grad_vertices);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// ======================================================================================================= self-collisions
// Intersecting face pairs (f, g), f < g, of each posed mesh on the scan tree above (the soup of shapy_closest_points):
//   self_face_kernel<false>  ONE THREAD PER FACE f: counts the faces g > f whose leaf box overlaps f's and that pass
//                            self_pair
//   self_scan_kernel    ONE CTA PER BODY: exclusive scan of the per-face counts -> each face's first output row
//   self_face_kernel<true>   ONE THREAD PER FACE: the face's pairs in increasing g, each traversal keeping the kSelfSel
//                       smallest g past the last one written, for as many rows as are left below max_pairs
// A pair is a function of the two triangles, the faces and the part filter only, so the rows do not depend on the
// tree's shape or on the rest of the batch, and every sum is over integers.
namespace shapy {

constexpr int kSelfSel = 8;

// Visits every leaf whose box overlaps qb (inclusive test), depth first.
template <typename Fn>
__device__ __forceinline__ void box_traverse(const BvhNode *nodes, const float *leaf_box, int P, const mmi::Box &qb,
                                             Fn &&leaf) {
  if (P == 1) {
    if (overlap6(qb, leaf_box)) leaf(0);
    return;
  }
  int st[kScanStack];
  int sp = 0, node = 0;
  while (true) {
    const int link[2] = {__ldg(&nodes[node].left), __ldg(&nodes[node].right)};
    bool go[2];
    for (int c = 0; c < 2; ++c) {
      const float *s = link[c] < 0 ? leaf_box + (size_t)(~link[c]) * 6 : nodes[link[c]].lo;
      float bx[6];
      for (int k = 0; k < 6; ++k) bx[k] = __ldg(s + k);
      const bool ov = overlap6(qb, bx);
      if (ov && link[c] < 0) leaf(~link[c]);
      go[c] = ov && link[c] >= 0;
    }
    if (go[0] && go[1]) {
      st[sp++] = link[1];
      node = link[0];
    } else if (go[0] || go[1]) {
      node = link[go[0] ? 0 : 1];
    } else {
      if (sp == 0) break;
      node = st[--sp];
    }
  }
}

// f < g, boxes known to overlap: no shared vertex, labels not an ignored pair, and the reference's 11-axis SAT with
// T_f first.  ignored: 64 masks, bit j of ignored[i] set when the label pair (i, j) is ignored (symmetric).
__device__ __forceinline__ bool self_pair(const int *__restrict__ faces, const int *__restrict__ labels,
                                          const unsigned long long *__restrict__ ignored, const float *sb, int f,
                                          int g, const int fv[3], const mmi::TriT<float> &tf) {
  const int g0 = __ldg(faces + 3 * g), g1 = __ldg(faces + 3 * g + 1), g2 = __ldg(faces + 3 * g + 2);
  for (int k = 0; k < 3; ++k)
    if (fv[k] == g0 || fv[k] == g1 || fv[k] == g2) return false;
  if (labels && ((__ldg(ignored + __ldg(labels + f)) >> __ldg(labels + g)) & 1ull)) return false;
  return mmi::sat11(tf, ld_tri(sb + (size_t)g * 9));
}

struct SelfWs {
  ScanWs scan;
  int *counts;   // [B][F]
  int *offsets;  // [B][F]
};

static size_t self_ws_layout(int B, int F, SelfWs *w, char *base) {
  size_t off = scan_ws_layout(B, F, w ? &w->scan : nullptr, base);
  const size_t n = align_up((size_t)B * F * 4, 256);
  if (w) { w->counts = (int *)(base + off); w->offsets = (int *)(base + off + n); }
  return off + 2 * n;
}

template <bool kWrite>
__global__ void __launch_bounds__(128) self_face_kernel(const int *__restrict__ faces, int F, SelfWs w,
                                                        const int *__restrict__ labels,
                                                        const unsigned long long *__restrict__ ignored, int max_pairs,
                                                        int *__restrict__ pairs) {
  const int b = blockIdx.y;
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const size_t o = (size_t)b * F + f;
  const float *sb = w.scan.soup + (size_t)b * F * 9;
  const int *ids = w.scan.bvh.ids + (size_t)b * F;
  const BvhNode *nodes = w.scan.bvh.nodes + (size_t)b * (F - 1);
  const float *leaf_box = w.scan.bvh.leaf_box + (size_t)b * F * 6;
  const mmi::TriT<float> tf = ld_tri(sb + (size_t)f * 9);
  const mmi::Box qb = mmi::tri_box(tf);
  const int fv[3] = {__ldg(faces + 3 * f), __ldg(faces + 3 * f + 1), __ldg(faces + 3 * f + 2)};
  if (!kWrite) {
    int n = 0;
    box_traverse(nodes, leaf_box, F, qb, [&](int j) {
      const int g = __ldg(ids + j);
      if (g > f && self_pair(faces, labels, ignored, sb, f, g, fv, tf)) ++n;
    });
    w.counts[o] = n;
    return;
  }
  const int first = w.offsets[o];
  const int room = min(w.counts[o], max_pairs - first);
  int *out = pairs + ((size_t)b * max_pairs + first) * 2;
  int last = f;
  for (int k = 0; k < room;) {
    int sel[kSelfSel];
    int ns = 0;
    box_traverse(nodes, leaf_box, F, qb, [&](int j) {
      const int g = __ldg(ids + j);
      if (g <= last || (ns == kSelfSel && g >= sel[kSelfSel - 1])) return;
      if (!self_pair(faces, labels, ignored, sb, f, g, fv, tf)) return;
      int i = ns < kSelfSel ? ns++ : kSelfSel - 1;  // insertion into the sorted kSelfSel smallest
      for (; i > 0 && sel[i - 1] > g; --i) sel[i] = sel[i - 1];
      sel[i] = g;
    });
    if (ns == 0) break;  // not reached: the count pass found `room` more
    for (int i = 0; i < ns && k < room; ++i, ++k) {
      out[2 * k] = f;
      out[2 * k + 1] = sel[i];
    }
    last = sel[ns - 1];
  }
}

__global__ void __launch_bounds__(1024) self_scan_kernel(int F, SelfWs w, int *__restrict__ count) {
  __shared__ int part[1024];
  const int b = blockIdx.x, t = threadIdx.x;
  const int per = (F + 1023) / 1024, lo = min(F, t * per), hi = min(F, lo + per);
  const int *c = w.counts + (size_t)b * F;
  int s = 0;
  for (int i = lo; i < hi; ++i) s += c[i];
  part[t] = s;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {  // inclusive Hillis-Steele scan of the thread sums
    const int v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  int run = part[t] - s;
  int *off = w.offsets + (size_t)b * F;
  for (int i = lo; i < hi; ++i) { off[i] = run; run += c[i]; }
  if (t == 1023) count[b] = part[1023];
}

}  // namespace shapy

extern "C" size_t shapy_self_collisions_workspace_bytes(int B, int F) {
  if (B <= 0 || F <= 0) return 0;
  return self_ws_layout(B, F, nullptr, nullptr) + 256;
}

extern "C" int shapy_self_collisions(const float *vertices, const int32_t *faces, int B, int V, int F,
                                     const int32_t *part_labels, const uint64_t *ignored_part_pairs, int refit,
                                     int max_pairs, int32_t *pairs, int32_t *count, void *workspace,
                                     size_t workspace_bytes, void *stream) {
  const char *name = "shapy_self_collisions";
  SHAPY_REQUIRE(B >= 0 && V > 0 && F > 0 && max_pairs >= 0, "%s: bad sizes", name);
  if (int rc = scan_limit(name, "faces", F)) return rc;
  if (B == 0) return SHAPY_OK;
  SHAPY_REQUIRE(vertices && faces && count && (pairs || max_pairs == 0), "%s: null argument", name);
  SHAPY_REQUIRE(!part_labels == !ignored_part_pairs, "%s: part_labels and ignored_part_pairs go together", name);
  SHAPY_REQUIRE(workspace && workspace_bytes >= shapy_self_collisions_workspace_bytes(B, F), "%s: workspace too small",
                name);
  cudaStream_t st = (cudaStream_t)stream;
  SelfWs w;
  self_ws_layout(B, F, &w, scan_base(workspace));
  const size_t n = (size_t)B * F * 3;
  scan_mesh_soup_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(vertices, faces, V, F, n, w.scan.soup);
  SHAPY_LAUNCH_CHECK();
  if (int rc = scan_tree(w.scan, B, F, refit != 0, st)) return rc;
  const dim3 grid(ceil_div(F, 128), B);
  const unsigned long long *ign = (const unsigned long long *)ignored_part_pairs;
  self_face_kernel<false><<<grid, 128, 0, st>>>(faces, F, w, part_labels, ign, max_pairs, pairs);
  SHAPY_LAUNCH_CHECK();
  self_scan_kernel<<<B, 1024, 0, st>>>(F, w, count);
  SHAPY_LAUNCH_CHECK();
  if (max_pairs > 0) {
    SHAPY_CUDA_TRY(cudaMemsetAsync(pairs, 0xFF, (size_t)B * max_pairs * 2 * sizeof(int32_t), st));
    self_face_kernel<true><<<grid, 128, 0, st>>>(faces, F, w, part_labels, ign, max_pairs, pairs);
    SHAPY_LAUNCH_CHECK();
  }
  return SHAPY_OK;
}
