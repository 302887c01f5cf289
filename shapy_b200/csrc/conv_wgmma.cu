// TMA + wgmma implicit-GEMM convolution for sm_90a (hand-written PTX, no CUTLASS).
//
//   D[pixel, cout] = sum_{tap, cin} X[pixel shifted by tap, cin] * Wt[tap][cout][cin]
//
// GEMM view: M = 128 output pixels, N = cout tile (<= 128), K = taps * cin walked in 64-channel k-blocks.
//   * A: one 4-D TMA box per (tap, k-block) straight out of the NHWC activation plane, the box origin shifted by the
//     tap; out-of-image rows / columns are ZERO-FILLED by the TMA unit = the padding (no im2col, no halo storage).
//     Stride-2 layers use four parity views of the same plane so every tap is again a dense box.  Channel counts that
//     are not a multiple of 64 still use 64-channel boxes: TMA zero-fills the channels past cin of both operands.
//   * B: 3-D TMA box of the pre-packed [tap][cout][cin] fp16 weights (BN scale folded in).
//   * Both operands land in the canonical K-major SWIZZLE_128B layout the wgmma shared-memory descriptor names, so no
//     thread touches operand data.
//   * warpgroup 0 = TMA producer (one elected thread), warpgroups 1 and 2 = consumers: each issues wgmma m64nNk16 for
//     64 of the 128 tile rows into fp32 register accumulators, then runs the epilogue of its rows.  The shared-memory
//     ring of `stages` slots (full / empty mbarriers) runs ahead across tile boundaries, so the loads of the next tile
//     overlap the epilogue of this one; persistent, one CTA per SM.
// Split-fp16 parity mode keeps activations and weights as fp16 hi + fp16 lo (x = hi + lo/2048) and issues
// A_hi.[B_hi|B_lo] as ONE N = 2 NT wgmma into [D0|D1] plus A_lo.B_hi into D1' (out = D0 + (D1 + D1')/2048).
// Epilogue: registers -> +bias (+residual) -> ReLU -> split to fp16 hi/lo -> global stores.
// Replaces cuDNN conv + BatchNorm + ReLU + residual add (4 launches, 4 HBM round trips) of
// regressor/human_shape/models/backbone/hrnet.py and torchvision BasicBlock / Bottleneck.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "conv.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace shapy {

constexpr int KCH = 64;   // channels per k-block: 128-byte rows, SWIZZLE_128B

// ------------------------------------------------------------------------------------ parameters
struct alignas(64) WgmmaParams {
  CUtensorMap a_hi[4], a_lo[4];  // [parity] (stride 2) or [0] (stride 1)
  CUtensorMap b_hi, b_lo;
  int N, Ho, Wo;                 // output extent
  int TW, TH, TN;                // M-tile box (TW * TH * TN <= 128 rows)
  int tiles_w, tiles_h, tiles_n;
  int cin, cout, ksize, stride;
  int kpt;                       // k-blocks per tap = ceil(cin / KCH)
  int stages;
  int relu;
  int pdl_late;                  // 1: release the programmatic dependents when this CTA starts its LAST tile, not at entry
  uint32_t a_bytes, b_bytes, b_stride;  // per k-block: TMA bytes of A / B, smem pitch of the B_hi(+B_lo) block
  const float *bias;
  __half *out_hi, *out_lo;
  int out_ctot, out_coff;
  const __half *res_hi, *res_lo;
  int res_ctot, res_coff;
};

constexpr int kThreads = 384;                // producer warpgroup + two consumer warpgroups
constexpr int kProdRegs = 40, kConsRegs = 232;

template <bool SPLIT, int NT>
__global__ void __launch_bounds__(kThreads, 1) conv_wgmma_kernel(const __grid_constant__ WgmmaParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr int NACC = (SPLIT ? 2 * NT : NT) / 2;   // fp32 accumulators per thread: [D0 | D1] of a 64 x NT(x2) tile
  constexpr int NLO = SPLIT ? NT / 2 : 1;           // A_lo . B_hi, kept apart: wgmma pipelines only disjoint or equal D
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t A_BLK = 128 * KCH * 2;
  const uint32_t kblk_bytes = A_BLK * (SPLIT ? 2 : 1) + p.b_stride;   // one stage = one k-block of one tap
  const uint32_t bar_base = smem_base + kblk_bytes * p.stages;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };
  const int wg = threadIdx.x >> 7;
  const int n_tiles = p.cout / NT;
  const int total_tiles = p.tiles_w * p.tiles_h * p.tiles_n * n_tiles;
  const int iters = p.ksize * p.ksize * p.kpt;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // Programmatic dependent launch: the next kernel of this stream may start its prologue once every CTA here has
  // released it.  Released at entry, its CTAs occupy SMs (which another lane's kernel could use) for this kernel's whole
  // duration; released when a CTA starts its last tile (pdl_late), they only cover this kernel's tail.
  if (!p.pdl_late) pdl_launch_dependents();
  pdl_wait();                // everything above touched no global memory; inputs of this kernel are now complete

  auto tile_coords = [&](int id, int &w0, int &h0, int &n0, int &c_out0) {
    c_out0 = (id % n_tiles) * NT; id /= n_tiles;
    w0 = (id % p.tiles_w) * p.TW; id /= p.tiles_w;
    h0 = (id % p.tiles_h) * p.TH; id /= p.tiles_h;
    n0 = id * p.TN;
  };

  if (wg == 0) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<kProdRegs>();
    if (threadIdx.x < 32 && elect_one()) {
      int s = 0;
      uint32_t ph = 0;
      const int pad = p.ksize / 2;
      const uint32_t tx = (p.a_bytes + p.b_bytes) * (SPLIT ? 2u : 1u);
      for (int id = blockIdx.x; id < total_tiles; id += gridDim.x) {
        int w0, h0, n0, c_out0;
        tile_coords(id, w0, h0, n0, c_out0);
        if (p.pdl_late && id + (int)gridDim.x >= total_tiles) pdl_launch_dependents();   // last tile of this CTA
#pragma unroll 1
        for (int it = 0; it < iters; ++it) {
          const int tap = it / p.kpt, c0 = (it % p.kpt) * KCH;
          const int ky = tap / p.ksize, kx = tap % p.ksize;
          int mi = 0, x, y;
          if (p.stride == 1) {
            x = w0 + kx - pad; y = h0 + ky - pad;
          } else {  // input row 2*oh + ky - 1: ky=0 -> odd rows, index oh-1; ky=1 -> even rows, oh; ky=2 -> odd rows, oh
            mi = (ky != 1) * 2 + (kx != 1);
            x = w0 + (kx == 0 ? -1 : 0); y = h0 + (ky == 0 ? -1 : 0);
          }
          mbar_wait(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), tx);
          const uint32_t kb = smem_base + kblk_bytes * s;
          tma_load_4d(kb, &p.a_hi[mi], full_bar(s), c0, x, y, n0);
          if (SPLIT) tma_load_4d(kb + A_BLK, &p.a_lo[mi], full_bar(s), c0, x, y, n0);
          const uint32_t bb = kb + A_BLK * (SPLIT ? 2 : 1);
          tma_load_3d(bb, &p.b_hi, full_bar(s), c0, c_out0, tap);
          if (SPLIT) tma_load_3d(bb + p.b_bytes, &p.b_lo, full_bar(s), c0, c_out0, tap);   // directly after the hi rows
          if (++s == p.stages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===================================================================== consumers: MMA + epilogue
    setmaxnreg_inc<kConsRegs>();
    const int cw = wg - 1;                        // rows 64 cw .. 64 cw + 63 of the tile
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    int s = 0;
    uint32_t ph = 0;
    float acc[NACC], acl[NLO];
    for (int id = blockIdx.x; id < total_tiles; id += gridDim.x) {
      int w0, h0, n0, c_out0;
      tile_coords(id, w0, h0, n0, c_out0);
#pragma unroll
      for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
#pragma unroll
      for (int i = 0; i < NLO; ++i) acl[i] = 0.f;
      int prev = -1;
#pragma unroll 1
      for (int it = 0; it < iters; ++it) {
        mbar_wait(full_bar(s), ph);
        const uint32_t kb = smem_base + kblk_bytes * s;
        const uint64_t a = wgmma_desc<KCH>(kb + cw * 64 * KCH * 2);
        const uint64_t al = wgmma_desc<KCH>(kb + A_BLK + cw * 64 * KCH * 2);
        const uint64_t b = wgmma_desc<KCH>(kb + A_BLK * (SPLIT ? 2 : 1));
#pragma unroll
        for (int i = 0; i < NACC; ++i) reg_fence(acc[i]);
#pragma unroll
        for (int i = 0; i < NLO; ++i) reg_fence(acl[i]);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < KCH / 16; ++ks) {   // +32 bytes along K = +2 descriptor units
          if (SPLIT) {
            wgmma_f16<2 * NT>(acc, a + 2 * ks, b + 2 * ks, 1);   // [D0 | D1] += A_hi . [B_hi | B_lo]^T
            wgmma_f16<NT>(acl, al + 2 * ks, b + 2 * ks, 1);       // D1' += A_lo . B_hi^T
          } else {
            wgmma_f16<NT>(acc, a + 2 * ks, b + 2 * ks, 1);
          }
        }
        wgmma_commit();
#pragma unroll
        for (int i = 0; i < NACC; ++i) reg_fence(acc[i]);
#pragma unroll
        for (int i = 0; i < NLO; ++i) reg_fence(acl[i]);
        wgmma_wait<1>();                          // the previous stage's wgmmas have read their operands
        if (prev >= 0 && t == 0) mbar_arrive(empty_bar(prev));
        prev = s;
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < NACC; ++i) reg_fence(acc[i]);
#pragma unroll
      for (int i = 0; i < NLO; ++i) reg_fence(acl[i]);
      if (prev >= 0 && t == 0) mbar_arrive(empty_bar(prev));

      // ---- epilogue: this thread holds rows r0 and r0 + 8, two adjacent columns of every 8-column group
      const int q4 = lane & 3;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = cw * 64 + warp * 16 + (lane >> 2) + 8 * half;
        const int dw = row % p.TW, dh = (row / p.TW) % p.TH, dn = row / (p.TW * p.TH);
        const int ow = w0 + dw, oh = h0 + dh, on = n0 + dn;
        if (!(dn < p.TN && ow < p.Wo && oh < p.Ho && on < p.N)) continue;
        const size_t pix = ((size_t)on * p.Ho + oh) * p.Wo + ow;
        const size_t oo = pix * p.out_ctot + p.out_coff + c_out0;
        const size_t ro = pix * p.res_ctot + p.res_coff + c_out0;
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) {
          const int c = 8 * j + 2 * q4;
          const int i = 4 * j + 2 * half;
          const float2 bq = __ldg(reinterpret_cast<const float2 *>(p.bias + c_out0 + c));
          float r0 = acc[i], r1 = acc[i + 1];
          if (SPLIT) {
            r0 += (acc[NT / 2 + i] + acl[SPLIT ? i : 0]) * kLoInv;
            r1 += (acc[NT / 2 + i + 1] + acl[SPLIT ? i + 1 : 0]) * kLoInv;
          }
          r0 += bq.x; r1 += bq.y;
          if (p.res_hi) {
            const __half2 rh = *reinterpret_cast<const __half2 *>(p.res_hi + ro + c);
            r0 += __low2float(rh); r1 += __high2float(rh);
            if (SPLIT && p.res_lo) {
              const __half2 rl = *reinterpret_cast<const __half2 *>(p.res_lo + ro + c);
              r0 += __low2float(rl) * kLoInv; r1 += __high2float(rl) * kLoInv;
            }
          }
          if (p.relu) { r0 = fmaxf(r0, 0.f); r1 = fmaxf(r1, 0.f); }
          __half h0_, h1_, l0_, l1_;
          split_store(r0, h0_, l0_);
          split_store(r1, h1_, l1_);
          *reinterpret_cast<__half2 *>(p.out_hi + oo + c) = __halves2half2(h0_, h1_);
          if (SPLIT && p.out_lo) *reinterpret_cast<__half2 *>(p.out_lo + oo + c) = __halves2half2(l0_, l1_);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------ host side
// Grid of a persistent kernel over `items` equal work items.  min(items, SMs) leaves a ragged last round (e.g. 896
// items on 132 CTAs are 104 CTAs with 7 items and 28 with 6); with CTAs = ceil(items / rounds) every CTA finishes
// together and the SMs the grid does not use run another lane's kernel for the whole time.
static int even_grid(int items, int sms) {
  if (items <= sms) return items;
  const int rounds = ceil_div(items, sms);
  return ceil_div(items, rounds);
}

static int sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

struct WgmmaPlan {
  WgmmaParams p;
  int NT;
  bool split;
  dim3 grid;
  size_t smem;
};

static const int kNts[] = {128, 96, 64, 48, 32, 16};   // cout tiles with a kernel instantiation

bool wgmma_supported(const ConvW &w, const ActView &in, const ActView &out) {
  if (w.cin % 16 || w.cout % 16) return false;
  if (!((w.ksize == 3 || w.ksize == 1) && (w.stride == 1 || (w.stride == 2 && w.ksize == 3)))) return false;
  if (w.stride == 2 && (in.H % 2 || in.W % 2)) return false;
  if (in.Ctot % 8 || in.coff % 8 || out.Ctot % 8 || out.coff % 8) return false;
  if (out.W > 128 && out.W % 128) return false;
  return get_encode() != nullptr;
}

WgmmaPlan *wgmma_plan_create(const ConvW &w, const ActView &in, const ActView &out, const ActView *res, bool relu) {
  if (!wgmma_supported(w, in, out)) {
    set_error("wgmma_plan_create: unsupported convolution (cin %d cout %d k %d s %d)", w.cin, w.cout, w.ksize, w.stride);
    return nullptr;
  }
  auto *pl = new WgmmaPlan();
  memset(&pl->p, 0, sizeof(pl->p));
  WgmmaParams &p = pl->p;
  const bool split = in.lo != nullptr;
  pl->split = split;
  const int sms = sm_count();
  p.N = out.N; p.Ho = out.H; p.Wo = out.W;
  p.TW = std::min(out.W, 128);
  p.TH = std::max(1, std::min(out.H, 128 / p.TW));
  p.TN = (p.TW == out.W && p.TH == out.H) ? std::max(1, std::min(out.N, 128 / (p.TW * p.TH))) : 1;
  p.tiles_w = ceil_div(out.W, p.TW); p.tiles_h = ceil_div(out.H, p.TH); p.tiles_n = ceil_div(out.N, p.TN);
  p.cin = w.cin; p.cout = w.cout; p.ksize = w.ksize; p.stride = w.stride;
  p.kpt = ceil_div(w.cin, KCH);
  {
    // cout tile: balance SM utilisation (tiles per CTA round) against the per-wgmma operand cost.  A 128-row tile is two
    // m64nNk16 per k-step; each reads 2 KB of A and N x 32 B of B from shared memory (128 B/cycle) and needs N / 2
    // tensor cycles, plus a fixed per-tile epilogue / barrier cost.
    const double m_tiles = (double)p.tiles_w * p.tiles_h * p.tiles_n;
    auto mma_cyc = [](double n) { return 2.0 * std::max((2048.0 + 32.0 * n) / 128.0, n * 0.5); };
    double best = 1e30;
    int best_nt = 0;
    for (int nt : kNts) {
      if (w.cout % nt || (split && nt > 96)) continue;   // split: 3 NT / 2 accumulators per thread must fit 232 registers
      const double per_k = split ? mma_cyc(2.0 * nt) + mma_cyc(nt) : mma_cyc(nt);
      const double cost = std::ceil(m_tiles * (w.cout / nt) / sms) *
                          (per_k * w.ksize * w.ksize * p.kpt * (KCH / 16) + 400.0 * nt / 16);
      if (cost < best) { best = cost; best_nt = nt; }
    }
    pl->NT = best_nt;
  }
  p.relu = relu;
  p.pdl_late = 1;
  const int rows = p.TW * p.TH * p.TN;
  p.a_bytes = (uint32_t)rows * KCH * 2;
  p.b_bytes = (uint32_t)pl->NT * KCH * 2;
  p.b_stride = (uint32_t)align_up((size_t)p.b_bytes * (split ? 2 : 1), 1024);
  const size_t stage = 128u * KCH * 2 * (split ? 2 : 1) + p.b_stride;
  // one persistent CTA per SM owns (almost) all of its 227 KB of shared memory
  p.stages = (int)std::max<size_t>(2, std::min<size_t>(8, (216 * 1024) / stage));
  pl->smem = stage * p.stages + 16 * p.stages + 1024;
  p.bias = w.bias;
  p.out_hi = out.hi; p.out_lo = out.lo; p.out_ctot = out.Ctot; p.out_coff = out.coff;
  p.res_hi = res ? res->hi : nullptr; p.res_lo = res ? res->lo : nullptr;
  p.res_ctot = res ? res->Ctot : 0; p.res_coff = res ? res->coff : 0;
  pl->grid = dim3(even_grid(p.tiles_w * p.tiles_h * p.tiles_n * (w.cout / pl->NT), sms), 1);
  if (getenv("SHAPY_CONV_DEBUG"))
    fprintf(stderr, "[wgmma] cin %d cout %d k %d s %d %dx%d N %d: NT %d tile %dx%dx%d grid %d stages %d\n", w.cin, w.cout,
            w.ksize, w.stride, out.H, out.W, out.N, pl->NT, p.TW, p.TH, p.TN, pl->grid.x, p.stages);
  bool ok = true;
  // activation maps
  const int nmaps = w.stride == 2 ? 4 : 1;
  for (int mi = 0; mi < nmaps && ok; ++mi) {
    const int phy = mi >> 1, phx = mi & 1;
    cuuint64_t dims[4], strides[3];
    size_t off;
    if (w.stride == 1) {
      dims[0] = in.C; dims[1] = in.W; dims[2] = in.H; dims[3] = in.N;
      strides[0] = (cuuint64_t)in.Ctot * 2; strides[1] = (cuuint64_t)in.W * in.Ctot * 2;
      strides[2] = (cuuint64_t)in.H * in.W * in.Ctot * 2;
      off = in.coff;
    } else {   // parity view: rows 2y + py, columns 2x + px of the input
      dims[0] = in.C; dims[1] = in.W / 2; dims[2] = in.H / 2; dims[3] = in.N;
      strides[0] = (cuuint64_t)in.Ctot * 4; strides[1] = (cuuint64_t)in.W * in.Ctot * 4;
      strides[2] = (cuuint64_t)in.H * in.W * in.Ctot * 2;
      off = (size_t)in.coff + ((size_t)phy * in.W + phx) * in.Ctot;
    }
    cuuint32_t box[4] = {(cuuint32_t)KCH, (cuuint32_t)p.TW, (cuuint32_t)p.TH, (cuuint32_t)p.TN};
    ok = ok && encode(&p.a_hi[mi], in.hi + off, 4, dims, strides, box, KCH);
    if (split) ok = ok && encode(&p.a_lo[mi], in.lo + off, 4, dims, strides, box, KCH);
  }
  if (ok) {
    cuuint64_t dims[3] = {(cuuint64_t)w.cin, (cuuint64_t)w.cout, (cuuint64_t)(w.ksize * w.ksize)};
    cuuint64_t strides[2] = {(cuuint64_t)w.cin * 2, (cuuint64_t)w.cin * w.cout * 2};
    cuuint32_t box[3] = {(cuuint32_t)KCH, (cuuint32_t)pl->NT, 1};
    ok = ok && encode(&p.b_hi, w.w_hi, 3, dims, strides, box, KCH);
    if (split) ok = ok && encode(&p.b_lo, w.w_lo, 3, dims, strides, box, KCH);
  }
  if (!ok) { delete pl; return nullptr; }
  return pl;
}

void wgmma_plan_destroy(WgmmaPlan *p) { delete p; }

template <bool SPLIT, int NT>
static int launch_t(const WgmmaPlan *pl, cudaStream_t st, bool pdl) {
  static std::atomic<unsigned long long> attr_done{0};
  auto kernel = conv_wgmma_kernel<SPLIT, NT>;
  SHAPY_CUDA_TRY(set_max_dynamic_smem(kernel, 227 * 1024, attr_done));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = pl->grid;
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = pl->smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  SHAPY_CUDA_TRY(cudaLaunchKernelEx(&cfg, kernel, pl->p));
  shapy::count_launch();
  return SHAPY_OK;
}

template <bool SPLIT>
static int launch_nt(const WgmmaPlan *pl, cudaStream_t st, bool pdl) {
  switch (pl->NT) {
    case 128:
      if constexpr (!SPLIT) return launch_t<SPLIT, 128>(pl, st, pdl);   // split mode plans NT <= 96
      set_error("wgmma engine: NT 128 in split mode");
      return SHAPY_ERR_STATE;
    case 96: return launch_t<SPLIT, 96>(pl, st, pdl);
    case 64: return launch_t<SPLIT, 64>(pl, st, pdl);
    case 48: return launch_t<SPLIT, 48>(pl, st, pdl);
    case 32: return launch_t<SPLIT, 32>(pl, st, pdl);
    default: return launch_t<SPLIT, 16>(pl, st, pdl);
  }
}

int wgmma_plan_launch(const WgmmaPlan *pl, cudaStream_t st, bool pdl) {
  return pl->split ? launch_nt<true>(pl, st, pdl) : launch_nt<false>(pl, st, pdl);
}

}  // namespace shapy
