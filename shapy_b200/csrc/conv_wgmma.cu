// TMA + wgmma implicit-GEMM convolution for sm_90a (hand-written PTX, no CUTLASS).
//
//   D[pixel, cout] = sum_{tap, cin} X[pixel shifted by tap, cin] * Wt[tap][cout][cin]
//
// GEMM view: M = 128 output pixels, N = cout tile (<= 128), K = taps * cin walked in 64-channel k-blocks.
//   * A: one 4-D TMA box per (tap, k-block) straight out of the NHWC activation plane, the box origin shifted by the
//     tap; out-of-image rows / columns are ZERO-FILLED by the TMA unit = the padding (no im2col, no halo storage).
//     Stride-2 layers use four parity views of the same plane so every tap is again a dense box.  A layer with
//     cin < 64 loads boxes of cin channels into the same 128-byte rows and leaves the rest of each row unwritten (no
//     issued k16 step reads it); wider channel counts that are not a multiple of 64 use 64-channel boxes, and TMA
//     zero-fills the channels past cin of both operands.
//   * Halo path (3x3 stride 1, one image per tile): a work item is TH output rows x the full width, computed on the
//     padded "wide" grid of pitch Wp = W + 2 (tile row r = output (h0 + r / Wp, r % Wp); columns >= W are computed and
//     dropped by the epilogue).  Each 64-channel block is loaded ONCE with its halo as one (64, Wp, TH + 2) box at
//     origin (-1, h0 - 1) into a separate halo ring; tap (ky, kx) is the same buffer read from row ky * Wp + kx on (the
//     descriptor start moves by whole 128-byte rows, the swizzle is a function of the absolute address).  Activations
//     then cross L2 -> shared memory ~1.4x per channel block instead of 9x; only the weights stream per (tap, block).
//   * Weight-resident path (halo path with cin <= 64 and one cout tile, where the whole weight set fits): operands
//     are stored as 16-channel k16 slices with 32-byte rows (SWIZZLE_32B) instead of zero-padded 128-byte rows, every
//     CTA loads the layer's [tap][cout][cin] weights ONCE (before waiting on the previous kernel), and each tile loads
//     only its halo band.  The k16 steps and their order are those of the halo path: taps 0..8, slices 0, 1, ...
//   * B: 3-D TMA box of the pre-packed [tap][cout][cin] fp16 weights (BN scale folded in).
//   * k16 steps that lie wholly past cin (the zero-filled tail of the last channel block, e.g. 1 of 4 at cin 48) are
//     not issued.
//   * Both operands land in the canonical K-major SWIZZLE_128B layout the wgmma shared-memory descriptor names, so no
//     thread touches operand data.
//   * warpgroup 0 = TMA producer (one elected thread), warpgroups 1 and 2 = consumers.  The shared-memory ring of
//     `stages` slots (full / empty mbarriers) runs ahead across tile boundaries; persistent, one CTA per SM.  Two
//     consumer schedules:
//       - cooperative: both consumers work on the same tile, each issuing wgmma m64nNk16 for 64 of its 128 rows, and
//         both run the epilogue of their rows at the same time into one staging box (the tensor cores idle meanwhile);
//       - ping-pong: each consumer owns whole tiles (two m64 accumulator sets, all 128 rows) and the two alternate
//         through the CTA's tile sequence.  A pair of hand-off mbarriers orders the mainloops: a consumer starts its
//         tile's k-blocks only after the other has issued all of the previous tile's, so one consumer's epilogue runs
//         under the other's MMAs, and the ring positions each consumer waits on are at most one phase ahead.
//     Both give every output row the same wgmma sequence and the same epilogue arithmetic.
// Split-fp16 parity mode keeps activations and weights as fp16 hi + fp16 lo (x = hi + lo/2048) and issues
// A_hi.[B_hi|B_lo] as ONE N = 2 NT wgmma into [D0|D1] plus A_lo.B_hi into D1' (out = D0 + (D1 + D1')/2048).
// Epilogue, the same in both schedules: registers -> +bias (+residual) -> ReLU -> split to fp16 hi/lo -> stmatrix into
// the tile's shared-memory staging box (ping-pong: the consumer's), into which TMA loaded the residual during the
// mainloop (read back with ldmatrix) -> TMA tensor stores.  The box is stored in column boxes of 64 / 32 / 16 channels
// with the TMA swizzle of their rows, so the 16-byte matrix rows and the TMA accesses are free of bank conflicts.
// Replaces cuDNN conv + BatchNorm + ReLU + residual add (4 launches, 4 HBM round trips) of
// regressor/human_shape/models/backbone/hrnet.py and torchvision BasicBlock / Bottleneck.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <type_traits>

#include "conv.cuh"
#include "tma.cuh"
#include "wgmma.cuh"

namespace shapy {

constexpr int KCH = 64;   // channels per k-block: 128-byte rows, SWIZZLE_128B

// ------------------------------------------------------------------------------------ parameters
struct alignas(64) WgmmaParams {
  CUtensorMap a_hi[4], a_lo[4];  // [parity] (stride 2) or [0] (stride 1)
  CUtensorMap b_hi, b_lo;
  int TW, TH, TN;                // M-tile box (TW * TH * TN <= 128 rows)
  int tiles_w, tiles_h, tiles_n;
  int cin, cout, ksize, stride;
  int kpt;                       // k-blocks per tap = ceil(cin / KCH)
  int ks_last;                   // k16 steps of the last k-block that hold channels < cin
  int stages;                    // (A +) B ring slots
  int hstages;                   // halo path: halo ring slots
  int relu;
  int pdl_late;                  // 1: release the programmatic dependents when this CTA starts its LAST tile, not at entry
  uint32_t a_bytes, b_bytes, b_stride;  // per k-block: TMA bytes of A, smem pitch of B_hi (B_lo follows) and of B_hi + B_lo
  uint32_t b_tx;                 // per k-block: TMA bytes of B (one plane)
  uint32_t h_plane;              // halo path: smem pitch of one halo plane (hi or lo)
  uint32_t h_slice;              // resident path: smem pitch of one 16-channel slice of a halo plane
  uint32_t w_bytes;              // resident path: TMA bytes (= smem bytes) of the whole weight set, all planes
  const float *bias;
  int res, res_lo;               // the epilogue adds a residual (hi plane; and lo plane, split mode)
  int out_lo;                    // split mode: the epilogue stores the output's lo plane
  // epilogue: output / residual maps over the [N][Ho][Wo] x cout view (boxes stage_cw(NT) x o_bw x TH x TN, the
  // padded grid's junk columns excluded), and the shared-memory staging box of the tile (one per consumer in ping-pong)
  CUtensorMap o_hi, o_lo, r_hi, r_lo;
  int o_bw;                      // box width: Wo on the halo path, TW on the per-tap path
  uint32_t o_plane;              // smem pitch of one staged plane (hi or lo): 128 rows x NT
  uint32_t o_bytes;              // TMA bytes of one plane's tile (all its column boxes)
};

constexpr int kThreads = 384;                // producer warpgroup + two consumer warpgroups
constexpr int kProdRegs = 40, kConsRegs = 232;

#ifdef SHAPY_CONV_STAMPS
// Cycle-stamp build (tools/conv_phase_stamps.py): per consumer warpgroup and tile, clock64 at the first full-barrier
// pass, the last commit, the return of wait<0> and the end of the epilogue, summed over all tiles of a launch as
// [wait before the first k-block, mainloop, drain, epilogue, tiles, operand waits inside the mainloop].
__device__ unsigned long long g_conv_stamps[6];
#endif

// fp32 accumulators per thread of one m64 set: [D0 | D1] of a 64 x NT(x2) tile, and A_lo . B_hi kept apart (wgmma
// pipelines only disjoint or equal D)
template <bool SPLIT, int NT>
constexpr int cons_accs() { return (SPLIT ? 2 * NT : NT) / 2 + (SPLIT ? NT / 2 : 0); }

// The staging box of a plane is NT / CW column boxes of 128 rows x CW channels, each stored with the TMA swizzle of its
// CW * 2-byte rows (128 / 64 / 32 B), CW the widest of 64, 32, 16 that divides NT: no padding, and the 8 rows of every
// stmatrix / ldmatrix matrix (8 consecutive box rows, one 16-byte chunk) fall in 8 distinct 16-byte bank groups.
constexpr int stage_cw(int nt) { return nt % 64 == 0 ? 64 : (nt % 32 == 0 ? 32 : 16); }

template <bool SPLIT, int NT, bool HALO, bool PP, bool RES>
__global__ void __launch_bounds__(kThreads, 1) conv_wgmma_kernel(const __grid_constant__ WgmmaParams p) {
  static_assert(!RES || HALO, "the weight-resident path is a halo path");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr int NACC = (SPLIT ? 2 * NT : NT) / 2;   // fp32 accumulators per thread: [D0 | D1] of a 64 x NT(x2) tile
  constexpr int NLO = SPLIT ? NT / 2 : 1;           // A_lo . B_hi, kept apart: wgmma pipelines only disjoint or equal D
  constexpr int PARTS = SPLIT ? 2 : 1;
  constexpr int MT = PP ? 2 : 1;                    // m64 accumulator sets per consumer: ping-pong owns all 128 rows
  constexpr int CONS = PP ? 1 : 2;                  // consumers that release each ring slot
  static_assert(!PP || MT * cons_accs<SPLIT, NT>() <= 192, "ping-pong accumulators must fit the consumer registers");
  constexpr int CW = stage_cw(NT);                // channels per column box of the staged tile
  constexpr uint32_t CB_BYTES = 128u * CW * 2;      // one column box (a multiple of its swizzle's 256 / 512 / 1024 B)
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  constexpr uint32_t A_BLK = 128 * KCH * 2;
  // shared memory: [halo ring (halo path)] [ring of k-block stages: A (per-tap path) + B | resident weights]
  //                [output staging box (ping-pong: of consumer 0, of consumer 1), 1024-aligned] [mbarriers]
  const uint32_t h_stage = p.h_plane * PARTS;
  const uint32_t ring_base = smem_base + (HALO ? h_stage * p.hstages : 0u);
  const uint32_t kblk_bytes = (HALO ? 0u : A_BLK * PARTS) + p.b_stride;   // one stage = one k-block of one tap
  const uint32_t o_base = (ring_base + (RES ? p.w_bytes : kblk_bytes * p.stages) + 1023u) & ~1023u;
  const uint32_t bar_base = o_base + (PP ? 2u : 1u) * p.o_plane * PARTS;
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (p.stages + s); };
  auto hfull_bar = [&](int s) { return bar_base + 8u * (2 * p.stages + s); };
  auto hempty_bar = [&](int s) { return bar_base + 8u * (2 * p.stages + p.hstages + s); };
  // ping-pong: consumer c arrives on handoff_bar(c) once it has issued every k-block of its tile
  auto handoff_bar = [&](int c) { return bar_base + 8u * (2 * p.stages + 2 * p.hstages + c); };
  // the residual of consumer c's tile (cooperative: of the tile, c = 0) has landed in its staging box
  auto res_bar = [&](int c) { return bar_base + 8u * (2 * p.stages + 2 * p.hstages + 2 + c); };
  // resident path: the weight set has landed
  const uint32_t w_bar = bar_base + 8u * (2 * p.stages + 2 * p.hstages + 4);
  // broadcast so ptxas sees a warp-uniform value: the ping-pong hand-off wait depends on it, and a wait it takes for
  // divergent makes it serialise every wgmma of the kernel
  const int wg = __shfl_sync(0xffffffffu, (int)threadIdx.x >> 7, 0);
  const int n_tiles = p.cout / NT;
  const int total_tiles = p.tiles_w * p.tiles_h * p.tiles_n * n_tiles;
  const int taps = p.ksize * p.ksize;
  const int iters = taps * p.kpt;
  // k-block `it` of a tile: tap-major on the per-tap path, channel-block-major on the halo path (one halo load per block)
  auto decode = [&](int it, int &tap, int &cb) {
    if (HALO) { cb = it / taps; tap = it - cb * taps; } else { tap = it / p.kpt; cb = it - tap * p.kpt; }
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), CONS); }
    for (int s = 0; s < (HALO ? p.hstages : 0); ++s) { mbar_init(hfull_bar(s), 1); mbar_init(hempty_bar(s), CONS); }
    for (int c = 0; c < 2; ++c) { mbar_init(handoff_bar(c), 1); mbar_init(res_bar(c), 1); }
    if (RES) mbar_init(w_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // The weights are packed once, before any launch, so no earlier kernel of the stream writes them: their load
  // overlaps the previous kernel's tail.  Slice (tap, j) holds cin 16 j .. 16 j + 15 of all cout, hi rows then lo rows.
  if (RES && threadIdx.x == 0) {
    const int S = p.cin / 16;
    mbar_expect_tx(w_bar, p.w_bytes);
    for (int i = 0; i < 9 * S; ++i) {
      const uint32_t wb = ring_base + (uint32_t)i * PARTS * p.b_tx;
      tma_load_3d(wb, &p.b_hi, w_bar, (i % S) * 16, 0, i / S);
      if (SPLIT) tma_load_3d(wb + p.b_tx, &p.b_lo, w_bar, (i % S) * 16, 0, i / S);
    }
  }
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
      int s = 0, hs = 0;
      uint32_t ph = 0, hph = 0;
      const int pad = p.ksize / 2;
      const uint32_t tx = (HALO ? p.b_tx : p.a_bytes + p.b_tx) * PARTS;
      for (int id = blockIdx.x; id < total_tiles; id += gridDim.x) {
        int w0, h0, n0, c_out0;
        tile_coords(id, w0, h0, n0, c_out0);
        if (p.pdl_late && id + (int)gridDim.x >= total_tiles) pdl_launch_dependents();   // last tile of this CTA
        if (RES) {                // the band with its halo, one box per 16-channel slice and plane
          mbar_wait(hempty_bar(hs), hph ^ 1);
          mbar_expect_tx(hfull_bar(hs), p.a_bytes * PARTS);
          const uint32_t hb = smem_base + h_stage * hs;
          for (int j = 0; j < p.cin / 16; ++j) {
            tma_load_4d(hb + j * p.h_slice, &p.a_hi[0], hfull_bar(hs), 16 * j, w0 - 1, h0 - 1, n0);
            if (SPLIT) tma_load_4d(hb + p.h_plane + j * p.h_slice, &p.a_lo[0], hfull_bar(hs), 16 * j, w0 - 1, h0 - 1, n0);
          }
          if (++hs == p.hstages) { hs = 0; hph ^= 1; }
          continue;
        }
#pragma unroll 1
        for (int it = 0; it < iters; ++it) {
          int tap, cb;
          decode(it, tap, cb);
          const int c0 = cb * KCH;
          if (HALO && tap == 0) {   // the channel block with its halo, once for all nine taps
            mbar_wait(hempty_bar(hs), hph ^ 1);
            mbar_expect_tx(hfull_bar(hs), p.a_bytes * PARTS);
            const uint32_t hb = smem_base + h_stage * hs;
            tma_load_4d(hb, &p.a_hi[0], hfull_bar(hs), c0, w0 - 1, h0 - 1, n0);
            if (SPLIT) tma_load_4d(hb + p.h_plane, &p.a_lo[0], hfull_bar(hs), c0, w0 - 1, h0 - 1, n0);
            if (++hs == p.hstages) { hs = 0; hph ^= 1; }
          }
          mbar_wait(empty_bar(s), ph ^ 1);
          mbar_expect_tx(full_bar(s), tx);
          const uint32_t kb = ring_base + kblk_bytes * s;
          if (!HALO) {
            const int ky = tap / p.ksize, kx = tap % p.ksize;
            int mi = 0, x, y;
            if (p.stride == 1) {
              x = w0 + kx - pad; y = h0 + ky - pad;
            } else {  // input row 2*oh + ky - 1: ky=0 -> odd rows, index oh-1; ky=1 -> even rows, oh; ky=2 -> odd rows, oh
              mi = (ky != 1) * 2 + (kx != 1);
              x = w0 + (kx == 0 ? -1 : 0); y = h0 + (ky == 0 ? -1 : 0);
            }
            tma_load_4d(kb, &p.a_hi[mi], full_bar(s), c0, x, y, n0);
            if (SPLIT) tma_load_4d(kb + A_BLK, &p.a_lo[mi], full_bar(s), c0, x, y, n0);
          }
          const uint32_t bb = kb + (HALO ? 0u : A_BLK * PARTS);
          tma_load_3d(bb, &p.b_hi, full_bar(s), c0, c_out0, tap);
          if (SPLIT) tma_load_3d(bb + p.b_bytes, &p.b_lo, full_bar(s), c0, c_out0, tap);   // directly after the hi rows
          if (++s == p.stages) { s = 0; ph ^= 1; }
        }
      }
    }
  } else {
    // ===================================================================== consumers: MMA + epilogue
    setmaxnreg_inc<kConsRegs>();
    const int cw = wg - 1;                        // cooperative: rows 64 cw .. 64 cw + 63 of every tile; ping-pong: the
                                                  // CTA's tiles cw, cw + 2, ...
    const int t = threadIdx.x & 127, warp = t >> 5, lane = t & 31;
    int s = 0, hs = 0;
    uint32_t ph = 0, hph = 0, hoph = 0, rph = 0;
    // the output staging box this consumer writes (hi plane, then lo); one thread loads the residual into it and stores
    // it, after a barrier over the threads that write it (ping-pong: this consumer; cooperative: both)
    const uint32_t ob = o_base + (PP ? (uint32_t)cw : 0u) * p.o_plane * PARTS;
    const bool issuer = t == 0 && (PP || cw == 0);
    const int ebar = PP ? 1 + cw : 1, ethreads = PP ? 128 : 256;
    const int rb = PP ? cw : 0;
    // ping-pong: step the ring positions over the k-blocks (and halo loads) of the other consumer's tile
    auto skip_tile = [&]() {
      const int q = s + iters, hq = hs + p.kpt;
      if (!RES) { ph ^= (uint32_t)(q / p.stages) & 1u; s = q % p.stages; }
      if (HALO) { hph ^= (uint32_t)(hq / p.hstages) & 1u; hs = hq % p.hstages; }
    };
    if (PP && cw == 1) skip_tile();
    float acc[MT][NACC], acl[MT][NLO];
    if (RES) mbar_wait(w_bar, 0);
#ifdef SHAPY_CONV_STAMPS
    long long st_end = clock64(), st0 = 0, st1 = 0, st2 = 0, st_w = 0;
#endif
    for (int id = blockIdx.x + (PP ? cw : 0) * gridDim.x, k = 0; id < total_tiles; id += (PP ? 2 : 1) * gridDim.x, ++k) {
      int w0, h0, n0, c_out0;
      tile_coords(id, w0, h0, n0, c_out0);
      if (PP && (k > 0 || cw == 1)) {             // the other consumer has issued the CTA's previous tile
        mbar_wait(handoff_bar(cw ^ 1), hoph);
        hoph ^= 1;
      }
      if (p.res && issuer) {                      // the residual loads under the mainloop
        bulk_wait_read();                         // once the previous tile's output has left the staging box
        mbar_expect_tx(res_bar(rb), p.o_bytes * ((SPLIT && p.res_lo) ? 2u : 1u));
#pragma unroll
        for (int k = 0; k < NT / CW; ++k) {
          tma_load_4d(ob + k * CB_BYTES, &p.r_hi, res_bar(rb), c_out0 + k * CW, w0, h0, n0);
          if (SPLIT && p.res_lo) tma_load_4d(ob + p.o_plane + k * CB_BYTES, &p.r_lo, res_bar(rb), c_out0 + k * CW, w0, h0, n0);
        }
      }
#pragma unroll
      for (int m = 0; m < MT; ++m) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[m][i] = 0.f;
#pragma unroll
        for (int i = 0; i < NLO; ++i) acl[m][i] = 0.f;
      }
      const uint32_t row0 = PP ? 0u : (uint32_t)cw * 64;   // first tile row of accumulator set 0
      int prev = -1, prev_h = -1;                 // stages the last committed wgmma group reads (prev_h: halo, if its last)
      if (RES) {                                  // every operand is in shared memory once the halo band has landed
        mbar_wait(hfull_bar(hs), hph);
#ifdef SHAPY_CONV_STAMPS
        st0 = clock64();
#endif
        const uint32_t hb = smem_base + h_stage * hs + row0 * 32;
        auto fence_accs = [&]() {
#pragma unroll
          for (int m = 0; m < MT; ++m) {
#pragma unroll
            for (int i = 0; i < NACC; ++i) reg_fence(acc[m][i]);
#pragma unroll
            for (int i = 0; i < NLO; ++i) reg_fence(acl[m][i]);
          }
        };
        fence_accs();
        wgmma_fence();
        // all k16 steps of the tile in the halo path's order (tap-major, then slice) as one group
        auto issue_res = [&](auto slices) {
#pragma unroll
          for (int tap = 0; tap < 9; ++tap) {
            const uint32_t a_tap = hb + (uint32_t)((tap / 3) * p.TW + tap % 3) * 32;   // 32-byte rows from ky Wp + kx
#pragma unroll
            for (int j = 0; j < decltype(slices)::value; ++j) {
              const uint64_t b = wgmma_desc<16>(ring_base + (uint32_t)(tap * decltype(slices)::value + j) * PARTS * p.b_tx);
#pragma unroll
              for (int m = 0; m < MT; ++m) {
                const uint32_t a_addr = a_tap + j * p.h_slice + m * 64 * 32;
                if (SPLIT) {
                  wgmma_f16<2 * NT>(acc[m], wgmma_desc<16>(a_addr), b, 1);
                  wgmma_f16<NT>(acl[m], wgmma_desc<16>(a_addr + p.h_plane), b, 1);
                } else {
                  wgmma_f16<NT>(acc[m], wgmma_desc<16>(a_addr), b, 1);
                }
              }
            }
          }
          wgmma_commit();
        };
        switch (p.cin / 16) {
          case 1: issue_res(std::integral_constant<int, 1>()); break;
          case 2: issue_res(std::integral_constant<int, 2>()); break;
          case 3: issue_res(std::integral_constant<int, 3>()); break;
          default: issue_res(std::integral_constant<int, 4>()); break;
        }
        fence_accs();
        prev_h = hs;
        if (++hs == p.hstages) { hs = 0; hph ^= 1; }
      }
#pragma unroll 1
      for (int it = 0; it < (RES ? 0 : iters); ++it) {
        int tap, cb;
        decode(it, tap, cb);
        const int nks = cb == p.kpt - 1 ? p.ks_last : KCH / 16;
        uint32_t a_addr, a_lo_off;
#ifdef SHAPY_CONV_STAMPS
        const long long st_w0 = clock64();
#endif
        if (HALO) {
          if (tap == 0) mbar_wait(hfull_bar(hs), hph);
          // tap (ky, kx): the halo rows from ky * Wp + kx on (p.TW is the pitch Wp of the padded grid)
          a_addr = smem_base + h_stage * hs + (row0 + (uint32_t)((tap / 3) * p.TW + tap % 3)) * (KCH * 2);
          a_lo_off = p.h_plane;
        }
        mbar_wait(full_bar(s), ph);
#ifdef SHAPY_CONV_STAMPS
        if (it == 0) st0 = clock64(); else st_w += clock64() - st_w0;
#endif
        const uint32_t kb = ring_base + kblk_bytes * s;
        if (!HALO) { a_addr = kb + row0 * KCH * 2; a_lo_off = A_BLK; }
        uint64_t a[MT], al[MT];
#pragma unroll
        for (int m = 0; m < MT; ++m) {            // set m: tile rows row0 + 64 m on
          a[m] = wgmma_desc<KCH>(a_addr + m * 64 * KCH * 2);
          al[m] = wgmma_desc<KCH>(a_addr + m * 64 * KCH * 2 + a_lo_off);
        }
        const uint64_t b = wgmma_desc<KCH>(kb + (HALO ? 0u : A_BLK * PARTS));
#pragma unroll
        for (int m = 0; m < MT; ++m) {
#pragma unroll
          for (int i = 0; i < NACC; ++i) reg_fence(acc[m][i]);
#pragma unroll
          for (int i = 0; i < NLO; ++i) reg_fence(acl[m][i]);
        }
        wgmma_fence();
        // the first nks k16 steps (channels past cin are zero-filled, nothing to add): one straight-line wgmma run and
        // its commit per count, so no branch joins inside a group (a join there makes ptxas add a dummy wgmma)
        auto issue = [&](auto nks_c) {
#pragma unroll
          for (int ks = 0; ks < decltype(nks_c)::value; ++ks) {   // +32 bytes along K = +2 descriptor units
#pragma unroll
            for (int m = 0; m < MT; ++m) {
              if (SPLIT) {
                wgmma_f16<2 * NT>(acc[m], a[m] + 2 * ks, b + 2 * ks, 1);   // [D0 | D1] += A_hi . [B_hi | B_lo]^T
                wgmma_f16<NT>(acl[m], al[m] + 2 * ks, b + 2 * ks, 1);       // D1' += A_lo . B_hi^T
              } else {
                wgmma_f16<NT>(acc[m], a[m] + 2 * ks, b + 2 * ks, 1);
              }
            }
          }
          wgmma_commit();
        };
        static_assert(KCH / 16 == 4, "k16 steps per k-block");
        switch (nks) {
          case 1: issue(std::integral_constant<int, 1>()); break;
          case 2: issue(std::integral_constant<int, 2>()); break;
          case 3: issue(std::integral_constant<int, 3>()); break;
          default: issue(std::integral_constant<int, 4>()); break;
        }
#pragma unroll
        for (int m = 0; m < MT; ++m) {
#pragma unroll
          for (int i = 0; i < NACC; ++i) reg_fence(acc[m][i]);
#pragma unroll
          for (int i = 0; i < NLO; ++i) reg_fence(acl[m][i]);
        }
        wgmma_wait<1>();                          // the previous stage's wgmmas have read their operands
        if (prev >= 0 && t == 0) {
          mbar_arrive(empty_bar(prev));
          if (prev_h >= 0) mbar_arrive(hempty_bar(prev_h));
        }
        prev = s;
        prev_h = -1;
        if (HALO && tap == taps - 1) {            // the last tap of this halo buffer
          prev_h = hs;
          if (++hs == p.hstages) { hs = 0; hph ^= 1; }
        }
        if (++s == p.stages) { s = 0; ph ^= 1; }
      }
      if (PP && t == 0) mbar_arrive(handoff_bar(cw));
#ifdef SHAPY_CONV_STAMPS
      st1 = clock64();
#endif
      wgmma_wait<0>();
#pragma unroll
      for (int m = 0; m < MT; ++m) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) reg_fence(acc[m][i]);
#pragma unroll
        for (int i = 0; i < NLO; ++i) reg_fence(acl[m][i]);
      }
      if (t == 0) {
        if (prev >= 0) mbar_arrive(empty_bar(prev));
        if (prev_h >= 0) mbar_arrive(hempty_bar(prev_h));
      }
      if (PP) skip_tile();
#ifdef SHAPY_CONV_STAMPS
      st2 = clock64();
#endif

      // ---- epilogue: this thread holds rows r0 and r0 + 8 of each m64 set, two adjacent columns of every 8-column group
      // (the mma C fragment).  The outputs are staged in shared memory over the residual, which TMA loaded there during
      // the mainloop, 16 x 16 blocks at a time with ldmatrix / stmatrix (each element read and written by the same
      // thread), and leave with one TMA store per column box and plane.
      float2 bq[NT / 8];
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) bq[j] = __ldg(reinterpret_cast<const float2 *>(p.bias + c_out0 + 8 * j + 2 * (lane & 3)));
      if (p.res) {
        mbar_wait(res_bar(rb), rph);
        rph ^= 1;
      } else {
        if (issuer) bulk_wait_read();
        named_bar_sync(ebar, ethreads);
      }
#pragma unroll
      for (int m = 0; m < MT; ++m) {
        // this lane's row address serves matrix lane / 8 of each x4: rows + 8 for odd matrices, channels + 8 for 2, 3
        const int row = (int)row0 + m * 64 + warp * 16 + (lane & 7) + (lane & 8);
        const int dw = row % p.TW, dh = (row / p.TW) % p.TH, dn = row / (p.TW * p.TH);
        // a tile row without a slot in the box (the padded grid's junk columns, rows past the box) goes to box row 127:
        // the box then has fewer than 128 rows, so no slot is there.  Rows past Ho / N have slots; TMA drops them.
        const uint32_t br = dn < p.TN && dw < p.o_bw ? (uint32_t)((dn * p.TH + dh) * p.o_bw + dw) : 127u;
#pragma unroll
        for (int jp = 0; jp < NT / 16; ++jp) {
          const uint32_t o = br * (CW * 2) + (uint32_t)((16 * jp) % CW / 8 + (lane >> 4)) * 16;
          const uint32_t a = ob + (16 * jp / CW) * CB_BYTES + (o ^ (((o >> 7) & (CW / 8 - 1)) << 4));   // the TMA swizzle
          uint32_t rh[4], rl[4], sh[4], sl[4];
          if (p.res) {
            ldmatrix_x4(rh, a);
            if (SPLIT && p.res_lo) ldmatrix_x4(rl, a + p.o_plane);
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {            // matrix k: rows + 8 (k & 1), 8-column group 2 jp + (k >> 1)
            const int j = 2 * jp + (k >> 1);
            const int i = 4 * j + 2 * (k & 1);
            float r0 = acc[m][i], r1 = acc[m][i + 1];
            if (SPLIT) {
              r0 += (acc[m][NT / 2 + i] + acl[m][SPLIT ? i : 0]) * kLoInv;
              r1 += (acc[m][NT / 2 + i + 1] + acl[m][SPLIT ? i + 1 : 0]) * kLoInv;
            }
            r0 += bq[j].x; r1 += bq[j].y;
            if (p.res) {
              const __half2 h = *reinterpret_cast<const __half2 *>(&rh[k]);
              r0 += __low2float(h); r1 += __high2float(h);
              if (SPLIT && p.res_lo) {
                const __half2 l = *reinterpret_cast<const __half2 *>(&rl[k]);
                r0 += __low2float(l) * kLoInv; r1 += __high2float(l) * kLoInv;
              }
            }
            if (p.relu) { r0 = fmaxf(r0, 0.f); r1 = fmaxf(r1, 0.f); }
            __half h0_, h1_, l0_, l1_;
            split_store(r0, h0_, l0_);
            split_store(r1, h1_, l1_);
            const __half2 hv = __halves2half2(h0_, h1_), lv = __halves2half2(l0_, l1_);
            sh[k] = *reinterpret_cast<const uint32_t *>(&hv);
            sl[k] = *reinterpret_cast<const uint32_t *>(&lv);
          }
          stmatrix_x4(a, sh);
          if (SPLIT && p.out_lo) stmatrix_x4(a + p.o_plane, sl);
        }
      }
      fence_proxy_async_smem();                   // the staged tile -> global memory; TMA drops rows past the map
      named_bar_sync(ebar, ethreads);
      if (issuer) {
#pragma unroll
        for (int k = 0; k < NT / CW; ++k) {
          tma_store_4d(&p.o_hi, ob + k * CB_BYTES, c_out0 + k * CW, w0, h0, n0);
          if (SPLIT && p.out_lo) tma_store_4d(&p.o_lo, ob + p.o_plane + k * CB_BYTES, c_out0 + k * CW, w0, h0, n0);
        }
        bulk_commit();
      }
#ifdef SHAPY_CONV_STAMPS
      if (t == 0) {                               // warp 0's end of the epilogue
        const long long st3 = clock64();
        atomicAdd(&g_conv_stamps[0], (unsigned long long)(st0 - st_end));
        atomicAdd(&g_conv_stamps[1], (unsigned long long)(st1 - st0));
        atomicAdd(&g_conv_stamps[2], (unsigned long long)(st2 - st1));
        atomicAdd(&g_conv_stamps[3], (unsigned long long)(st3 - st2));
        atomicAdd(&g_conv_stamps[4], 1ull);
        atomicAdd(&g_conv_stamps[5], (unsigned long long)st_w);
        st_end = st3;
        st_w = 0;
      }
#endif
    }
    if (issuer) bulk_wait();                      // the last stores have completed before shared memory is released
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
  bool split, halo, pingpong, resident;
  dim3 grid;
  size_t smem;
  double tma_bytes, mma_flops;   // per launch, as planned: TMA loads of both operands, tensor-core FLOPs issued
};

// SHAPY_CONV_HALO=0: every plan of WGMMA_AUTO takes the per-tap path
static bool halo_enabled() {
  static const bool v = []() { const char *e = getenv("SHAPY_CONV_HALO"); return !(e && e[0] == '0'); }();
  return v;
}

// SHAPY_CONV_PINGPONG=0: every plan without a forced schedule takes the cooperative one
static bool pingpong_enabled() {
  static const bool v = []() { const char *e = getenv("SHAPY_CONV_PINGPONG"); return !(e && e[0] == '0'); }();
  return v;
}

// SHAPY_CONV_RESIDENT=0: no plan of WGMMA_AUTO takes the weight-resident path
static bool resident_enabled() {
  static const bool v = []() { const char *e = getenv("SHAPY_CONV_RESIDENT"); return !(e && e[0] == '0'); }();
  return v;
}

// the ping-pong schedule holds two m64 accumulator sets per consumer thread
static bool pingpong_fits(bool split, int nt) { return split ? nt <= 64 : nt <= 128; }

#ifdef SHAPY_CONV_STAMPS
void wgmma_stamps_reset() {
  const unsigned long long z[6] = {0, 0, 0, 0, 0, 0};
  cudaMemcpyToSymbol(g_conv_stamps, z, sizeof(z));
}
void wgmma_stamps_print(const WgmmaPlan *pl) {
  unsigned long long v[6];
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(v, g_conv_stamps, sizeof(v));
  const double n = v[4] ? (double)v[4] : 1.0;
  fprintf(stderr,
          "[stamps] %s NT %d: %llu warpgroup-tiles, cycles per tile: wait %.0f mainloop %.0f (operand waits %.0f) "
          "drain %.0f epilogue %.0f\n",
          pl->pingpong ? "ping-pong" : "cooperative", pl->NT, v[4], v[0] / n, v[1] / n, v[5] / n, v[2] / n, v[3] / n);
}
#endif

void wgmma_plan_stats(const WgmmaPlan *pl, double *tma_bytes, double *mma_flops) {
  *tma_bytes = pl->tma_bytes;
  *mma_flops = pl->mma_flops;
}

void wgmma_plan_describe(const WgmmaPlan *pl, int *path, int *pingpong, int *nt) {
  *path = pl->resident ? WGMMA_RESIDENT : (pl->halo ? WGMMA_HALO : WGMMA_PER_TAP);
  *pingpong = pl->pingpong ? 1 : 0;
  *nt = pl->NT;
}

static const int kNts[] = {128, 96, 64, 48, 32, 16};   // cout tiles with a kernel instantiation

bool wgmma_supported(const ConvW &w, const ActView &in, const ActView &out) {
  if (w.cin % 16 || w.cout % 16) return false;
  if (!((w.ksize == 3 || w.ksize == 1) && (w.stride == 1 || (w.stride == 2 && w.ksize == 3)))) return false;
  if (w.stride == 2 && (in.H % 2 || in.W % 2)) return false;
  if (in.Ctot % 8 || in.coff % 8 || out.Ctot % 8 || out.coff % 8) return false;
  if (out.W > 128 && out.W % 128) return false;
  return get_encode() != nullptr;
}

WgmmaPlan *wgmma_plan_create(const ConvW &w, const ActView &in, const ActView &out, const ActView *res, bool relu,
                             int path, int nt) {
  if (!wgmma_supported(w, in, out)) {
    set_error("wgmma_plan_create: unsupported convolution (cin %d cout %d k %d s %d)", w.cin, w.cout, w.ksize, w.stride);
    return nullptr;
  }
  const int data_path = path & (WGMMA_PER_TAP | WGMMA_HALO | WGMMA_RESIDENT);
  const int sched = path & (WGMMA_COOP | WGMMA_PINGPONG);
  const bool split = in.lo != nullptr;
  if (nt && (std::find(std::begin(kNts), std::end(kNts), nt) == std::end(kNts) || w.cout % nt || (split && nt > 96) ||
             (sched == WGMMA_PINGPONG && !pingpong_fits(split, nt)) || (data_path == WGMMA_RESIDENT && nt != w.cout))) {
    set_error("wgmma_plan_create: no kernel for cout tile %d (cin %d cout %d, split %d)", nt, w.cin, w.cout, (int)split);
    return nullptr;
  }
  auto *pl = new WgmmaPlan();
  memset(&pl->p, 0, sizeof(pl->p));
  WgmmaParams &p = pl->p;
  const int PARTS = split ? 2 : 1;
  pl->split = split;
  const int sms = sm_count();
  p.TW = std::min(out.W, 128);
  p.TH = std::max(1, std::min(out.H, 128 / p.TW));
  p.TN = (p.TW == out.W && p.TH == out.H) ? std::max(1, std::min(out.N, 128 / (p.TW * p.TH))) : 1;
  p.tiles_w = ceil_div(out.W, p.TW); p.tiles_h = ceil_div(out.H, p.TH); p.tiles_n = ceil_div(out.N, p.TN);
  p.cin = w.cin; p.cout = w.cout; p.ksize = w.ksize; p.stride = w.stride;
  p.kpt = ceil_div(w.cin, KCH);
  p.ks_last = (w.cin - (p.kpt - 1) * KCH) / 16;
  // Halo path: 3x3 stride 1, bands of TH rows of one image on the padded grid of pitch Wp.  TH is balanced over the
  // image (56 -> 2, 28 -> 4, 14 -> 7 rather than 8).  Taken where it is not more M tiles than the per-tap tiling and
  // loads fewer activation bytes; multi-image per-tap tiles (7 x 7 maps) stay per-tap.
  // A halo slot holds the rows the furthest tap reads, 128 + 2 Wp + 2: rows past the (TH + 2) Wp the TMA writes are
  // stale, but only discarded output rows read them (wgmma rows are independent).
  const int Wp = out.W + 2;
  const uint32_t h_plane = (uint32_t)align_up((size_t)(128 + 2 * Wp + 2) * KCH * 2, 1024);
  {
    // two halo slots, at least two weight slots and the staging box of the widest cout tile must fit the shared-memory
    // budget
    const int nt_max = std::min(w.cout, split ? 96 : 128);
    const size_t b_max = align_up((size_t)nt_max * KCH * 2 * PARTS, 1024);
    const bool possible = w.ksize == 3 && w.stride == 1 && Wp <= 128 &&
                          2 * (h_plane * PARTS + b_max) + (size_t)nt_max * 128 * 2 * PARTS <= 222 * 1024;
    bool better = false;
    int th = 0;
    if (possible) {
      const int per = 128 / Wp;
      th = ceil_div(out.H, ceil_div(out.H, per));
      const double pt_tiles = (double)p.tiles_w * p.tiles_h * p.tiles_n, h_tiles = (double)ceil_div(out.H, th) * out.N;
      const double pt_a = pt_tiles * 9 * p.TW * p.TH * p.TN, h_a = h_tiles * Wp * (th + 2);   // rows loaded per k-block
      better = p.TN == 1 && h_tiles <= pt_tiles && h_a < pt_a;
    }
    if ((data_path == WGMMA_HALO || data_path == WGMMA_RESIDENT) && !possible) {
      set_error("wgmma_plan_create: no halo path for cin %d cout %d k %d s %d %dx%d", w.cin, w.cout, w.ksize, w.stride,
                out.H, out.W);
      delete pl;
      return nullptr;
    }
    pl->halo = data_path == WGMMA_HALO || data_path == WGMMA_RESIDENT || (data_path == WGMMA_AUTO && better && halo_enabled());
    if (pl->halo) {
      p.TW = Wp; p.TH = th; p.TN = 1;
      p.tiles_w = 1; p.tiles_h = ceil_div(out.H, th); p.tiles_n = out.N;
    }
  }
  {
    // Cout tile and consumer schedule: the pair of least modelled time, the model fitted to the launch times of every
    // candidate of every HRNet layer in both modes (tools/conv_plan_sweep.py, H100 SXM at 700 W, README).  One k16 step
    // of a 128-row tile is two m64nNk16 (split: N = 2 NT and N = NT), each the larger of its shared-memory operand reads
    // (2 KB of A and N x 32 B of B at 128 B/cycle) and N / 2 tensor cycles, plus 32 cycles of issue, over the k16 steps
    // actually issued; a tile adds 1 000 cycles of operand wait, drain and staged epilogue.  Cooperative: each wave of
    // tiles pays mainloop + epilogue.  Ping-pong: a consumer's epilogue runs under the other's mainloop, so a wave pays
    // the larger of the two, plus one exposed epilogue.  One consumer issuing both m64 halves takes sqrt(64 / NT) x the
    // cooperative mainloop in split mode, 0.3 x more on the halo path with several channel blocks (c96, c192: the
    // consumers' tiles alternate over the 2-slot halo ring), and 0.9 x in fp16.  Waves count whole: a partial wave costs
    // a full tile in the measured launches (384 -> 384 @7² fp16: NT 32 at 1.45 waves takes 1.8 x NT 48 at 0.97).
    const double m_tiles = (double)p.tiles_w * p.tiles_h * p.tiles_n;
    const int steps = w.ksize * w.ksize * ((p.kpt - 1) * (KCH / 16) + p.ks_last);
    auto mma_cyc = [](double n) { return 2.0 * std::max((2048.0 + 32.0 * n) / 128.0, n * 0.5) + 32.0; };
    auto main_cyc = [&](int c) { return (split ? mma_cyc(2.0 * c) + mma_cyc(c) : mma_cyc(c)) * steps; };
    auto rounds = [&](int c) { return std::ceil(m_tiles * (w.cout / c) / sms); };
    const double epi = 1000.0;
    const double pp_halo = pl->halo && p.kpt > 1 ? 0.3 : 0.0;
    auto coop_cost = [&](int c) { return rounds(c) * (main_cyc(c) + epi); };
    auto pp_cost = [&](int c) {
      const double slow = split ? std::sqrt(64.0 / c) + pp_halo : 0.9;
      return rounds(c) * std::max(slow * main_cyc(c), epi) + epi;
    };
    const bool pp_ok = sched == WGMMA_PINGPONG || (sched == 0 && pingpong_enabled());
    double best = 1e30;
    for (int c : kNts) {
      if (w.cout % c || (split && c > 96) || (nt && c != nt)) continue;   // split: 3 NT / 2 accumulators per thread must fit 232 registers
      if (sched != WGMMA_PINGPONG && coop_cost(c) < best) { best = coop_cost(c); pl->NT = c; pl->pingpong = false; }
      if (pp_ok && pingpong_fits(split, c) && pp_cost(c) < best) { best = pp_cost(c); pl->NT = c; pl->pingpong = true; }
    }
  }
  // Weight-resident path: a halo layer with one cout tile (kernels exist for cout 48 and 64) and cin <= 64, in 16-channel
  // slices.  Forced, it takes that cout tile and the requested (or the planner's) schedule.
  const bool res_shape = pl->halo && w.cin % 16 == 0 && w.cin <= KCH && (w.cout == 48 || w.cout == 64);
  if (data_path == WGMMA_RESIDENT) {
    if (!res_shape) {
      set_error("wgmma_plan_create: no weight-resident path for cin %d cout %d", w.cin, w.cout);
      delete pl;
      return nullptr;
    }
    pl->NT = w.cout;
    pl->pingpong = sched == WGMMA_PINGPONG || (sched == 0 && pingpong_enabled() && pingpong_fits(split, pl->NT));
  }
  pl->resident = res_shape && pl->NT == w.cout && (data_path == WGMMA_RESIDENT || (data_path == WGMMA_AUTO && resident_enabled()));
  p.relu = relu;
  p.pdl_late = 1;
  // output staging: one box per plane (ping-pong: per consumer and plane) of 128 rows x NT; the output tile without the
  // padded grid's junk columns fills its first o_bw x TH x TN rows
  p.o_bw = pl->halo ? out.W : p.TW;
  p.o_bytes = (uint32_t)pl->NT * p.o_bw * p.TH * p.TN * 2;
  p.o_plane = (uint32_t)pl->NT * 128 * 2;
  auto staging = [&]() { return (pl->pingpong ? 2 : 1) * (size_t)p.o_plane * PARTS; };
  if (pl->resident) {
    // two halo slots of cin / 16 slices per plane, each slice the rows the furthest tap reads in 32-byte rows, the
    // whole weight set, the 1024-aligned staging boxes: up to the 227 KB a CTA may own
    const int S = w.cin / 16;
    p.h_slice = (uint32_t)align_up((size_t)(128 + 2 * Wp + 2) * 32, 256);
    p.h_plane = p.h_slice * S;
    p.hstages = 2;
    p.stages = 0;
    p.b_tx = (uint32_t)pl->NT * 32;
    p.w_bytes = 9u * S * PARTS * p.b_tx;
    p.a_bytes = (uint32_t)p.TW * (p.TH + 2) * w.cin * 2;
    pl->smem = align_up((size_t)p.h_plane * PARTS * p.hstages + p.w_bytes, 1024) + staging() + 8 * (2 * p.hstages + 5) +
               1024;
    if (pl->smem > 227 * 1024) {
      if (data_path == WGMMA_RESIDENT) {
        set_error("wgmma_plan_create: the weight-resident path does not fit shared memory (cin %d cout %d, %zu B)",
                  w.cin, w.cout, pl->smem);
        delete pl;
        return nullptr;
      }
      pl->resident = false;
    }
  }
  // Channels per TMA box.  With cin < 64 a box of cin channels fills the first cin * 2 bytes of each 128-byte row; a
  // 64-channel box would also write the zero fill past cin, which no issued k16 step reads, and the c48 mainloop is
  // short of shared-memory bandwidth rather than of loaded stages (README).
  // The resident path loads 16-channel boxes into 32-byte rows.
  const int kbox = pl->resident ? 16 : (p.kpt == 1 ? w.cin : KCH);
  if (!pl->resident) {
    // per k-block TMA bytes of one plane: the A box (halo path: the band with its halo rows) and the weight box
    const int a_rows = pl->halo ? p.TW * (p.TH + 2) : p.TW * p.TH * p.TN;
    p.a_bytes = (uint32_t)a_rows * kbox * 2;
    p.b_bytes = (uint32_t)pl->NT * KCH * 2;
    p.b_tx = (uint32_t)pl->NT * kbox * 2;
    p.b_stride = (uint32_t)align_up((size_t)p.b_bytes * PARTS, 1024);
  }
  // one persistent CTA per SM owns (almost) all of its 227 KB of shared memory: the staging box(es) and the rings take
  // up to 222 KB
  auto plan_smem = [&]() {
    const size_t budget = 222 * 1024 - staging();
    if (pl->halo) {
      p.h_plane = h_plane;
      p.hstages = 2;
      const size_t halo = (size_t)h_plane * PARTS * p.hstages;
      p.stages = halo + 2 * p.b_stride <= budget ? (int)std::min<size_t>(8, (budget - halo) / p.b_stride) : 0;
      pl->smem = halo + staging() + (size_t)p.b_stride * p.stages + 16 * (p.stages + p.hstages + 2) + 1024;
    } else {
      const size_t stage = 128u * KCH * 2 * PARTS + p.b_stride;
      p.stages = (int)std::min<size_t>(8, budget / stage);
      pl->smem = staging() + stage * p.stages + 16 * (p.stages + 2) + 1024;
    }
    // a planned ping-pong needs three weight slots: with two, the ring stalls the mainloop (split b64, NT 64: 111.8
    // against 103.9 us cooperative)
    return p.stages >= (pl->pingpong && sched != WGMMA_PINGPONG ? 3 : 2);
  };
  if (!pl->resident && !plan_smem()) {
    if (sched == WGMMA_PINGPONG) {
      set_error("wgmma_plan_create: no room for the ping-pong staging boxes (cin %d cout %d %dx%d)", w.cin, w.cout,
                out.H, out.W);
      delete pl;
      return nullptr;
    }
    pl->pingpong = false;                         // the cooperative schedule at the same cout tile
    if (!plan_smem()) {
      set_error("wgmma_plan_create: no room for the ring and the staging box (cin %d cout %d %dx%d)", w.cin, w.cout,
                out.H, out.W);
      delete pl;
      return nullptr;
    }
  }
  p.bias = w.bias;
  p.out_lo = out.lo != nullptr;
  p.res = res != nullptr; p.res_lo = res && res->lo;
  const int items = p.tiles_w * p.tiles_h * p.tiles_n * (w.cout / pl->NT);
  pl->grid = dim3(even_grid(items, sms), 1);
  {
    const int taps = w.ksize * w.ksize;
    const double a_loads = pl->halo ? p.kpt : taps * p.kpt;   // A boxes per work item
    pl->tma_bytes = pl->resident ? (double)items * PARTS * p.a_bytes + (double)pl->grid.x * p.w_bytes   // weights once per CTA
                                 : (double)items * PARTS * (a_loads * p.a_bytes + (double)taps * p.kpt * p.b_tx);
    const double k = (double)taps * ((p.kpt - 1) * KCH + p.ks_last * 16);   // K actually issued per work item
    pl->mma_flops = (double)items * 2.0 * 128 * pl->NT * k * (split ? 3 : 1);
  }
  if (getenv("SHAPY_CONV_DEBUG"))
    fprintf(stderr,
            "[wgmma] cin %d cout %d k %d s %d %dx%d N %d: %s %s NT %d tile %dx%dx%d grid %d stages %d+%d, staging "
            "%dx%ux%u B, smem %zu B, TMA %.1f MB, MMA %.2f GFLOP\n",
            w.cin, w.cout, w.ksize, w.stride, out.H, out.W, out.N,
            pl->resident ? "resident" : (pl->halo ? "halo" : "per-tap"),
            pl->pingpong ? "ping-pong" : "cooperative", pl->NT, p.TW, p.TH, p.TN, pl->grid.x, p.hstages, p.stages,
            pl->pingpong ? 2 : 1, (unsigned)PARTS, p.o_plane, pl->smem, pl->tma_bytes * 1e-6, pl->mma_flops * 1e-9);
  bool ok = true;
  const int swz = pl->resident ? 16 : KCH;   // row width of the shared-memory operands in channels: picks the swizzle
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
    // halo path: the band plus one row above and below; p.TW = Wp already spans the two padding columns
    cuuint32_t box[4] = {(cuuint32_t)kbox, (cuuint32_t)p.TW, (cuuint32_t)(p.TH + (pl->halo ? 2 : 0)), (cuuint32_t)p.TN};
    ok = ok && encode(&p.a_hi[mi], in.hi + off, 4, dims, strides, box, swz);
    if (split) ok = ok && encode(&p.a_lo[mi], in.lo + off, 4, dims, strides, box, swz);
  }
  if (ok) {
    cuuint64_t dims[3] = {(cuuint64_t)w.cin, (cuuint64_t)w.cout, (cuuint64_t)(w.ksize * w.ksize)};
    cuuint64_t strides[2] = {(cuuint64_t)w.cin * 2, (cuuint64_t)w.cin * w.cout * 2};
    cuuint32_t box[3] = {(cuuint32_t)kbox, (cuuint32_t)pl->NT, 1};
    ok = ok && encode(&p.b_hi, w.w_hi, 3, dims, strides, box, swz);
    if (split) ok = ok && encode(&p.b_lo, w.w_lo, 3, dims, strides, box, swz);
  }
  // epilogue maps: the output view (out_coff / out_ctot as the activation maps carry coff / Ctot) and the residual
  // view, in column boxes of the staged tile with the swizzle of their rows
  auto view_map = [&](CUtensorMap *m, const __half *base, const ActView &v) {
    const int cw = stage_cw(pl->NT);
    cuuint64_t dims[4] = {(cuuint64_t)w.cout, (cuuint64_t)v.W, (cuuint64_t)v.H, (cuuint64_t)v.N};
    cuuint64_t strides[3] = {(cuuint64_t)v.Ctot * 2, (cuuint64_t)v.W * v.Ctot * 2, (cuuint64_t)v.H * v.W * v.Ctot * 2};
    cuuint32_t box[4] = {(cuuint32_t)cw, (cuuint32_t)p.o_bw, (cuuint32_t)p.TH, (cuuint32_t)p.TN};
    return encode(m, base + v.coff, 4, dims, strides, box, cw);
  };
  if (ok) {
    ok = view_map(&p.o_hi, out.hi, out) && (!out.lo || view_map(&p.o_lo, out.lo, out));
    if (ok && res) ok = view_map(&p.r_hi, res->hi, *res) && (!split || !res->lo || view_map(&p.r_lo, res->lo, *res));
  }
  if (!ok) { delete pl; return nullptr; }
  return pl;
}

void wgmma_plan_destroy(WgmmaPlan *p) { delete p; }

template <bool SPLIT, int NT, bool HALO, bool PP, bool RES = false>
static int launch_h(const WgmmaPlan *pl, cudaStream_t st, bool pdl) {
  static std::atomic<unsigned long long> attr_done{0};
  auto kernel = conv_wgmma_kernel<SPLIT, NT, HALO, PP, RES>;
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

template <bool SPLIT, int NT, bool PP>
static int launch_s(const WgmmaPlan *pl, cudaStream_t st, bool pdl) {
  if (pl->resident) {
    if constexpr (NT == 48 || NT == 64) return launch_h<SPLIT, NT, true, PP, true>(pl, st, pdl);
    set_error("wgmma engine: no weight-resident kernel for NT %d", NT);
    return SHAPY_ERR_STATE;
  }
  return pl->halo ? launch_h<SPLIT, NT, true, PP>(pl, st, pdl) : launch_h<SPLIT, NT, false, PP>(pl, st, pdl);
}

template <bool SPLIT, int NT>
static int launch_t(const WgmmaPlan *pl, cudaStream_t st, bool pdl) {
  if (!pl->pingpong) return launch_s<SPLIT, NT, false>(pl, st, pdl);
  if constexpr (SPLIT ? NT <= 64 : NT <= 128) return launch_s<SPLIT, NT, true>(pl, st, pdl);   // pingpong_fits
  set_error("wgmma engine: no ping-pong kernel for NT %d in split mode", NT);
  return SHAPY_ERR_STATE;
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
