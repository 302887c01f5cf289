// Shared declarations of the HRNet convolution engines.
//
// Activation storage ("split-fp16 planes"): every activation is an NHWC tensor held as an fp16
// `hi` plane and, in parity mode, a second fp16 `lo` plane with  x = hi + lo / 2048.  The pair carries
// ~22 mantissa bits, so three fp16 tensor-core MMAs (hi*hi, hi*lo, lo*hi; lo*lo is < 2^-22 relative and
// dropped) reproduce an fp32 convolution to ~1e-6 -- enough for the 1e-4 end-to-end bar through ~110
// layers -- at 3x (not 6x, as 3xTF32 would cost) the fp16 tensor rate and 4 B / element of HBM traffic.
// Mode 0 keeps only the `hi` plane: plain fp16 operands, fp32 accumulation (BASELINE config 2).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace shapy {

constexpr float kLoScale = 2048.0f;
constexpr float kLoInv = 1.0f / 2048.0f;

struct ActView {
  __half *hi = nullptr, *lo = nullptr;  // lo == nullptr in mode 0
  int N = 0, H = 0, W = 0, C = 0;       // logical extent of the view
  int Ctot = 0, coff = 0;               // channels per pixel in memory, first channel of the view
};

struct ConvW {
  __half *w_hi = nullptr, *w_lo = nullptr;  // [taps][cout][cin], BN scale folded in
  float *bias = nullptr;                    // [cout], BN shift (+ conv bias) folded
  float *w_f32 = nullptr;                   // stem only: [27][cout]
  int cin = 0, cout = 0, ksize = 0, stride = 0;
};

// 32 consecutive bytes as two 16-byte accesses (16-byte aligned addresses)
__device__ __forceinline__ void ldg32b(const void *p, uint4 &a, uint4 &b) {
  const uint4 *q = reinterpret_cast<const uint4 *>(p);
  a = __ldg(q);
  b = __ldg(q + 1);
}
__device__ __forceinline__ void stg32b(void *p, const uint4 &a, const uint4 &b) {
  uint4 *q = reinterpret_cast<uint4 *>(p);
  q[0] = a;
  q[1] = b;
}

__device__ __forceinline__ void split_store(float v, __half &hi, __half &lo) {
  v = fminf(fmaxf(v, -65504.f), 65504.f);
  hi = __float2half_rn(v);
  lo = __float2half_rn((v - __half2float(hi)) * kLoScale);
}

// ---- engines (each returns SHAPY_OK or an error code; all launches on `st`)
int launch_conv_simt(const ConvW &w, const ActView &in, const ActView &out, const ActView *res, bool relu,
                     cudaStream_t st);
int launch_stem(const ConvW &w, const float *images, const float *const *images_cell, int N, int H, int W,
                const ActView &out, cudaStream_t st);
int launch_fuse(const ActView *ins, const int *shifts, int n_in, const ActView &out, bool relu, cudaStream_t st);
int launch_pool(const ActView &in, float *feats, float *const *feats_cell, cudaStream_t st);
int launch_set_io_cells(void **cells, const float *images, float *feats, cudaStream_t st);   // cells[0] = images, [1] = feats
int launch_nhwc_split(const float *x, const ActView &out, cudaStream_t st);          // fp32 NHWC -> planes
int launch_nhwc_merge(const ActView &in, float *y, bool to_nchw, cudaStream_t st);   // planes -> fp32

// TMA + wgmma implicit-GEMM engine (conv_wgmma.cu).  `WgmmaPlan` holds the TMA descriptors + geometry of one launch.
struct WgmmaPlan;
bool wgmma_supported(const ConvW &w, const ActView &in, const ActView &out);
WgmmaPlan *wgmma_plan_create(const ConvW &w, const ActView &in, const ActView &out, const ActView *res, bool relu);
void wgmma_plan_destroy(WgmmaPlan *p);
int wgmma_plan_launch(const WgmmaPlan *p, cudaStream_t st, bool pdl);   // pdl: programmatic dependent launch

}  // namespace shapy
