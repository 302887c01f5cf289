// SIMT (CUDA-core, fp32 accumulate) engines of the HRNet path: the 3-channel stem convolution, the
// multi-resolution fuse sum, the final spatial mean, layout converters, and a generic implicit-GEMM
// convolution on the same split-fp16 planes the wgmma engine uses.  The SIMT convolution is the
// debug / cross-check engine (`engine = 1`): identical operands and rounding points, no tensor cores.
// Reference: regressor/human_shape/models/backbone/hrnet.py:426-498 (forward), 175-193 (fuse).
#include "conv.cuh"

namespace shapy {

struct SimtConvParams {
  const __half *in_hi, *in_lo;
  int N, H, W, Cin, in_ctot, in_coff;
  const __half *w_hi, *w_lo;
  const float *bias;
  int Cout, ksize, stride, Ho, Wo;
  __half *out_hi, *out_lo;
  int out_ctot, out_coff;
  const __half *res_hi, *res_lo;
  int res_ctot, res_coff;
  int relu;
};

// 64 pixels x 64 output channels per CTA, K chunks of 16 input channels per filter tap.
__global__ void __launch_bounds__(256) conv_simt_kernel(SimtConvParams p) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int m0 = blockIdx.x * 64, n0 = blockIdx.y * 64;
  const int M = p.N * p.Ho * p.Wo;
  const int pad = p.ksize / 2;
  // loader role: pixel lp, 4 channels starting at lc
  const int lp = t >> 2, lc = (t & 3) * 4;
  const int gm = m0 + lp;
  int ln = 0, loh = 0, low = 0;
  const bool mok = gm < M;
  if (mok) { ln = gm / (p.Ho * p.Wo); int r = gm % (p.Ho * p.Wo); loh = r / p.Wo; low = r % p.Wo; }
  const int wco = n0 + lp;  // weight row handled by this loader thread
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int tap = 0; tap < p.ksize * p.ksize; ++tap) {
    const int ky = tap / p.ksize, kx = tap % p.ksize;
    const int ih = loh * p.stride + ky - pad, iw = low * p.stride + kx - pad;
    const bool inb = mok && ih >= 0 && ih < p.H && iw >= 0 && iw < p.W;
    const size_t ioff = (((size_t)ln * p.H + ih) * p.W + iw) * p.in_ctot + p.in_coff;
    const size_t woff = ((size_t)tap * p.Cout + wco) * p.Cin;
    for (int c0 = 0; c0 < p.Cin; c0 += 16) {
      float a[4] = {0.f, 0.f, 0.f, 0.f}, w[4] = {0.f, 0.f, 0.f, 0.f};
      if (inb) {
        const __half2 *h = reinterpret_cast<const __half2 *>(p.in_hi + ioff + c0 + lc);
        float2 x0 = __half22float2(h[0]), x1 = __half22float2(h[1]);
        a[0] = x0.x; a[1] = x0.y; a[2] = x1.x; a[3] = x1.y;
        if (p.in_lo) {
          const __half2 *l = reinterpret_cast<const __half2 *>(p.in_lo + ioff + c0 + lc);
          float2 y0 = __half22float2(l[0]), y1 = __half22float2(l[1]);
          a[0] += y0.x * kLoInv; a[1] += y0.y * kLoInv; a[2] += y1.x * kLoInv; a[3] += y1.y * kLoInv;
        }
      }
      if (wco < p.Cout) {
        const __half2 *h = reinterpret_cast<const __half2 *>(p.w_hi + woff + c0 + lc);
        float2 x0 = __half22float2(h[0]), x1 = __half22float2(h[1]);
        w[0] = x0.x; w[1] = x0.y; w[2] = x1.x; w[3] = x1.y;
        if (p.w_lo) {
          const __half2 *l = reinterpret_cast<const __half2 *>(p.w_lo + woff + c0 + lc);
          float2 y0 = __half22float2(l[0]), y1 = __half22float2(l[1]);
          w[0] += y0.x * kLoInv; w[1] += y0.y * kLoInv; w[2] += y1.x * kLoInv; w[3] += y1.y * kLoInv;
        }
      }
      __syncthreads();
#pragma unroll
      for (int i = 0; i < 4; ++i) { As[lc + i][lp] = a[i]; Bs[lc + i][lp] = w[i]; }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        float4 av = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
        float4 bv = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
        const float aa[4] = {av.x, av.y, av.z, av.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] += aa[i] * bb[j];
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int co = n0 + tx * 4 + j;
      if (co >= p.Cout) continue;
      float v = acc[i][j] + p.bias[co];
      if (p.res_hi) {
        size_t ro = (size_t)m * p.res_ctot + p.res_coff + co;
        v += __half2float(p.res_hi[ro]) + (p.res_lo ? __half2float(p.res_lo[ro]) * kLoInv : 0.f);
      }
      if (p.relu) v = fmaxf(v, 0.f);
      size_t oo = (size_t)m * p.out_ctot + p.out_coff + co;
      __half hi, lo;
      split_store(v, hi, lo);
      p.out_hi[oo] = hi;
      if (p.out_lo) p.out_lo[oo] = lo;
    }
  }
}

int launch_conv_simt(const ConvW &w, const ActView &in, const ActView &out, const ActView *res, bool relu,
                     cudaStream_t st) {
  SHAPY_REQUIRE(w.cin % 16 == 0, "conv_simt: cin %d not a multiple of 16", w.cin);
  SHAPY_REQUIRE(in.C == w.cin && out.C == w.cout, "conv_simt: channel mismatch");
  SimtConvParams p;
  p.in_hi = in.hi; p.in_lo = in.lo; p.N = in.N; p.H = in.H; p.W = in.W; p.Cin = w.cin;
  p.in_ctot = in.Ctot; p.in_coff = in.coff;
  p.w_hi = w.w_hi; p.w_lo = in.lo ? w.w_lo : nullptr; p.bias = w.bias;
  p.Cout = w.cout; p.ksize = w.ksize; p.stride = w.stride; p.Ho = out.H; p.Wo = out.W;
  p.out_hi = out.hi; p.out_lo = out.lo; p.out_ctot = out.Ctot; p.out_coff = out.coff;
  p.res_hi = res ? res->hi : nullptr; p.res_lo = res ? res->lo : nullptr;
  p.res_ctot = res ? res->Ctot : 0; p.res_coff = res ? res->coff : 0;
  p.relu = relu;
  dim3 grid(ceil_div(out.N * out.H * out.W, 64), ceil_div(w.cout, 64));
  conv_simt_kernel<<<grid, 256, 0, st>>>(p);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// ---------------------------------------------------------------------------------------------
// Stem: 3x3 stride-2 conv on the fp32 NCHW network input (hrnet.py:209-211), BN + ReLU folded.
// `cell` (optional): device cell holding the image pointer, read at run time, so that a captured CUDA graph of the
// network can be replayed on any input buffer (hrnet.cu); null = use `img`.
__global__ void __launch_bounds__(256) stem_kernel(const float *__restrict__ img_direct, const float *const *cell, int N, int H, int W,
                                                   const float *__restrict__ wf, const float *__restrict__ bias, int Cout,
                                                   __half *out_hi, __half *out_lo, int ctot, int coff) {
  const float *__restrict__ img = cell ? *cell : img_direct;
  // one thread = one output pixel x 16 output channels; the 4 (Cout = 64) threads of a pixel are adjacent lanes, so a
  // warp writes 8 pixels x 128 contiguous bytes per plane and reads its weights as 4 distinct broadcast LDS.128.
  extern __shared__ __align__(16) float ws[];  // [27][Cout] + bias[Cout]
  for (int i = threadIdx.x; i < 27 * Cout + Cout; i += blockDim.x) ws[i] = i < 27 * Cout ? wf[i] : bias[i - 27 * Cout];
  __syncthreads();
  const int Ho = H / 2, Wo = W / 2;
  const int groups = Cout / 16;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long pix = idx / groups;
  const int g = (int)(idx % groups);
  if (pix >= (long long)N * Ho * Wo) return;
  const int n = (int)(pix / (Ho * Wo)), r = (int)(pix % (Ho * Wo)), oh = r / Wo, ow = r % Wo;
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = ws[27 * Cout + g * 16 + j];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int ih = oh * 2 + ky - 1;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int iw = ow * 2 + kx - 1;
      const bool ok = ih >= 0 && ih < H && iw >= 0 && iw < W;
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float x = ok ? __ldg(img + (((size_t)n * 3 + ci) * H + ih) * W + iw) : 0.f;
        const float4 *wr = reinterpret_cast<const float4 *>(ws + ((ky * 3 + kx) * 3 + ci) * Cout + g * 16);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 w4 = wr[q];
          acc[4 * q] += x * w4.x; acc[4 * q + 1] += x * w4.y; acc[4 * q + 2] += x * w4.z; acc[4 * q + 3] += x * w4.w;
        }
      }
    }
  }
  __align__(16) __half hi[16], lo[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) split_store(fmaxf(acc[j], 0.f), hi[j], lo[j]);
  const size_t o = (size_t)pix * ctot + coff + g * 16;
  reinterpret_cast<uint4 *>(out_hi + o)[0] = reinterpret_cast<const uint4 *>(hi)[0];
  reinterpret_cast<uint4 *>(out_hi + o)[1] = reinterpret_cast<const uint4 *>(hi)[1];
  if (out_lo) {
    reinterpret_cast<uint4 *>(out_lo + o)[0] = reinterpret_cast<const uint4 *>(lo)[0];
    reinterpret_cast<uint4 *>(out_lo + o)[1] = reinterpret_cast<const uint4 *>(lo)[1];
  }
}

// Same convolution, 4 consecutive output pixels x 16 output channels per thread: every weight vector read from shared
// memory feeds 4 pixels (1 LDS.128 per 16 FMAs instead of per 4; the one-pixel variant above is LDS-bound at ~355 us
// for 64 x 224 x 224), and the 9 input columns of a row are two aligned LDG.128 plus one scalar.
__global__ void __launch_bounds__(256, 2) stem4_kernel(const float *__restrict__ img_direct, const float *const *cell, int N, int H, int W,
                                                    const float *__restrict__ wf, const float *__restrict__ bias, int Cout,
                                                    __half *out_hi, __half *out_lo, int ctot, int coff) {
  const float *__restrict__ img = cell ? *cell : img_direct;
  extern __shared__ __align__(16) float ws[];  // [27][Cout] + bias[Cout]
  for (int i = threadIdx.x; i < 27 * Cout + Cout; i += blockDim.x) ws[i] = i < 27 * Cout ? wf[i] : bias[i - 27 * Cout];
  __syncthreads();
  const int Ho = H / 2, Wo = W / 2, Wg = Wo / 4;
  const int groups = Cout / 16;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long pg = idx / groups;
  const int g = (int)(idx % groups);
  if (pg >= (long long)N * Ho * Wg) return;
  const int n = (int)(pg / (Ho * Wg)), r = (int)(pg % (Ho * Wg)), oh = r / Wg, ow0 = (r % Wg) * 4;
  float acc[4][16];
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[p][j] = ws[27 * Cout + g * 16 + j];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int ih = oh * 2 + ky - 1;
    if (ih < 0 || ih >= H) continue;
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
      const float *row = img + (((size_t)n * 3 + ci) * H + ih) * W + 2 * ow0;   // 32-byte aligned: ow0 % 4 == 0, W % 8 == 0
      float x[9];
      x[0] = ow0 > 0 ? __ldg(row - 1) : 0.f;
      const float4 a = __ldg(reinterpret_cast<const float4 *>(row)), b = __ldg(reinterpret_cast<const float4 *>(row) + 1);
      x[1] = a.x; x[2] = a.y; x[3] = a.z; x[4] = a.w; x[5] = b.x; x[6] = b.y; x[7] = b.z; x[8] = b.w;
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) {
        const float4 *wr = reinterpret_cast<const float4 *>(ws + ((ky * 3 + kx) * 3 + ci) * Cout + g * 16);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float4 w4 = wr[q];
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            const float xv = x[2 * p + kx];
            acc[p][4 * q] += xv * w4.x; acc[p][4 * q + 1] += xv * w4.y;
            acc[p][4 * q + 2] += xv * w4.z; acc[p][4 * q + 3] += xv * w4.w;
          }
        }
      }
    }
  }
  const size_t pix0 = ((size_t)n * Ho + oh) * Wo + ow0;
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    __align__(16) __half hi[16], lo[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) split_store(fmaxf(acc[p][j], 0.f), hi[j], lo[j]);
    const size_t o = (pix0 + p) * ctot + coff + g * 16;   // 32-byte aligned (launch_stem checks ctot, coff, base)
    stg32b(out_hi + o, reinterpret_cast<const uint4 *>(hi)[0], reinterpret_cast<const uint4 *>(hi)[1]);
    if (out_lo) stg32b(out_lo + o, reinterpret_cast<const uint4 *>(lo)[0], reinterpret_cast<const uint4 *>(lo)[1]);
  }
}

// images_cell != null: the kernels read the image pointer from that device cell (`images` is then only used for the
// alignment decision and may be any pointer with the alignment the cell's future contents will have)
int launch_stem(const ConvW &w, const float *images, const float *const *images_cell, int N, int H, int W, const ActView &out,
                cudaStream_t st) {
  SHAPY_REQUIRE(w.cin == 3 && w.ksize == 3 && w.stride == 2 && w.cout % 16 == 0 && w.w_f32, "stem: unsupported conv");
  SHAPY_REQUIRE(H % 2 == 0 && W % 2 == 0, "stem: odd input size");
  size_t smem = (size_t)(27 * w.cout + w.cout) * sizeof(float);
  if (W % 8 == 0 && ((uintptr_t)images & 15) == 0 && out.Ctot % 16 == 0 && out.coff % 16 == 0 &&
      ((uintptr_t)out.hi & 31) == 0 && (!out.lo || ((uintptr_t)out.lo & 31) == 0)) {
    long long total4 = (long long)N * (H / 2) * (W / 8) * (w.cout / 16);
    stem4_kernel<<<(unsigned)((total4 + 255) / 256), 256, smem, st>>>(images, images_cell, N, H, W, w.w_f32, w.bias, w.cout,
                                                                      out.hi, out.lo, out.Ctot, out.coff);
    SHAPY_LAUNCH_CHECK();
    return SHAPY_OK;
  }
  long long total = (long long)N * (H / 2) * (W / 2) * (w.cout / 16);
  stem_kernel<<<(unsigned)((total + 255) / 256), 256, smem, st>>>(images, images_cell, N, H, W, w.w_f32, w.bias, w.cout,
                                                                  out.hi, out.lo, out.Ctot, out.coff);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// ---------------------------------------------------------------------------------------------
// Fuse: out = relu(sum_i nearest_up_{2^s_i}(in_i))  (hrnet.py:184-191).  8 channels per thread.
struct FuseParams {
  const __half *hi[4], *lo[4];
  int ctot[4], coff[4], shift[4];
  int n_in, N, H, W, C, relu;
  __half *out_hi, *out_lo;
  int out_ctot, out_coff;
};

// CH = 8: 128-bit accesses; CH = 16: 256-bit accesses (rows 32-byte aligned), half the memory requests.
template <int CH>
__global__ void __launch_bounds__(256) fuse_kernel(FuseParams p) {
  // programmatic dependent launch (see conv_wgmma.cu): this grid may be scheduled while the producer of its inputs is
  // draining, and lets the next launch do the same; the wait returns once every earlier grid has completed
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int cg = p.C / CH;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long pix = idx / cg;
  const int g = (int)(idx % cg);
  if (pix >= (long long)p.N * p.H * p.W) return;
  const int n = (int)(pix / (p.H * p.W)), r = (int)(pix % (p.H * p.W)), h = r / p.W, w = r % p.W;
  float acc[CH];
#pragma unroll
  for (int j = 0; j < CH; ++j) acc[j] = 0.f;
  for (int i = 0; i < p.n_in; ++i) {
    const int s = p.shift[i];
    const int Hi = p.H >> s, Wi = p.W >> s;
    size_t o = (((size_t)n * Hi + (h >> s)) * Wi + (w >> s)) * p.ctot[i] + p.coff[i] + g * CH;
    uint4 hv[CH / 8], lv[CH / 8];
    if (CH == 16) ldg32b(p.hi[i] + o, hv[0], hv[CH / 8 - 1]); else hv[0] = *reinterpret_cast<const uint4 *>(p.hi[i] + o);
    const __half *hh = reinterpret_cast<const __half *>(hv);
    if (p.lo[i]) {
      if (CH == 16) ldg32b(p.lo[i] + o, lv[0], lv[CH / 8 - 1]); else lv[0] = *reinterpret_cast<const uint4 *>(p.lo[i] + o);
      const __half *ll = reinterpret_cast<const __half *>(lv);
#pragma unroll
      for (int j = 0; j < CH; ++j) acc[j] += __half2float(hh[j]) + __half2float(ll[j]) * kLoInv;
    } else {
#pragma unroll
      for (int j = 0; j < CH; ++j) acc[j] += __half2float(hh[j]);
    }
  }
  __align__(16) __half hi[CH], lo[CH];
#pragma unroll
  for (int j = 0; j < CH; ++j) split_store(p.relu ? fmaxf(acc[j], 0.f) : acc[j], hi[j], lo[j]);
  size_t o = (size_t)pix * p.out_ctot + p.out_coff + g * CH;
  const uint4 *h4 = reinterpret_cast<const uint4 *>(hi), *l4 = reinterpret_cast<const uint4 *>(lo);
  if (CH == 16) {
    stg32b(p.out_hi + o, h4[0], h4[CH / 8 - 1]);
    if (p.out_lo) stg32b(p.out_lo + o, l4[0], l4[CH / 8 - 1]);
  } else {
    *reinterpret_cast<uint4 *>(p.out_hi + o) = h4[0];
    if (p.out_lo) *reinterpret_cast<uint4 *>(p.out_lo + o) = l4[0];
  }
}

int launch_fuse(const ActView *ins, const int *shifts, int n_in, const ActView &out, bool relu, cudaStream_t st) {
  SHAPY_REQUIRE(n_in >= 1 && n_in <= 4 && out.C % 8 == 0, "fuse: unsupported arity / channels");
  FuseParams p;
  for (int i = 0; i < 4; ++i) { p.hi[i] = p.lo[i] = nullptr; p.ctot[i] = p.coff[i] = p.shift[i] = 0; }
  for (int i = 0; i < n_in; ++i) {
    SHAPY_REQUIRE(ins[i].C == out.C && (ins[i].H << shifts[i]) == out.H && (ins[i].W << shifts[i]) == out.W,
                  "fuse: input %d shape mismatch", i);
    p.hi[i] = ins[i].hi; p.lo[i] = ins[i].lo; p.ctot[i] = ins[i].Ctot; p.coff[i] = ins[i].coff; p.shift[i] = shifts[i];
  }
  p.n_in = n_in; p.N = out.N; p.H = out.H; p.W = out.W; p.C = out.C; p.relu = relu;
  p.out_hi = out.hi; p.out_lo = out.lo; p.out_ctot = out.Ctot; p.out_coff = out.coff;
  auto al32 = [](const ActView &v) {
    return v.Ctot % 16 == 0 && v.coff % 16 == 0 && ((uintptr_t)v.hi & 31) == 0 && (!v.lo || ((uintptr_t)v.lo & 31) == 0);
  };
  bool wide = out.C % 16 == 0 && al32(out);
  for (int i = 0; i < n_in; ++i) wide = wide && al32(ins[i]);
  static const bool pdl = []() { const char *e = getenv("SHAPY_PDL"); return !(e && e[0] == '0'); }();
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.blockDim = dim3(256);
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  if (wide) {
    long long total = (long long)out.N * out.H * out.W * (out.C / 16);
    cfg.gridDim = dim3((unsigned)((total + 255) / 256));
    SHAPY_CUDA_TRY(cudaLaunchKernelEx(&cfg, fuse_kernel<16>, p));
  } else {
    long long total = (long long)out.N * out.H * out.W * (out.C / 8);
    cfg.gridDim = dim3((unsigned)((total + 255) / 256));
    SHAPY_CUDA_TRY(cudaLaunchKernelEx(&cfg, fuse_kernel<8>, p));
  }
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// ---------------------------------------------------------------------------------------------
// xf.mean(dim=(2,3))  (hrnet.py:484): one thread per (image, channel).
__global__ void pool_kernel(const __half *hi, const __half *lo, int N, int HW, int C, int ctot, int coff, float *feats_direct,
                            float *const *cell) {
  float *feats = cell ? *cell : feats_direct;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  int n = i / C, c = i % C;
  float s = 0.f;
  for (int q = 0; q < HW; ++q) {
    size_t o = ((size_t)n * HW + q) * ctot + coff + c;
    s += __half2float(hi[o]) + (lo ? __half2float(lo[o]) * kLoInv : 0.f);
  }
  feats[i] = s / (float)HW;
}

int launch_pool(const ActView &in, float *feats, float *const *feats_cell, cudaStream_t st) {
  int total = in.N * in.C;
  pool_kernel<<<ceil_div(total, 128), 128, 0, st>>>(in.hi, in.lo, in.N, in.H * in.W, in.C, in.Ctot, in.coff, feats, feats_cell);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// ---------------------------------------------------------------------------------------------
__global__ void set_io_cells_kernel(const void **cells, const void *images, void *feats) {
  cells[0] = images;
  cells[1] = feats;
}

int launch_set_io_cells(void **cells, const float *images, float *feats, cudaStream_t st) {
  set_io_cells_kernel<<<1, 1, 0, st>>>((const void **)cells, images, feats);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

// ---------------------------------------------------------------------------------------------
__global__ void nhwc_split_kernel(const float *x, long long n_pix, int C, __half *hi, __half *lo, int ctot, int coff) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pix * C) return;
  long long pix = i / C;
  int c = (int)(i % C);
  __half h, l;
  split_store(x[i], h, l);
  hi[pix * ctot + coff + c] = h;
  if (lo) lo[pix * ctot + coff + c] = l;
}

int launch_nhwc_split(const float *x, const ActView &out, cudaStream_t st) {
  long long n_pix = (long long)out.N * out.H * out.W;
  nhwc_split_kernel<<<(unsigned)((n_pix * out.C + 255) / 256), 256, 0, st>>>(x, n_pix, out.C, out.hi, out.lo, out.Ctot,
                                                                            out.coff);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

__global__ void nhwc_merge_kernel(const __half *hi, const __half *lo, int N, int H, int W, int C, int ctot, int coff,
                                  float *y, int to_nchw) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)N * H * W * C;
  if (i >= total) return;
  long long pix = i / C;
  int c = (int)(i % C);
  size_t o = (size_t)pix * ctot + coff + c;
  float v = __half2float(hi[o]) + (lo ? __half2float(lo[o]) * kLoInv : 0.f);
  if (to_nchw) {
    int n = (int)(pix / (H * W)), r = (int)(pix % (H * W));
    y[((size_t)n * C + c) * H * W + r] = v;
  } else {
    y[i] = v;
  }
}

int launch_nhwc_merge(const ActView &in, float *y, bool to_nchw, cudaStream_t st) {
  long long total = (long long)in.N * in.H * in.W * in.C;
  nhwc_merge_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in.hi, in.lo, in.N, in.H, in.W, in.C, in.Ctot,
                                                                    in.coff, y, to_nchw ? 1 : 0);
  SHAPY_LAUNCH_CHECK();
  return SHAPY_OK;
}

}  // namespace shapy
