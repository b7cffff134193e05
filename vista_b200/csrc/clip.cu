// The conditioner's CLIP ViT-H/14 image tower (FrozenOpenCLIPImageEmbedder, vwm/modules/encoders/modules.py:251-399):
// the two pieces the tap-GEMM / LayerNorm kernels do not cover.
//   clip_preprocess : kornia resize to 224 x 224 (Gaussian anti-alias blur, then bicubic, align_corners) -> (x + 1) / 2
//                     -> CLIP mean / std -> 14 x 14 patchify into the A operand of the patch-embedding GEMM.
//   attn_d80        : softmax(Q K^T / sqrt(80)) V per (image, head) for head width 80, on mma.sync (fp32 softmax and
//                     accumulation).
#include <math.h>

#include "../../include/vista_b200.h"
#include "host.cuh"
#include "ptx.cuh"

namespace vb {

// ------------------------------------------------------------------------------------------------------------------
// Preprocess.  Blur and bicubic resample are both separable and linear, and their border rules (reflect for the blur,
// clamped indices for the resample) act on one axis at a time, so output row y is a short filter over input rows and
// output column x a short filter over input columns.  Each CTA folds the bicubic weights and the Gaussian taps of its
// 14 output rows and of all 224 output columns into merged weight windows (shared memory), resamples the 14 rows
// vertically into shared memory, then horizontally, normalises and scatters into the patch rows.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kClipImg = 224, kClipPatch = 14, kClipGrid = 16, kClipTokens = 257, kClipK = 3 * 14 * 14;
constexpr int kMaxBlur = 45;                 // Gaussian taps per axis
constexpr int kMaxTaps = kMaxBlur + 3;       // merged window: 4 bicubic taps spread by the blur
constexpr int kPrepThreads = 256;

struct ClipPrepParams {
  const float* x;
  int H, W;
  void* out;
  int ldo, out_f32;
  float gy[kMaxBlur], gx[kMaxBlur];
  int ky, kx;
  float sy, sx;                  // bicubic source scale (in - 1) / (out - 1)
  float mean[3], stdv[3];
};

__device__ __forceinline__ int reflect_idx(int i, int n) {   // F.pad(mode="reflect"): no repeated edge sample
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// torch's upsample_bicubic2d coefficients (A = -0.75) at output coordinate o, merged with the Gaussian taps g[0..kn).
__device__ void merged_taps(int o, float scale, int n, const float* g, int kn, float* w, int* lo_out, int* cnt_out) {
  const float real = scale * (float)o;
  int i0 = (int)floorf(real);
  if (i0 > n - 1) i0 = n - 1;
  float t = real - (float)i0;
  t = fminf(fmaxf(t, 0.f), 1.f);
  const float A = -0.75f;
  float c[4];
  {
    const float x0 = t + 1.f, x1 = t, x2 = 1.f - t, x3 = 2.f - t;
    c[0] = ((A * x0 - 5.f * A) * x0 + 8.f * A) * x0 - 4.f * A;
    c[1] = ((A + 2.f) * x1 - (A + 3.f)) * x1 * x1 + 1.f;
    c[2] = ((A + 2.f) * x2 - (A + 3.f)) * x2 * x2 + 1.f;
    c[3] = ((A * x3 - 5.f * A) * x3 + 8.f * A) * x3 - 4.f * A;
  }
  const int h = kn / 2;
  int lo = n, hi = -1;
  for (int i = 0; i < 4; ++i) {
    const int r = min(max(i0 - 1 + i, 0), n - 1);
    for (int k = 0; k < kn; ++k) {
      const int idx = reflect_idx(r + k - h, n);
      lo = min(lo, idx);
      hi = max(hi, idx);
    }
  }
  for (int j = 0; j < kMaxTaps; ++j) w[j] = 0.f;
  for (int i = 0; i < 4; ++i) {
    const int r = min(max(i0 - 1 + i, 0), n - 1);
    for (int k = 0; k < kn; ++k) w[reflect_idx(r + k - h, n) - lo] += c[i] * g[k];
  }
  *lo_out = lo;
  *cnt_out = hi - lo + 1;
}

__device__ __forceinline__ void store_out(const ClipPrepParams& p, size_t i, float v) {
  if (p.out_f32) reinterpret_cast<float*>(p.out)[i] = v;
  else reinterpret_cast<__half*>(p.out)[i] = __float2half_rn(v);
}

__global__ void __launch_bounds__(kPrepThreads) clip_preprocess_kernel(const ClipPrepParams p) {
  extern __shared__ float smem_f[];
  float* wx = smem_f;                                  // [224][kMaxTaps]
  float* wy = wx + kClipImg * kMaxTaps;                // [14][kMaxTaps]
  int* lox = reinterpret_cast<int*>(wy + kClipPatch * kMaxTaps);   // [224]
  int* cntx = lox + kClipImg;                          // [224]
  int* loy = cntx + kClipImg;                          // [14]
  int* cnty = loy + kClipPatch;                        // [14]
  float* rows = reinterpret_cast<float*>(cnty + kClipPatch);        // [14][W]: vertically resampled rows
  const int pr = blockIdx.x, ch = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x;
  if (tid < kClipImg)
    merged_taps(tid, p.sx, p.W, p.gx, p.kx, wx + tid * kMaxTaps, lox + tid, cntx + tid);
  else if (tid < kClipImg + kClipPatch) {
    const int r = tid - kClipImg;
    merged_taps(pr * kClipPatch + r, p.sy, p.H, p.gy, p.ky, wy + r * kMaxTaps, loy + r, cnty + r);
  }
  __syncthreads();
  const float* img = p.x + ((size_t)b * 3 + ch) * (size_t)p.H * p.W;
  for (int i = tid; i < kClipPatch * p.W; i += kPrepThreads) {
    const int r = i / p.W, x = i - r * p.W;
    const float* src = img + (size_t)loy[r] * p.W + x;
    const float* w = wy + r * kMaxTaps;
    float acc = 0.f;
    for (int j = 0; j < cnty[r]; ++j) acc = fmaf(w[j], __ldg(src + (size_t)j * p.W), acc);
    rows[i] = acc;
  }
  __syncthreads();
  const float mean = p.mean[ch], stdv = p.stdv[ch];
  const size_t row0 = (size_t)b * kClipTokens + 1 + pr * kClipGrid;   // token row of patch (pr, 0)
  for (int i = tid; i < kClipPatch * kClipImg; i += kPrepThreads) {
    const int r = i / kClipImg, xo = i - r * kClipImg;
    const float* src = rows + r * p.W + lox[xo];
    const float* w = wx + xo * kMaxTaps;
    float acc = 0.f;
    for (int j = 0; j < cntx[xo]; ++j) acc = fmaf(w[j], src[j], acc);
    const float v = ((acc + 1.0f) / 2.0f - mean) / stdv;
    const int pc = xo / kClipPatch, px = xo - pc * kClipPatch;
    store_out(p, (row0 + pc) * p.ldo + ch * (kClipPatch * kClipPatch) + r * kClipPatch + px, v);
  }
  if (ch == 0) {                                       // K padding of this CTA's 16 patch rows, and the class-token slot
    const int padw = p.ldo - kClipK;
    for (int i = tid; i < kClipGrid * padw; i += kPrepThreads)
      store_out(p, (row0 + i / padw) * p.ldo + kClipK + i % padw, 0.f);
    if (pr == 0)
      for (int i = tid; i < p.ldo; i += kPrepThreads) store_out(p, (row0 - 1) * p.ldo + i, 0.f);
  }
}

// Gaussian of kornia's anti-aliasing blur for a size factor: sigma = max((factor - 1) / 2, 0.001), kernel size
// int(max(4 sigma, 3)) made odd, taps exp(-x^2 / (2 sigma^2)) normalised to sum 1; factor <= 1 everywhere: no blur.
static int blur_taps(double factor, bool blur, float* g) {
  if (!blur) {
    g[0] = 1.f;
    return 1;
  }
  const double sigma = fmax((factor - 1.0) / 2.0, 0.001);
  int ks = (int)fmax(2.0 * 2.0 * sigma, 3.0);
  if (ks % 2 == 0) ks += 1;
  if (ks > kMaxBlur) return -1;
  const float s2 = (float)(2.0 * sigma * sigma);
  float sum = 0.f;
  for (int i = 0; i < ks; ++i) {
    const float x = (float)(i - ks / 2);
    g[i] = expf(-(x * x) / s2);
    sum += g[i];
  }
  for (int i = 0; i < ks; ++i) g[i] /= sum;
  return ks;
}

// ------------------------------------------------------------------------------------------------------------------
// Attention, head width 80.  4 warps x 16 query rows per CTA; keys in blocks of 64 staged in shared memory (K row-major,
// V transposed so that both B fragments are 32-bit loads); S = Q K^T and O += P V on mma.m16n8k16 with fp32
// accumulators, online softmax in fp32 (exp2, running row maximum), P rounded to fp16 as the A operand of P V.
// ------------------------------------------------------------------------------------------------------------------
constexpr int kD80 = 80, kAQ = 64, kAKB = 64;
constexpr int kKStride = kD80 + 8;     // halfs per K row in shared memory (conflict-free B loads)
constexpr int kVStride = kAKB + 8;     // halfs per row of V^T

__device__ __forceinline__ void mma16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 t = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

__global__ void __launch_bounds__(128) attn_d80_kernel(const __half* __restrict__ q, long long ldq,
                                                       const __half* __restrict__ k, long long ldk,
                                                       const __half* __restrict__ v, long long ldv, __half* __restrict__ out,
                                                       long long ldo, int seq, float scale_log2) {
  __shared__ __align__(16) __half sK[kAKB * kKStride];
  __shared__ __align__(16) __half sVt[kD80 * kVStride];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, c = lane & 3;
  const int head = blockIdx.y, b = blockIdx.z;
  const int r0 = blockIdx.x * kAQ + warp * 16 + g, r1 = r0 + 8;
  const size_t tok0 = (size_t)b * seq;
  const __half* qb = q + head * kD80;
  const __half* kb = k + tok0 * ldk + head * kD80;
  const __half* vb = v + tok0 * ldv + head * kD80;

  uint32_t qa[5][4];
#pragma unroll
  for (int ks = 0; ks < 5; ++ks) {
    const int col = ks * 16 + 2 * c;
    const __half* p0 = qb + (tok0 + r0) * ldq + col;
    const __half* p1 = qb + (tok0 + r1) * ldq + col;
    qa[ks][0] = r0 < seq ? *reinterpret_cast<const uint32_t*>(p0) : 0u;
    qa[ks][1] = r1 < seq ? *reinterpret_cast<const uint32_t*>(p1) : 0u;
    qa[ks][2] = r0 < seq ? *reinterpret_cast<const uint32_t*>(p0 + 8) : 0u;
    qa[ks][3] = r1 < seq ? *reinterpret_cast<const uint32_t*>(p1 + 8) : 0u;
  }
  float o[10][4];
#pragma unroll
  for (int i = 0; i < 10; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

  for (int k0 = 0; k0 < seq; k0 += kAKB) {
    __syncthreads();                                   // the previous block has been consumed
    for (int i = tid; i < kAKB * (kD80 / 8); i += 128) {
      const int key = i / (kD80 / 8), chunk = i - key * (kD80 / 8);
      uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
      if (k0 + key < seq) {
        kv = __ldg(reinterpret_cast<const uint4*>(kb + (size_t)(k0 + key) * ldk + chunk * 8));
        vv = __ldg(reinterpret_cast<const uint4*>(vb + (size_t)(k0 + key) * ldv + chunk * 8));
      }
      *reinterpret_cast<uint4*>(sK + key * kKStride + chunk * 8) = kv;
      const __half* vh = reinterpret_cast<const __half*>(&vv);
#pragma unroll
      for (int e = 0; e < 8; ++e) sVt[(chunk * 8 + e) * kVStride + key] = vh[e];
    }
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      const __half* krow = sK + (nt * 8 + g) * kKStride + 2 * c;
#pragma unroll
      for (int ks = 0; ks < 5; ++ks)
        mma16816(s[nt], qa[ks], *reinterpret_cast<const uint32_t*>(krow + ks * 16),
                 *reinterpret_cast<const uint32_t*>(krow + ks * 16 + 8));
    }
    const int kv_left = seq - k0;
    if (kv_left < kAKB) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (nt * 8 + 2 * c + e >= kv_left) s[nt][e] = s[nt][2 + e] = -INFINITY;
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
    float mneg[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      const float m_new = fmaxf(m_run[hh], mx[hh] * scale_log2);   // finite: key k0 is always in range
      const float alpha = ex2_f(m_run[hh] - m_new);
      m_run[hh] = m_new;
      mneg[hh] = -m_new;
      l_run[hh] *= alpha;
#pragma unroll
      for (int dt = 0; dt < 10; ++dt) {
        o[dt][2 * hh] *= alpha;
        o[dt][2 * hh + 1] *= alpha;
      }
    }
    uint32_t pa[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = ex2_f(fmaf(s[nt][0], scale_log2, mneg[0]));
      const float p1 = ex2_f(fmaf(s[nt][1], scale_log2, mneg[0]));
      const float p2 = ex2_f(fmaf(s[nt][2], scale_log2, mneg[1]));
      const float p3 = ex2_f(fmaf(s[nt][3], scale_log2, mneg[1]));
      l_run[0] += p0 + p1;
      l_run[1] += p2 + p3;
      pa[nt >> 1][(nt & 1) * 2 + 0] = pack_half2(p0, p1);
      pa[nt >> 1][(nt & 1) * 2 + 1] = pack_half2(p2, p3);
    }
#pragma unroll
    for (int dt = 0; dt < 10; ++dt) {
      const __half* vrow = sVt + (dt * 8 + g) * kVStride + 2 * c;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        mma16816(o[dt], pa[j], *reinterpret_cast<const uint32_t*>(vrow + j * 16),
                 *reinterpret_cast<const uint32_t*>(vrow + j * 16 + 8));
    }
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 1);
    l_run[hh] += __shfl_xor_sync(0xffffffffu, l_run[hh], 2);
    l_run[hh] = 1.0f / l_run[hh];
  }
  __half* ob = out + head * kD80 + 2 * c;
#pragma unroll
  for (int dt = 0; dt < 10; ++dt) {
    if (r0 < seq)
      *reinterpret_cast<uint32_t*>(ob + (tok0 + r0) * ldo + dt * 8) = pack_half2(o[dt][0] * l_run[0], o[dt][1] * l_run[0]);
    if (r1 < seq)
      *reinterpret_cast<uint32_t*>(ob + (tok0 + r1) * ldo + dt * 8) = pack_half2(o[dt][2] * l_run[1], o[dt][3] * l_run[1]);
  }
}

}  // namespace vb

extern "C" int b200v_clip_preprocess(const float* x, int32_t n, int32_t H, int32_t W, int32_t antialias, void* out,
                                     int64_t ldo, int32_t out_f32, void* stream) {
  using namespace vb;
  VB_REQUIRE(x && out, "clip_preprocess: null pointer");
  VB_REQUIRE(n > 0 && H > 1 && W > 1, "clip_preprocess: bad sizes n=%d H=%d W=%d", n, H, W);
  VB_REQUIRE(ldo >= kClipK && ldo % 8 == 0, "clip_preprocess: ldo=%lld must be >= 588 and a multiple of 8", (long long)ldo);
  ClipPrepParams p;
  memset(&p, 0, sizeof(p));
  p.x = x;
  p.H = H;
  p.W = W;
  p.out = out;
  p.ldo = (int)ldo;
  p.out_f32 = out_f32 != 0;
  // kornia.geometry.resize: blur only when some axis shrinks (antialias and max(factors) > 1); an input already 224 x 224
  // is returned unchanged, which the identity weights below reproduce
  const double fy = (double)H / kClipImg, fx = (double)W / kClipImg;
  const bool blur = antialias && fmax(fy, fx) > 1.0;
  p.ky = blur_taps(fy, blur, p.gy);
  p.kx = blur_taps(fx, blur, p.gx);
  VB_REQUIRE(p.ky > 0 && p.kx > 0, "clip_preprocess: %d x %d is too large for the anti-alias blur (kernel > %d taps)", H, W,
             kMaxBlur);
  VB_REQUIRE(H > p.ky / 2 && W > p.kx / 2, "clip_preprocess: input smaller than the blur's reflect padding");
  p.sy = (float)(H - 1) / (float)(kClipImg - 1);
  p.sx = (float)(W - 1) / (float)(kClipImg - 1);
  const float mean[3] = {0.48145466f, 0.4578275f, 0.40821073f}, stdv[3] = {0.26862954f, 0.26130258f, 0.27577711f};
  for (int i = 0; i < 3; ++i) {
    p.mean[i] = mean[i];
    p.stdv[i] = stdv[i];
  }
  const size_t smem = (size_t)(kClipImg + kClipPatch) * kMaxTaps * 4 + (2 * kClipImg + 2 * kClipPatch) * 4 +
                      (size_t)kClipPatch * W * 4;
  constexpr size_t kMaxSmem = 227 * 1024;
  VB_REQUIRE(smem <= kMaxSmem, "clip_preprocess: W=%d too wide", W);
  static bool attr_set[64] = {false};
  if (first_use_on_device(attr_set))
    VB_CHECK_CUDA(cudaFuncSetAttribute(clip_preprocess_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem));
  clip_preprocess_kernel<<<dim3(kClipGrid, 3, n), kPrepThreads, smem, (cudaStream_t)stream>>>(p);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_attention_d80(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v, int64_t ld_v,
                                   void* out, int64_t ld_o, int32_t batch, int32_t seq, int32_t heads, void* stream) {
  using namespace vb;
  VB_REQUIRE(q && k && v && out, "attention_d80: null pointer");
  VB_REQUIRE(batch > 0 && batch <= 65535 && seq > 0 && heads > 0 && heads <= 65535, "attention_d80: bad sizes");
  VB_REQUIRE(ld_q % 8 == 0 && ld_k % 8 == 0 && ld_v % 8 == 0 && ld_o % 8 == 0,
             "attention_d80: row strides must be multiples of 8 elements");
  VB_REQUIRE(((reinterpret_cast<uintptr_t>(q) | reinterpret_cast<uintptr_t>(k) | reinterpret_cast<uintptr_t>(v) |
               reinterpret_cast<uintptr_t>(out)) & 15) == 0,
             "attention_d80: pointers must be 16-byte aligned");
  dim3 grid((seq + kAQ - 1) / kAQ, heads, batch);
  const float scale_log2 = (float)(1.4426950408889634 / sqrt(80.0));
  attn_d80_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __half*>(q), ld_q, reinterpret_cast<const __half*>(k), ld_k,
      reinterpret_cast<const __half*>(v), ld_v, reinterpret_cast<__half*>(out), ld_o, seq, scale_log2);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
