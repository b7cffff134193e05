// HBM-bound kernels of the path: GroupNorm (stats / apply+SiLU), LayerNorm, temporal attention
// (sequence = frames of one pixel), thin direct convolutions, data movement, embedding helpers,
// the fused EDM/Euler sampler step and the layout converters.  All activations are token-major
// fp16 with explicit row strides; every kernel uses 16-byte vector accesses along channels.
#include "../../include/vista_b200.h"
#include "host.cuh"
#include "ptx.cuh"

namespace vb {

__device__ __forceinline__ void h8_to_f(const uint4& u, float (&f)[8]) {
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 f_to_h8(const float (&f)[8]) {
  uint4 u;
  __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return u;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------
// GroupNorm statistics, deterministic.  grid = (chunks, frames); a block walks `chunk` tokens of one
// frame; thread (row, lane) owns the 8-channel vectors lane, lane+L, ... and keeps per-channel fp32
// sums of d = x - K and d^2 around a pivot K, its first value of the channel: a group whose mean is
// large next to its spread would lose its variance in fp32 sums of x^2 (E x^2 - mean^2 cancels).  The
// thread turns them into fp64 raw sums (c K + sum d, c K^2 + 2 K sum d + sum d^2) in shared memory;
// rows are combined in a fixed order there, groups are summed in fp64 and written as one partial per
// (frame, chunk, group).  The last block to finish a statistic (ticket counter)
// adds the partials in a fixed order and writes (mean, rstd): bit-identical from run to run, no
// floating-point atomics, no memset (the counter resets itself).
// ------------------------------------------------------------------------------------------
constexpr int kGnThreads = 256;
constexpr int kGnMaxJ = 4;  // max vectors per thread (C <= 8 * 256 * kGnMaxJ); kernels are templated on 1 / 2 / 4
constexpr int kGnMinChunk = 16;   // b200v_groupnorm_chunk(): lower bound of the tokens one block walks
// Tokens per block: about 16 blocks per SM over the whole launch (small feature maps would otherwise leave most
// SMs idle; huge ones would leave the last block of a statistic tens of thousands of partial sums to add), a
// multiple of 8, at least kGnMinChunk.  A pure function of the shape: results stay bit-reproducible.
static inline int gn_pick_chunk(int frames, int tokens_per_frame) {
  long long c = ((long long)frames * tokens_per_frame + 2367) / 2368;
  c = (c + 7) / 8 * 8;
  if (c < kGnMinChunk) c = kGnMinChunk;
  if (c > tokens_per_frame) c = (tokens_per_frame + 7) / 8 * 8;
  return (int)c;
}

template <int JT>
__global__ void __launch_bounds__(kGnThreads)
gn_stats_kernel(const __half* __restrict__ x, long long ldx, int tokens_per_frame, int C, int groups,
                int frames_per_stat, int chunk, int L, int J, float eps, double* __restrict__ partials,
                int* __restrict__ counters, float* __restrict__ mean_rstd, double* __restrict__ raw_out) {
  extern __shared__ double sh[];  // [rows][2*C]
  __shared__ int s_last;
  const int frame = blockIdx.y;
  const int t0 = blockIdx.x * chunk;
  const int t1 = min(t0 + chunk, tokens_per_frame);
  const int nvec = C >> 3;
  const int rows = kGnThreads / L;
  const int lane = threadIdx.x % L, row = threadIdx.x / L;
  if (row < rows) {
    const __half* base = x + ((long long)frame * tokens_per_frame) * ldx;
    const int n_tok = t0 + row < t1 ? (t1 - t0 - row + rows - 1) / rows : 0;   // tokens t0 + row, + rows, ... < t1
    float s[JT][8], q[JT][8], piv[JT][8];
    uint4 u0[JT];
#pragma unroll
    for (int j = 0; j < JT; ++j) {
      const int v = lane + j * L;
      u0[j] = make_uint4(0, 0, 0, 0);
      if (n_tok > 0 && j < J && v < nvec)
        u0[j] = __ldg(reinterpret_cast<const uint4*>(base + (long long)(t0 + row) * ldx + v * 8));
      h8_to_f(u0[j], piv[j]);
#pragma unroll
      for (int i = 0; i < 8; ++i) s[j][i] = q[j][i] = 0.f;
    }
    // 4 tokens per iteration: 4 independent 16-byte loads in flight per thread and vector
    for (int t = t0 + row; t < t1; t += 4 * rows) {
#pragma unroll
      for (int j = 0; j < JT; ++j) {
        const int v = lane + j * L;
        if (j < J && v < nvec) {
          uint4 u[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int tt = t + k * rows;
            u[k] = tt < t1 ? __ldg(reinterpret_cast<const uint4*>(base + (long long)tt * ldx + v * 8)) : u0[j];
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            float f[8];
            h8_to_f(u[k], f);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float d = f[i] - piv[j][i];   // a token past t1 reads the pivot: d = 0
              s[j][i] += d;
              q[j][i] = fmaf(d, d, q[j][i]);
            }
          }
        }
      }
    }
    double* mine = sh + (size_t)row * 2 * C;
    const double cnt = (double)n_tok;
#pragma unroll
    for (int j = 0; j < JT; ++j) {
      const int v = lane + j * L;
      if (j < J && v < nvec) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const double K = (double)piv[j][i], sd = (double)s[j][i];
          mine[v * 8 + i] = fma(cnt, K, sd);
          mine[C + v * 8 + i] = fma(cnt * K, K, fma(2.0 * K, sd, (double)q[j][i]));
        }
      }
    }
  }
  __syncthreads();
  const int cpg = C / groups;
  const int chunks = gridDim.x;
  for (int g = threadIdx.x; g < groups; g += kGnThreads) {
    double a = 0.0, b = 0.0;
    for (int r = 0; r < rows; ++r) {
      const double* p = sh + (size_t)r * 2 * C;
      for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
        a += p[c];
        b += p[C + c];
      }
    }
    double* dst = partials + (((long long)frame * chunks + blockIdx.x) * groups + g) * 2;
    dst[0] = a;
    dst[1] = b;
  }
  __threadfence();
  __syncthreads();
  const int stat = frame / frames_per_stat;
  if (threadIdx.x == 0) {
    const int ticket = atomicAdd(&counters[stat], 1);
    s_last = (ticket == frames_per_stat * chunks - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // Final reduction, fixed order: 8 threads per group each add every 8th partial in index order, thread 0 of the
  // group adds the 8 sub-sums in order (the partial count reaches frames_per_stat * chunks ~ 10^3).
  const double cnt = (double)cpg * tokens_per_frame * frames_per_stat;
  double* red = sh;   // [groups][8][2]; the row partials in sh are dead by now
  const int n_part = frames_per_stat * chunks;
  for (int idx = threadIdx.x; idx < groups * 8; idx += kGnThreads) {
    const int g = idx >> 3, sub = idx & 7;
    double a = 0.0, b = 0.0;
    const double* src = partials + ((long long)stat * n_part * groups + g) * 2;
    for (int i = sub; i < n_part; i += 8) {
      a += __ldcg(src + (long long)i * groups * 2);
      b += __ldcg(src + (long long)i * groups * 2 + 1);
    }
    red[idx * 2] = a;
    red[idx * 2 + 1] = b;
  }
  __syncthreads();
  for (int g = threadIdx.x; g < groups; g += kGnThreads) {
    double a = 0.0, b = 0.0;
    for (int sub = 0; sub < 8; ++sub) {
      a += red[(g * 8 + sub) * 2];
      b += red[(g * 8 + sub) * 2 + 1];
    }
    if (raw_out) {   // frame-sharded mode: the caller reduces the sums across ranks and finalises
      raw_out[((long long)stat * groups + g) * 2] = a;
      raw_out[((long long)stat * groups + g) * 2 + 1] = b;
    } else {
      const double mean = a / cnt;
      double var = b / cnt - mean * mean;
      if (var < 0.0) var = 0.0;
      mean_rstd[((long long)stat * groups + g) * 2] = (float)mean;
      mean_rstd[((long long)stat * groups + g) * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
    }
  }
  if (threadIdx.x == 0) counters[stat] = 0;  // ready for the next launch
}

// apply: grid = (chunks, frames); y = (x-mean)*rstd*gamma + beta, optional SiLU.  Same thread layout as the
// statistics kernel: thread (row, lane) owns channel vectors lane, lane+L, ... so the per-channel scale / shift
// live in registers; 4 tokens per iteration keep 4 loads in flight per vector.
template <int JT>
__global__ void __launch_bounds__(kGnThreads)
gn_apply_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ y, long long ldy,
                int tokens_per_frame, int C, int groups, int frames_per_stat, int chunk, int L, int J,
                const float* __restrict__ mean_rstd, const float* __restrict__ gamma, const float* __restrict__ beta,
                int silu) {
  const int frame = blockIdx.y;
  const int cpg = C / groups;
  const int nvec = C >> 3;
  const int rows = kGnThreads / L;
  const int lane = threadIdx.x % L, row = threadIdx.x / L;
  if (row >= rows) return;
  const float* st = mean_rstd + (long long)(frame / frames_per_stat) * groups * 2;
  float sc[JT][8], sf[JT][8];
#pragma unroll
  for (int j = 0; j < JT; ++j) {
    const int v = lane + j * L;
    if (j < J && v < nvec) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = v * 8 + i;
        const int g = c / cpg;
        const float s_ = __ldg(st + 2 * g + 1) * __ldg(gamma + c);
        sc[j][i] = s_;
        sf[j][i] = __ldg(beta + c) - __ldg(st + 2 * g) * s_;
      }
    }
  }
  const int t0 = blockIdx.x * chunk;
  const int t1 = min(t0 + chunk, tokens_per_frame);
  const __half* xb = x + ((long long)frame * tokens_per_frame) * ldx;
  __half* yb = y + ((long long)frame * tokens_per_frame) * ldy;
  for (int t = t0 + row; t < t1; t += 4 * rows) {
#pragma unroll
    for (int j = 0; j < JT; ++j) {
      const int v = lane + j * L;
      if (j < J && v < nvec) {
        uint4 u[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int tt = t + k * rows;
          if (tt < t1) u[k] = __ldg(reinterpret_cast<const uint4*>(xb + (long long)tt * ldx + v * 8));
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int tt = t + k * rows;
          if (tt < t1) {
            float f[8];
            h8_to_f(u[k], f);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float r = fmaf(f[i], sc[j][i], sf[j][i]);
              f[i] = silu ? silu_f(r) : r;
            }
            *reinterpret_cast<uint4*>(yb + (long long)tt * ldy + v * 8) = f_to_h8(f);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// LayerNorm: one warp per token, the row lives in registers (NV 16-byte vectors per lane), two-pass
// statistics.  Templated on NV so that the common widths (C = 320: NV 2, 640: 3, 1280: 5) keep the
// register count low and the SM full of warps (the kernel is a pure HBM stream).
// ------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ y, long long ldy, long long tokens,
                 int C, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                 const float* __restrict__ addvec, long long ld_addvec, int av_div, int av_mod) {
  // Grid-stride over tokens, one warp per token, the NEXT token's row is already in flight while the current one is
  // reduced and written (a warp that handled one token per launch left the memory system idle between its load, its two
  // reductions and its store: 2.3 TB/s; kept busy it is an HBM stream).
  const int lane = threadIdx.x & 31;
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  long long token = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (token >= tokens) return;
  const int nvec = C >> 3;
  uint4 raw[NV];
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    const int vi = lane + j * 32;
    if (vi < nvec) raw[j] = __ldg(reinterpret_cast<const uint4*>(x + token * ldx + vi * 8));
  }
  while (true) {
    const long long next = token + n_warps;
    uint4 nxt[NV];
    if (next < tokens) {
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        const int vi = lane + j * 32;
        if (vi < nvec) nxt[j] = __ldg(reinterpret_cast<const uint4*>(x + next * ldx + vi * 8));
      }
    }
    float v[NV][8];
    const float* av = addvec ? addvec + ((token / av_div) % av_mod) * ld_addvec : nullptr;
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int vi = lane + j * 32;
      if (vi < nvec) {
        h8_to_f(raw[j], v[j]);
        if (av) {
          const float4 a0 = __ldg(reinterpret_cast<const float4*>(av + vi * 8));
          const float4 a1 = __ldg(reinterpret_cast<const float4*>(av + vi * 8 + 4));
          v[j][0] += a0.x; v[j][1] += a0.y; v[j][2] += a0.z; v[j][3] += a0.w;
          v[j][4] += a1.x; v[j][5] += a1.y; v[j][6] += a1.z; v[j][7] += a1.w;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) sum += v[j][i];
      }
    }
    const float mean = warp_sum(sum) / (float)C;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int vi = lane + j * 32;
      if (vi < nvec) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float d = v[j][i] - mean;
          sq += d * d;
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      const int vi = lane + j * 32;
      if (vi < nvec) {
        const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8));
        const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + vi * 8 + 4));
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(beta + vi * 8 + 4));
        const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
        const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        float o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = (v[j][i] - mean) * rstd * gg[i] + bb[i];
        *reinterpret_cast<uint4*>(y + token * ldy + vi * 8) = f_to_h8(o);
      }
    }
    if (next >= tokens) break;
    token = next;
#pragma unroll
    for (int j = 0; j < NV; ++j) raw[j] = nxt[j];
  }
}

// LayerNorm for C = 40 * LPR (320 / 640 / 1280: LPR = 8 / 16 / 32 lanes per row, every lane 5 16-byte vectors, no idle
// lanes; a warp normalises 32 / LPR rows per iteration).  gamma / beta live in registers for the whole grid-stride loop
// (the one-warp-per-token kernel re-read them from L1 for every token: 128 of its 160 load sectors per token and a third
// of its instructions), the next rows are prefetched while the current ones are reduced: an HBM stream.
template <int LPR>
__global__ void __launch_bounds__(128, 3)
layernorm40_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ y, long long ldy, long long tokens,
                   const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                   const float* __restrict__ addvec, long long ld_addvec, int av_div, int av_mod) {
  constexpr int RPW = 32 / LPR;
  constexpr int C = LPR * 40;
  const int lane = threadIdx.x & 31;
  const int sub = lane % LPR, rowi = lane / LPR;
  float g[5][8], b[5][8];
#pragma unroll
  for (int j = 0; j < 5; ++j) {
    const int c0 = (sub + j * LPR) * 8;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c0)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c0 + 4));
    g[j][0] = g0.x; g[j][1] = g0.y; g[j][2] = g0.z; g[j][3] = g0.w; g[j][4] = g1.x; g[j][5] = g1.y; g[j][6] = g1.z; g[j][7] = g1.w;
    b[j][0] = b0.x; b[j][1] = b0.y; b[j][2] = b0.z; b[j][3] = b0.w; b[j][4] = b1.x; b[j][5] = b1.y; b[j][6] = b1.z; b[j][7] = b1.w;
  }
  const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
  long long token = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + rowi;
  const long long stride = n_warps * RPW;
  uint4 raw[5];
  if (token < tokens) {
#pragma unroll
    for (int j = 0; j < 5; ++j) raw[j] = __ldg(reinterpret_cast<const uint4*>(x + token * ldx + (sub + j * LPR) * 8));
  }
  // every lane of a warp runs the same number of iterations (the shuffles need the whole warp): loop on the warp's first row
  for (long long base = token - rowi; base < tokens; base += stride, token += stride) {
    const long long next = token + stride;
    uint4 nxt[5];
    if (next < tokens) {
#pragma unroll
      for (int j = 0; j < 5; ++j) nxt[j] = __ldg(reinterpret_cast<const uint4*>(x + next * ldx + (sub + j * LPR) * 8));
    }
    const bool live = token < tokens;
    float v[5][8];
    float sum = 0.f;
    if (live) {
      const float* av = addvec ? addvec + ((token / av_div) % av_mod) * ld_addvec : nullptr;
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        h8_to_f(raw[j], v[j]);
        if (av) {
          const int c0 = (sub + j * LPR) * 8;
          const float4 a0 = __ldg(reinterpret_cast<const float4*>(av + c0)), a1 = __ldg(reinterpret_cast<const float4*>(av + c0 + 4));
          v[j][0] += a0.x; v[j][1] += a0.y; v[j][2] += a0.z; v[j][3] += a0.w;
          v[j][4] += a1.x; v[j][5] += a1.y; v[j][6] += a1.z; v[j][7] += a1.w;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) sum += v[j][i];
      }
    } else {
#pragma unroll
      for (int j = 0; j < 5; ++j)
#pragma unroll
        for (int i = 0; i < 8; ++i) v[j][i] = 0.f;
    }
#pragma unroll
    for (int off = LPR / 2; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    const float mean = sum / (float)C;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < 5; ++j)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        v[j][i] -= mean;
        sq = fmaf(v[j][i], v[j][i], sq);
      }
#pragma unroll
    for (int off = LPR / 2; off > 0; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
    const float rstd = rsqrtf(sq / (float)C + eps);
    if (live) {
#pragma unroll
      for (int j = 0; j < 5; ++j) {
        float o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = fmaf(v[j][i] * rstd, g[j][i], b[j][i]);
        *reinterpret_cast<uint4*>(y + token * ldy + (sub + j * LPR) * 8) = f_to_h8(o);
      }
    }
#pragma unroll
    for (int j = 0; j < 5; ++j) raw[j] = nxt[j];
  }
}

// ------------------------------------------------------------------------------------------
// Temporal attention: sequence = the T <= 32 frames of one pixel, head dim 64.  One warp per
// (clip, pixel, head): q/k/v rows (128 B each, strided over frames) are brought to shared memory with
// cp.async (all ~20 loads of a lane in flight), S = Q K^T and O = P V run on mma.sync m16n8k16
// (32 x 32 x 64 and 32 x 64 x 32 with zero padding), softmax in the accumulator fragments.  The kernel is
// a pure HBM stream: it reads q, k, v and writes o exactly once.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t h2_bits(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

constexpr int kTaWarps = 4;

__global__ void __launch_bounds__(kTaWarps * 32)
attn_temporal_kernel(const __half* __restrict__ q, long long ld_q, const __half* __restrict__ k, long long ld_k,
                     const __half* __restrict__ v, long long ld_v, __half* __restrict__ out, long long ld_o, int nb,
                     int Tq, int T, int S, int heads, const long long* __restrict__ kv_frame_tok) {
  __shared__ __align__(128) uint8_t tiles[kTaWarps][3][32 * 128];   // per warp: Q, K, V tiles of 32 rows x 128 B
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t sQ = smem_u32(tiles[warp][0]), sK = smem_u32(tiles[warp][1]), sV = smem_u32(tiles[warp][2]);
  // zero the tiles once: rows >= T of K and V are never written afterwards, so padded keys score against zeros (and
  // are masked) and padded V rows add nothing.  The Q tile's rows >= Tq are not reloaded and hold the previous item's
  // O staging; they only feed S / O rows >= Tq, which are never stored.
  for (int i = lane; i < 3 * 32 * 8; i += 32) reinterpret_cast<uint4*>(tiles[warp][0])[i] = make_uint4(0, 0, 0, 0);
  __syncwarp();
  const long long items = (long long)nb * S * heads;
  const int quad = lane >> 2, tq = lane & 3;
  for (long long item = (long long)blockIdx.x * kTaWarps + warp; item < items; item += (long long)gridDim.x * kTaWarps) {
    const int head = (int)(item % heads);
    const long long ps = item / heads;
    const int s = (int)(ps % S);
    const int b = (int)(ps / S);
    const long long tok0 = (long long)b * Tq * S + s;   // query / output rows: local frames, clip-major
    // ---- stage q, k, v rows: chunk c (16 B) of row t goes to slot c ^ (t & 7).  K/V frame t of clip b starts at
    //      token kv_frame_tok[b*T + t] (frame-sharded mode: gathered from all ranks) or b*T*S + t*S (local).
    for (int i = lane; i < T * 8; i += 32) {
      const int t = i >> 3, c = i & 7;
      const long long ktok = (kv_frame_tok ? kv_frame_tok[b * T + t] : ((long long)b * T + t) * S) + s;
      const uint32_t off = t * 128 + ((c ^ (t & 7)) << 4);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sK + off), "l"(k + ktok * ld_k + head * 64 + c * 8) : "memory");
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sV + off), "l"(v + ktok * ld_v + head * 64 + c * 8) : "memory");
      if (t < Tq) {
        const long long tok = tok0 + (long long)t * S;
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sQ + off), "l"(q + tok * ld_q + head * 64 + c * 8) : "memory");
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncwarp();
    // ---- S = Q K^T  (rows: 2 m16 tiles, keys: 4 n8 tiles, dims: 4 k16 steps)
    float sc[2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) sc[mt][nt][i] = 0.f;
    {
      const int mrow = (lane & 7) + ((lane >> 3) & 1) * 8;   // ldmatrix row supplied by this lane (A operand)
      const int mchk = lane >> 4;                            // 0: k-chunk 2kk, 1: k-chunk 2kk+1
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        uint32_t a[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const int row = mt * 16 + mrow, chk = 2 * kk + mchk;
          ldsm_x4(sQ + row * 128 + ((chk ^ (row & 7)) << 4), a[mt]);
        }
#pragma unroll
        for (int nt = 0; nt < 4; nt += 2) {
          // B fragments of two key tiles: matrices (keys 8nt.., chunk 2kk), (8nt.., 2kk+1), (8(nt+1).., 2kk), (.., 2kk+1)
          uint32_t bfr[4];
          const int row = nt * 8 + (lane & 7) + (lane >> 4) * 8, chk = 2 * kk + ((lane >> 3) & 1);
          ldsm_x4(sK + row * 128 + ((chk ^ (row & 7)) << 4), bfr);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            mma_16816(sc[mt][nt], a[mt], bfr[0], bfr[1]);
            mma_16816(sc[mt][nt + 1], a[mt], bfr[2], bfr[3]);
          }
        }
      }
    }
    // ---- softmax over keys (< T), rows live in quads: cols 8nt + 2tq + {0,1}; regs {0,1}: row quad, {2,3}: row quad+8
    uint32_t pa[2][2][4];   // P as A fragments: [mt][k16 step][4]
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int key = nt * 8 + 2 * tq + (i & 1);
          float x = key < T ? sc[mt][nt][i] * 0.125f : -INFINITY;
          sc[mt][nt][i] = x;
          if (i < 2) mx0 = fmaxf(mx0, x); else mx1 = fmaxf(mx1, x);
        }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      float l0 = 0.f, l1 = 0.f;
#pragma unroll
      for (int nt = 0; nt < 4; ++nt)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float e = __expf(sc[mt][nt][i] - (i < 2 ? mx0 : mx1));
          sc[mt][nt][i] = e;
          if (i < 2) l0 += e; else l1 += e;
        }
      l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
      l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
      l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
      const float i0 = 1.0f / l0, i1 = 1.0f / l1;
#pragma unroll
      for (int k2 = 0; k2 < 2; ++k2) {
        pa[mt][k2][0] = h2_bits(sc[mt][2 * k2][0] * i0, sc[mt][2 * k2][1] * i0);
        pa[mt][k2][1] = h2_bits(sc[mt][2 * k2][2] * i1, sc[mt][2 * k2][3] * i1);
        pa[mt][k2][2] = h2_bits(sc[mt][2 * k2 + 1][0] * i0, sc[mt][2 * k2 + 1][1] * i0);
        pa[mt][k2][3] = h2_bits(sc[mt][2 * k2 + 1][2] * i1, sc[mt][2 * k2 + 1][3] * i1);
      }
    }
    // ---- O = P V  (dims: 8 n8 tiles, keys: 2 k16 steps); V^T fragments via ldmatrix.trans
    __syncwarp();   // every lane is done reading Q: its tile is reused to stage O
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      uint32_t bfr[4];
      const int row = lane;   // matrices 0..3 = keys 0-7, 8-15, 16-23, 24-31; all take 16-byte chunk dt
      ldsm_x4_trans(sV + row * 128 + ((dt ^ (row & 7)) << 4), bfr);
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        float o[4] = {0.f, 0.f, 0.f, 0.f};
        mma_16816(o, pa[mt][0], bfr[0], bfr[1]);
        mma_16816(o, pa[mt][1], bfr[2], bfr[3]);
        // stage: rows mt*16 + quad (+8), dims 8dt + 2tq + {0,1}  -> 4-byte pieces of chunk dt
        const int r0 = mt * 16 + quad, r1 = r0 + 8;
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sQ + r0 * 128 + ((dt ^ (r0 & 7)) << 4) + tq * 4), "r"(h2_bits(o[0], o[1])) : "memory");
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sQ + r1 * 128 + ((dt ^ (r1 & 7)) << 4) + tq * 4), "r"(h2_bits(o[2], o[3])) : "memory");
      }
    }
    __syncwarp();
    for (int i = lane; i < Tq * 8; i += 32) {
      const int t = i >> 3, c = i & 7;
      const long long tok = tok0 + (long long)t * S;
      uint4 val;
      asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(val.x), "=r"(val.y), "=r"(val.z), "=r"(val.w)
                   : "r"(sQ + t * 128 + ((c ^ (t & 7)) << 4)));
      *reinterpret_cast<uint4*>(out + tok * ld_o + head * 64 + c * 8) = val;
    }
    __syncwarp();   // O staging fully read before the next item's cp.async overwrite the Q tile
  }
}

// ------------------------------------------------------------------------------------------
// Thin direct convolutions
// ------------------------------------------------------------------------------------------
// Cin <= 8 : x is token-major fp16 [tokens, 8] (channels >= cin are ignored), out [tokens, ldo] fp16.
// block = 256 threads handles 32 tokens; thread n loops over output channels.
__global__ void __launch_bounds__(256)
conv3x3_small_cin_kernel(const __half* __restrict__ x, int cin, const float* __restrict__ w,
                         const float* __restrict__ bias, __half* __restrict__ out, long long ldo, int NB, int H, int W,
                         int cout) {
  __shared__ float patch[32][72];
  const long long tok0 = (long long)blockIdx.x * 32;
  const long long tokens = (long long)NB * H * W;
  for (int i = threadIdx.x; i < 32 * 9; i += blockDim.x) {
    const int t = i / 9, tap = i - t * 9;
    const long long tok = tok0 + t;
    float f[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (tok < tokens) {
      const int wq = (int)(tok % W), hq = (int)((tok / W) % H);
      const long long b = tok / ((long long)W * H);
      const int hh = hq + tap / 3 - 1, ww = wq + tap % 3 - 1;
      if (hh >= 0 && hh < H && ww >= 0 && ww < W)
        h8_to_f(__ldg(reinterpret_cast<const uint4*>(x + ((b * H + hh) * W + ww) * 8)), f);
    }
    // channels >= cin are not staged: a NaN / Inf there must not reach the sum through a zero weight (NaN * 0 = NaN)
#pragma unroll
    for (int c = 0; c < 8; ++c) patch[t][tap * 8 + c] = c < cin ? f[c] : 0.f;
  }
  __syncthreads();
  for (int n = threadIdx.x; n < cout; n += blockDim.x) {
    float wr[72];
#pragma unroll
    for (int i = 0; i < 72; ++i) wr[i] = 0.f;
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
      for (int tap = 0; tap < 9; ++tap)
        if (c < cin) wr[tap * 8 + c] = __ldg(w + ((long long)n * cin + c) * 9 + tap);
    const float bv = bias ? __ldg(bias + n) : 0.f;
    for (int t = 0; t < 32; ++t) {
      const long long tok = tok0 + t;
      if (tok >= tokens) break;
      float a = bv;
#pragma unroll
      for (int i = 0; i < 72; ++i) a = fmaf(patch[t][i], wr[i], a);
      out[tok * ldo + n] = __float2half_rn(a);
    }
  }
}

// Cout <= 4: one warp per token; weights [cout][9][cin] fp32 staged in shared memory as fp16.
__global__ void __launch_bounds__(256)
conv3x3_small_cout_kernel(const __half* __restrict__ x, long long ldx, int cin, const float* __restrict__ w,
                          const float* __restrict__ bias, float* __restrict__ out, int NB, int H, int W, int cout) {
  extern __shared__ __half shw[];  // [cout][9][cin]
  for (int i = threadIdx.x; i < cout * 9 * cin; i += blockDim.x) {
    const int o = i / (9 * cin), r = i - o * 9 * cin;
    const int tap = r / cin, c = r - tap * cin;
    shw[i] = __float2half_rn(__ldg(w + ((long long)o * cin + c) * 9 + tap));
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long tokens = (long long)NB * H * W;
  const long long tok = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (tok >= tokens) return;
  const int wq = (int)(tok % W), hq = (int)((tok / W) % H);
  const long long b = tok / ((long long)W * H);
  const int nvec = cin >> 3;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int tap = 0; tap < 9; ++tap) {
    const int hh = hq + tap / 3 - 1, ww = wq + tap % 3 - 1;
    if (hh < 0 || hh >= H || ww < 0 || ww >= W) continue;
    const __half* xp = x + ((b * H + hh) * W + ww) * ldx;
    for (int v = lane; v < nvec; v += 32) {
      float f[8];
      h8_to_f(__ldg(reinterpret_cast<const uint4*>(xp + v * 8)), f);
#pragma unroll
      for (int o = 0; o < 4; ++o) {
        if (o < cout) {
          float g[8];
          h8_to_f(*reinterpret_cast<const uint4*>(shw + ((long long)o * 9 + tap) * cin + v * 8), g);
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[o] = fmaf(f[i], g[i], acc[o]);
        }
      }
    }
  }
#pragma unroll
  for (int o = 0; o < 4; ++o) acc[o] = warp_sum(acc[o]);
  if (lane == 0) {
    for (int o = 0; o < cout; ++o) out[tok * cout + o] = acc[o] + (bias ? __ldg(bias + o) : 0.f);
  }
}

// ------------------------------------------------------------------------------------------
// Data movement
// ------------------------------------------------------------------------------------------
// out[(b, ho, wo), tap*C + c] = x[b, 2ho + kh - 1, 2wo + kw - 1, c] (zero padded), Ho = (H+1)/2
__global__ void im2col_s2_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ out, int NB, int H,
                                 int W, int C) {
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const int nvec = C >> 3;
  const long long total = (long long)NB * Ho * Wo * 9 * nvec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    long long r = i / nvec;
    const int tap = (int)(r % 9);
    r /= 9;
    const int wo = (int)(r % Wo), ho = (int)((r / Wo) % Ho);
    const long long b = r / ((long long)Wo * Ho);
    const int hh = 2 * ho + tap / 3 - 1, ww = 2 * wo + tap % 3 - 1;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (hh >= 0 && hh < H && ww >= 0 && ww < W)
      val = __ldg(reinterpret_cast<const uint4*>(x + ((b * H + hh) * W + ww) * ldx + v * 8));
    *reinterpret_cast<uint4*>(out + r * (9LL * C) + (long long)tap * C + v * 8) = val;
  }
}

// VAE-encoder Downsample (model.py:69-83): zero pad by one on the right / bottom only, conv3x3 stride 2 without
// padding: out[(b, ho, wo), tap*C + c] = x[b, 2ho + kh, 2wo + kw, c] (zero beyond H, W), Ho = (H - 2) / 2 + 1.
__global__ void im2col_s2_asym_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ out, int NB,
                                      int H, int W, int C) {
  const int Ho = (H - 2) / 2 + 1, Wo = (W - 2) / 2 + 1;
  const int nvec = C >> 3;
  const long long total = (long long)NB * Ho * Wo * 9 * nvec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    long long r = i / nvec;
    const int tap = (int)(r % 9);
    r /= 9;
    const int wo = (int)(r % Wo), ho = (int)((r / Wo) % Ho);
    const long long b = r / ((long long)Wo * Ho);
    const int hh = 2 * ho + tap / 3, ww = 2 * wo + tap % 3;
    uint4 val = make_uint4(0, 0, 0, 0);
    if (hh < H && ww < W)
      val = __ldg(reinterpret_cast<const uint4*>(x + ((b * H + hh) * W + ww) * ldx + v * 8));
    *reinterpret_cast<uint4*>(out + r * (9LL * C) + (long long)tap * C + v * 8) = val;
  }
}

__global__ void upsample2x_kernel(const __half* __restrict__ x, long long ldx, __half* __restrict__ out, long long ldo,
                                  int NB, int H, int W, int C) {
  const int nvec = C >> 3;
  const int Ho = 2 * H, Wo = 2 * W;
  const long long total = (long long)NB * Ho * Wo * nvec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    const long long r = i / nvec;
    const int wo = (int)(r % Wo), ho = (int)((r / Wo) % Ho);
    const long long b = r / ((long long)Wo * Ho);
    *reinterpret_cast<uint4*>(out + r * ldo + v * 8) =
        __ldg(reinterpret_cast<const uint4*>(x + ((b * H + (ho >> 1)) * W + (wo >> 1)) * ldx + v * 8));
  }
}

// ------------------------------------------------------------------------------------------
// Embedding helpers
// ------------------------------------------------------------------------------------------
__global__ void timestep_embedding_kernel(const float* __restrict__ t, int n, int dim, float max_period,
                                          __half* __restrict__ out, long long ldo) {
  const int half_dim = dim >> 1;
  const int i = blockIdx.x;
  for (int k = threadIdx.x; k < half_dim; k += blockDim.x) {
    const float freq = expf(-logf(max_period) * (float)k / (float)half_dim);
    const float a = t[i] * freq;
    out[i * ldo + k] = __float2half_rn(cosf(a));
    out[i * ldo + half_dim + k] = __float2half_rn(sinf(a));
  }
}

__global__ void blend_emb_kernel(const float* __restrict__ e_plain, const float* __restrict__ e_cond,
                                 const float* __restrict__ label, const float* __restrict__ mask,
                                 float* __restrict__ emb, __half* __restrict__ silu_emb, int rows, int dim) {
  const long long total = (long long)rows * dim;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / dim);
    const float m = mask ? mask[r] : 0.f;
    float e = e_plain[i] * (1.f - m);
    if (e_cond) e += e_cond[i] * m;
    if (label) e += label[i];
    if (emb) emb[i] = e;
    if (silu_emb) silu_emb[i] = __float2half_rn(silu_f(e));
  }
}

// ------------------------------------------------------------------------------------------
// Sampler step (fp32 state)
// ------------------------------------------------------------------------------------------
// one thread per latent pixel (t, y, x); handles the 4 channels
__global__ void sampler_prepare_kernel(float* __restrict__ x, const float* __restrict__ cond_frame,
                                       const float* __restrict__ mask, const float* __restrict__ concat_u,
                                       const float* __restrict__ concat_c, const float* __restrict__ sigmas, const int* __restrict__ step_idx,
                                       __half* __restrict__ unet_in, long long ld_in, float* __restrict__ c_noise, int T,
                                       int h, int w) {
  const float sigma = sigmas[*step_idx];
  const float c_in = rsqrtf(sigma * sigma + 1.0f);
  const int hw = h * w;
  const long long total = (long long)T * hw;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 2 * T && c_noise) c_noise[i] = 0.25f * logf(sigma);
  if (i >= total) return;
  const int t = (int)(i / hw), pix = (int)(i % hw);
  const float m = mask ? mask[t] : 0.f;
  float xv[8], cu[8];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const long long idx = ((long long)t * 4 + c) * hw + pix;
    float v = x[idx];
    if (mask && cond_frame) {
      v = v * (1.f - m) + cond_frame[idx] * m;
      x[idx] = v;
    }
    xv[c] = v * c_in;
    cu[c] = xv[c];
    xv[4 + c] = concat_u ? concat_u[idx] : 0.f;        // uncond rows (zeros in sample.py:243)
    cu[4 + c] = concat_c ? concat_c[idx] : 0.f;        // cond rows
  }
  *reinterpret_cast<uint4*>(unet_in + ((long long)t * hw + pix) * ld_in) = f_to_h8(xv);
  *reinterpret_cast<uint4*>(unet_in + (((long long)T + t) * hw + pix) * ld_in) = f_to_h8(cu);
}

// kMultistep <false>: the Euler step.  <true>: the DPM-Solver++(2M) step x = a x - b (c D - e D_prev), D_prev = D, with
// {a, b, c, e} = coefs[step] from the host (vista_b200.diffusion.dpmpp2m_coefficients); e == 0 marks a first-order
// row, on which D_prev is not read (it is uninitialised at a sample's first step).
// kActionCfg <true>: action guidance (vista_b200.diffusion.ActionCFG).  D_img, the denoised value of the conditional rows
// with the action slots zeroed, is row t of net_img; D = D_u + s_img (D_img - D_u) + s_act (D_c - D_img), in the torch
// guider's order, with s_img = scales[t] and s_act = action_scales[t] read on the device (a captured graph replays them).
template <bool kMultistep, bool kActionCfg>
__global__ void sampler_update_kernel(float* __restrict__ x, const float* __restrict__ net,
                                      const float* __restrict__ cond_frame, const float* __restrict__ mask,
                                      const float* __restrict__ scales, const float* __restrict__ sigmas,
                                      const int* __restrict__ step_idx, int num_steps, int T, int h, int w,
                                      long long ld_net, const float4* __restrict__ coefs, float* __restrict__ d_prev,
                                      const float* __restrict__ net_img, long long ld_img,
                                      const float* __restrict__ action_scales) {
  const int step = *step_idx;
  const float sigma = sigmas[step], sigma_next = sigmas[step + 1];
  const float c_skip = 1.0f / (sigma * sigma + 1.0f);
  const float c_out = -sigma * rsqrtf(sigma * sigma + 1.0f);
  const int hw = h * w;
  const long long total = (long long)T * hw;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int t = (int)(i / hw), pix = (int)(i % hw);
  const float4 nu = *reinterpret_cast<const float4*>(net + ((long long)t * hw + pix) * ld_net);
  const float4 nc = *reinterpret_cast<const float4*>(net + (((long long)T + t) * hw + pix) * ld_net);
  const float un[4] = {nu.x, nu.y, nu.z, nu.w}, cn[4] = {nc.x, nc.y, nc.z, nc.w};
  const float sc = scales[t];
  float in[4] = {0.f, 0.f, 0.f, 0.f}, sa = 0.f;
  if constexpr (kActionCfg) {
    const float4 ni = *reinterpret_cast<const float4*>(net_img + ((long long)t * hw + pix) * ld_img);
    in[0] = ni.x; in[1] = ni.y; in[2] = ni.z; in[3] = ni.w;
    sa = action_scales[t];
  }
  const bool final_step = (step + 1 == num_steps);
  const float m = mask ? mask[t] : 0.f;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const long long idx = ((long long)t * 4 + c) * hw + pix;
    const float xv = x[idx];
    const float du = un[c] * c_out + xv * c_skip;
    const float dc = cn[c] * c_out + xv * c_skip;
    float den;
    if constexpr (kActionCfg) {
      const float di = in[c] * c_out + xv * c_skip;
      den = du + sc * (di - du);
      den = den + sa * (dc - di);
    } else {
      den = du + sc * (dc - du);
    }
    float xn;
    if constexpr (kMultistep) {
      const float4 k = coefs[step];
      float dd = k.z * den;
      if (k.w != 0.f) dd -= k.w * d_prev[idx];
      xn = k.x * xv - k.y * dd;
      d_prev[idx] = den;
    } else {
      const float d = (xv - den) / sigma;
      xn = xv + d * (sigma_next - sigma);
    }
    if (final_step && mask && cond_frame) xn = xn * (1.f - m) + cond_frame[idx] * m;
    x[idx] = xn;
  }
}
__global__ void step_inc_kernel(int* step_idx) { *step_idx += 1; }

// ------------------------------------------------------------------------------------------
// Layout converters
// ------------------------------------------------------------------------------------------
__global__ void nchw_to_tokens_kernel(const float* __restrict__ x, __half* __restrict__ out, long long ldo, int NB,
                                      int C, int H, int W) {
  const long long total = (long long)NB * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long tok = i / C;
    const int pix = (int)(tok % ((long long)H * W));
    const long long b = tok / ((long long)H * W);
    out[tok * ldo + c] = __float2half_rn(x[(b * C + c) * (long long)H * W + pix]);
  }
}
__global__ void tokens_to_nchw_kernel(const void* __restrict__ x, int is_f32, long long ldx, float* __restrict__ out,
                                      int NB, int C, int H, int W) {
  const long long total = (long long)NB * H * W * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pix = (int)(i % ((long long)H * W));
    const long long bc = i / ((long long)H * W);
    const int c = (int)(bc % C);
    const long long b = bc / C;
    const long long tok = b * H * W + pix;
    out[i] = is_f32 ? reinterpret_cast<const float*>(x)[tok * ldx + c]
                    : __half2float(reinterpret_cast<const __half*>(x)[tok * ldx + c]);
  }
}

static inline int grid_for(long long total, int block, int cap = 132 * 16) {
  long long g = (total + block - 1) / block;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace vb

using namespace vb;

static int gn_stats_impl(const void* x, int64_t ldx, int32_t frames, int32_t tokens_per_frame, int32_t C, int32_t groups,
                         int32_t frames_per_stat, float eps, double* partials, int32_t* counters, float* mean_rstd,
                         double* raw_sums, void* stream) {
  VB_REQUIRE(x && partials && counters && (mean_rstd || raw_sums), "groupnorm_stats: null pointer");
  VB_REQUIRE(C % 8 == 0 && C % groups == 0 && ldx % 8 == 0, "groupnorm_stats: C=%d groups=%d ldx=%lld invalid", C, groups,
             (long long)ldx);
  VB_REQUIRE(frames_per_stat > 0 && frames % frames_per_stat == 0, "groupnorm_stats: frames %% frames_per_stat != 0");
  const int nvec = C / 8;
  int L = nvec, J = 1;
  while (L > kGnThreads) {  // split vectors over J passes
    ++J;
    L = (nvec + J - 1) / J;
  }
  VB_REQUIRE(J <= kGnMaxJ, "groupnorm_stats: C=%d too large", C);
  const int rows = kGnThreads / L;
  const int chunk = gn_pick_chunk(frames, tokens_per_frame);
  dim3 grid((tokens_per_frame + chunk - 1) / chunk, frames);
  size_t smem = (size_t)rows * 2 * C * sizeof(double);
  if (smem < (size_t)groups * 8 * 2 * sizeof(double)) smem = (size_t)groups * 8 * 2 * sizeof(double);
  static bool attr_set[64] = {false};
  if (vb::first_use_on_device(attr_set)) {
    VB_CHECK_CUDA(cudaFuncSetAttribute(gn_stats_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    VB_CHECK_CUDA(cudaFuncSetAttribute(gn_stats_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    VB_CHECK_CUDA(cudaFuncSetAttribute(gn_stats_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
  }
  VB_REQUIRE(smem <= 160 * 1024, "groupnorm_stats: shared memory %zu too large", smem);
#define VB_GN_STATS(JT)                                                                                              \
  gn_stats_kernel<JT><<<grid, kGnThreads, smem, (cudaStream_t)stream>>>(                                             \
      (const __half*)x, ldx, tokens_per_frame, C, groups, frames_per_stat, chunk, L, J, eps, partials, counters,     \
      mean_rstd, raw_sums)
  if (J == 1) VB_GN_STATS(1);
  else if (J == 2) VB_GN_STATS(2);
  else VB_GN_STATS(4);
#undef VB_GN_STATS
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_groupnorm_stats(const void* x, int64_t ldx, int32_t frames, int32_t tokens_per_frame, int32_t C,
                                     int32_t groups, int32_t frames_per_stat, float eps, double* partials,
                                     int32_t* counters, float* mean_rstd, void* stream) {
  return gn_stats_impl(x, ldx, frames, tokens_per_frame, C, groups, frames_per_stat, eps, partials, counters, mean_rstd,
                       nullptr, stream);
}

extern "C" int b200v_groupnorm_sums(const void* x, int64_t ldx, int32_t frames, int32_t tokens_per_frame, int32_t C,
                                    int32_t groups, int32_t frames_per_stat, double* partials, int32_t* counters,
                                    double* sums, void* stream) {
  return gn_stats_impl(x, ldx, frames, tokens_per_frame, C, groups, frames_per_stat, 0.f, partials, counters, nullptr,
                       sums, stream);
}

namespace vb {
__global__ void gn_finalize_kernel(const double* __restrict__ sums, int n, double count, float eps,
                                   float* __restrict__ mean_rstd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double mean = sums[2 * i] / count;
  double var = sums[2 * i + 1] / count - mean * mean;
  if (var < 0.0) var = 0.0;
  mean_rstd[2 * i] = (float)mean;
  mean_rstd[2 * i + 1] = (float)(1.0 / sqrt(var + (double)eps));
}
}  // namespace vb

extern "C" int b200v_groupnorm_finalize(const double* sums, int32_t n_stat_groups, double count, float eps,
                                        float* mean_rstd, void* stream) {
  VB_REQUIRE(sums && mean_rstd && n_stat_groups > 0 && count > 0, "groupnorm_finalize: bad args");
  vb::gn_finalize_kernel<<<(n_stat_groups + 127) / 128, 128, 0, (cudaStream_t)stream>>>(sums, n_stat_groups, count, eps,
                                                                                         mean_rstd);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// (mean, rstd) from the column partials of the producing tap-GEMM (gemm_tc.cu, STATS variants).  grid = (groups, stats);
// a partial is (s, m2) of 32 rows (sum, squared deviations from s / 32: every quarter of a frame's tiles is full, as
// tokens_per_frame % 128 == 0 and the tiles of a STATS GEMM are whole); thread t adds the raw sums s and m2 + s^2 / 32 of
// partial rows t, t + 256, ... of its group's columns in fp64, the 256 sub-sums are combined by a fixed tree:
// bit-identical from run to run.  fp64 sums of x^2 cancel only at ~2^-53 (mean / std)^2 in the finalisation.
namespace vb {
__global__ void __launch_bounds__(256)
gn_from_partials_kernel(const float* __restrict__ partials, long long ld, int rows_per_stat, int cpg, int groups, float eps,
                        double count, float* __restrict__ mean_rstd, double* __restrict__ raw) {
  __shared__ double red[2][256];
  const int g = blockIdx.x, st = blockIdx.y;
  const float* base = partials + ((long long)st * rows_per_stat * ld + (long long)g * cpg) * 2;
  double a = 0.0, b = 0.0;
  for (int r = threadIdx.x; r < rows_per_stat; r += 256) {
    const float2* row = reinterpret_cast<const float2*>(base + (long long)r * ld * 2);
    for (int c = 0; c < cpg; ++c) {
      const float2 v = __ldg(row + c);
      a += (double)v.x;
      b += fma((double)v.x * (1.0 / 32.0), (double)v.x, (double)v.y);
    }
  }
  red[0][threadIdx.x] = a;
  red[1][threadIdx.x] = b;
  __syncthreads();
  for (int off = 128; off > 0; off >>= 1) {
    if (threadIdx.x < off) {
      red[0][threadIdx.x] += red[0][threadIdx.x + off];
      red[1][threadIdx.x] += red[1][threadIdx.x + off];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const long long o = ((long long)st * groups + g) * 2;
    if (raw) {
      raw[o] = red[0][0];
      raw[o + 1] = red[1][0];
    } else {
      const double mean = red[0][0] / count;
      double var = red[1][0] / count - mean * mean;
      if (var < 0.0) var = 0.0;
      mean_rstd[o] = (float)mean;
      mean_rstd[o + 1] = (float)(1.0 / sqrt(var + (double)eps));
    }
  }
}
}  // namespace vb

extern "C" int b200v_groupnorm_from_partials(const float* partials, int64_t stats_ld, int32_t n_stats, int32_t frames_per_stat,
                                             int32_t tokens_per_frame, int32_t C, int32_t groups, float eps,
                                             float* mean_rstd, double* raw_sums, void* stream) {
  VB_REQUIRE(partials && (mean_rstd || raw_sums), "b200v_groupnorm_from_partials: null pointer");
  VB_REQUIRE(n_stats > 0 && frames_per_stat > 0 && groups > 0 && C % groups == 0 && stats_ld >= C,
             "b200v_groupnorm_from_partials: bad sizes");
  VB_REQUIRE(tokens_per_frame % 128 == 0, "b200v_groupnorm_from_partials: tokens_per_frame=%d must be a multiple of 128",
             tokens_per_frame);
  const int rows_per_stat = frames_per_stat * (tokens_per_frame / 128) * 4;
  const int cpg = C / groups;
  dim3 grid(groups, n_stats);
  vb::gn_from_partials_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(partials, stats_ld, rows_per_stat, cpg, groups, eps,
                                                                        (double)cpg * tokens_per_frame * frames_per_stat,
                                                                        mean_rstd, raw_sums);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_groupnorm_chunk(void) { return vb::kGnMinChunk; }
extern "C" int b200v_groupnorm_chunk_for(int32_t frames, int32_t tokens_per_frame) {
  return vb::gn_pick_chunk(frames, tokens_per_frame);
}

extern "C" int b200v_groupnorm_apply(const void* x, int64_t ldx, void* y, int64_t ldy, int32_t frames,
                                     int32_t tokens_per_frame, int32_t C, int32_t groups, int32_t frames_per_stat,
                                     const float* mean_rstd, const float* gamma, const float* beta, int32_t silu,
                                     void* stream) {
  VB_REQUIRE(x && y && mean_rstd && gamma && beta, "groupnorm_apply: null pointer");
  VB_REQUIRE(C % 8 == 0 && C % groups == 0 && ldx % 8 == 0 && ldy % 8 == 0, "groupnorm_apply: bad C/ld");
  VB_REQUIRE(frames_per_stat > 0 && frames % frames_per_stat == 0, "groupnorm_apply: frames %% frames_per_stat != 0");
  const int nvec = C / 8;
  int L = nvec, J = 1;
  while (L > kGnThreads) {
    ++J;
    L = (nvec + J - 1) / J;
  }
  VB_REQUIRE(J <= kGnMaxJ, "groupnorm_apply: C=%d too large", C);
  int chunk = gn_pick_chunk(frames, tokens_per_frame);
  if (chunk > 128) chunk = 128;
  dim3 grid((tokens_per_frame + chunk - 1) / chunk, frames);
#define VB_GN_APPLY(JT)                                                                                              \
  gn_apply_kernel<JT><<<grid, kGnThreads, 0, (cudaStream_t)stream>>>(                                                \
      (const __half*)x, ldx, (__half*)y, ldy, tokens_per_frame, C, groups, frames_per_stat, chunk, L, J, mean_rstd,  \
      gamma, beta, silu)
  if (J == 1) VB_GN_APPLY(1);
  else if (J == 2) VB_GN_APPLY(2);
  else VB_GN_APPLY(4);
#undef VB_GN_APPLY
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_layernorm(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t tokens, int32_t C,
                               const float* gamma, const float* beta, float eps, const float* addvec,
                               int64_t ld_addvec, int32_t av_div, int32_t av_mod, void* stream) {
  VB_REQUIRE(x && y && gamma && beta, "layernorm: null pointer");
  VB_REQUIRE(C % 8 == 0 && C <= 2560 && ldx % 8 == 0 && ldy % 8 == 0, "layernorm: C=%d unsupported", C);
  VB_REQUIRE(!addvec || (av_div > 0 && av_mod > 0 && ld_addvec % 4 == 0), "layernorm: bad addvec args");
  const int wpb = 8;
  const long long blocks_needed = (tokens + wpb - 1) / wpb;
  const int nv = (C / 8 + 31) / 32;
  const int ad = av_div > 0 ? av_div : 1, am = av_mod > 0 ? av_mod : 1;
  if (C == 320 || C == 640 || C == 1280) {
    // the UNet's three widths: lanes-per-row kernel (gamma / beta in registers, no idle lanes)
    using namespace vb;
#define VB_LAYERNORM40_LAUNCH(LPR)                                                                                   \
  {                                                                                                                  \
    static int per_sm = 0;                                                                                           \
    if (per_sm == 0 && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, layernorm40_kernel<LPR>, 128, 0) !=   \
                            cudaSuccess || per_sm <= 0))                                                            \
      per_sm = 3;                                                                                                    \
    const long long need = (tokens + 4 * (32 / LPR) - 1) / (4 * (32 / LPR));                                         \
    long long blocks = (long long)device_sm_count() * per_sm;                                                        \
    if (blocks > need) blocks = need;                                                                                \
    layernorm40_kernel<LPR><<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>(                                     \
        (const __half*)x, ldx, (__half*)y, ldy, tokens, gamma, beta, eps, addvec, ld_addvec, ad, am);                \
  }
    if (C == 320) VB_LAYERNORM40_LAUNCH(8)
    else if (C == 640) VB_LAYERNORM40_LAUNCH(16)
    else VB_LAYERNORM40_LAUNCH(32)
#undef VB_LAYERNORM40_LAUNCH
    VB_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  // one resident wave of blocks (occupancy by register count), the warps stride over the tokens
#define VB_LN_LAUNCH(NV)                                                                                             \
  {                                                                                                                  \
    static int per_sm = 0;                                                                                           \
    if (per_sm == 0 && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, layernorm_kernel<NV>, wpb * 32, 0) != \
                            cudaSuccess || per_sm <= 0))                                                            \
      per_sm = 2;                                                                                                    \
    long long blocks = (long long)vb::device_sm_count() * per_sm;                                                    \
    if (blocks > blocks_needed) blocks = blocks_needed;                                                              \
    layernorm_kernel<NV><<<(unsigned)blocks, wpb * 32, 0, (cudaStream_t)stream>>>(                                   \
        (const __half*)x, ldx, (__half*)y, ldy, tokens, C, gamma, beta, eps, addvec, ld_addvec, ad, am);             \
  }
  if (nv <= 1) VB_LN_LAUNCH(1)
  else if (nv <= 2) VB_LN_LAUNCH(2)
  else if (nv <= 3) VB_LN_LAUNCH(3)
  else if (nv <= 5) VB_LN_LAUNCH(5)
  else VB_LN_LAUNCH(10)
#undef VB_LN_LAUNCH
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int attn_temporal_impl(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v, int64_t ld_v,
                              void* out, int64_t ld_o, int32_t nb, int32_t Tq, int32_t T, int32_t S, int32_t heads,
                              const int64_t* kv_frame_tok, void* stream) {
  VB_REQUIRE(q && k && v && out, "attention_temporal: null pointer");
  VB_REQUIRE(T >= 1 && T <= 32 && Tq >= 1 && Tq <= T && heads >= 1, "attention_temporal: T=%d Tq=%d heads=%d unsupported", T,
             Tq, heads);
  VB_REQUIRE(ld_q % 8 == 0 && ld_k % 8 == 0 && ld_v % 8 == 0 && ld_o % 8 == 0, "attention_temporal: bad ld");
  const long long items = (long long)nb * S * heads;
  long long blocks = (items + kTaWarps - 1) / kTaWarps;
  const long long cap = (long long)device_sm_count() * 16;
  if (blocks > cap) blocks = cap;
  attn_temporal_kernel<<<(unsigned)blocks, kTaWarps * 32, 0, (cudaStream_t)stream>>>(
      (const __half*)q, ld_q, (const __half*)k, ld_k, (const __half*)v, ld_v, (__half*)out, ld_o, nb, Tq, T, S, heads,
      reinterpret_cast<const long long*>(kv_frame_tok));
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_attention_temporal(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v,
                                        int64_t ld_v, void* out, int64_t ld_o, int32_t nb, int32_t T, int32_t S,
                                        int32_t heads, void* stream) {
  return attn_temporal_impl(q, ld_q, k, ld_k, v, ld_v, out, ld_o, nb, T, T, S, heads, nullptr, stream);
}

extern "C" int b200v_attention_temporal_sharded(const void* q, int64_t ld_q, const void* k, int64_t ld_k, const void* v,
                                                int64_t ld_v, void* out, int64_t ld_o, int32_t nb, int32_t Tq, int32_t T,
                                                int32_t S, int32_t heads, const int64_t* kv_frame_tok, void* stream) {
  VB_REQUIRE(kv_frame_tok, "attention_temporal_sharded: null frame table");
  return attn_temporal_impl(q, ld_q, k, ld_k, v, ld_v, out, ld_o, nb, Tq, T, S, heads, kv_frame_tok, stream);
}

extern "C" int b200v_conv3x3_small_cin(const void* x, int32_t cin, const float* w, const float* bias, void* out,
                                       int64_t ldo, int32_t NB, int32_t H, int32_t W, int32_t cout, void* stream) {
  VB_REQUIRE(x && w && out, "conv3x3_small_cin: null pointer");
  VB_REQUIRE(cin >= 1 && cin <= 8, "conv3x3_small_cin: cin=%d > 8", cin);
  const long long tokens = (long long)NB * H * W;
  conv3x3_small_cin_kernel<<<(unsigned)((tokens + 31) / 32), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)x, cin, w, bias, (__half*)out, ldo, NB, H, W, cout);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_conv3x3_small_cout(const void* x, int64_t ldx, int32_t cin, const float* w, const float* bias,
                                        float* out, int32_t NB, int32_t H, int32_t W, int32_t cout, void* stream) {
  VB_REQUIRE(x && w && out, "conv3x3_small_cout: null pointer");
  VB_REQUIRE(cout >= 1 && cout <= 4 && cin % 8 == 0 && ldx % 8 == 0, "conv3x3_small_cout: cout=%d cin=%d unsupported",
             cout, cin);
  const long long tokens = (long long)NB * H * W;
  const size_t smem = (size_t)cout * 9 * cin * sizeof(__half);
  conv3x3_small_cout_kernel<<<(unsigned)((tokens + 7) / 8), 256, smem, (cudaStream_t)stream>>>(
      (const __half*)x, ldx, cin, w, bias, out, NB, H, W, cout);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_im2col_s2(const void* x, int64_t ldx, void* out, int32_t NB, int32_t H, int32_t W, int32_t C,
                               void* stream) {
  VB_REQUIRE(x && out && C % 8 == 0 && ldx % 8 == 0, "im2col_s2: bad args");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  const long long total = (long long)NB * Ho * Wo * 9 * (C / 8);
  im2col_s2_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x, ldx, (__half*)out, NB, H,
                                                                           W, C);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_im2col_s2_asym(const void* x, int64_t ldx, void* out, int32_t NB, int32_t H, int32_t W, int32_t C,
                                    void* stream) {
  VB_REQUIRE(x && out && C % 8 == 0 && ldx % 8 == 0 && H >= 2 && W >= 2, "im2col_s2_asym: bad args");
  const int Ho = (H - 2) / 2 + 1, Wo = (W - 2) / 2 + 1;
  const long long total = (long long)NB * Ho * Wo * 9 * (C / 8);
  im2col_s2_asym_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x, ldx, (__half*)out, NB,
                                                                                H, W, C);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_upsample2x(const void* x, int64_t ldx, void* out, int64_t ldo, int32_t NB, int32_t H, int32_t W,
                                int32_t C, void* stream) {
  VB_REQUIRE(x && out && C % 8 == 0 && ldx % 8 == 0 && ldo % 8 == 0, "upsample2x: bad args");
  const long long total = (long long)NB * 4 * H * W * (C / 8);
  upsample2x_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const __half*)x, ldx, (__half*)out, ldo,
                                                                            NB, H, W, C);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_timestep_embedding(const float* t, int32_t n, int32_t dim, float max_period, void* out_f16,
                                        int64_t ldo, void* stream) {
  VB_REQUIRE(t && out_f16 && dim % 2 == 0, "timestep_embedding: bad args");
  timestep_embedding_kernel<<<n, 128, 0, (cudaStream_t)stream>>>(t, n, dim, max_period, (__half*)out_f16, ldo);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_blend_emb(const float* e_plain, const float* e_cond, const float* label, const float* mask,
                               float* emb_f32, void* silu_emb_f16, int32_t rows, int32_t dim, void* stream) {
  VB_REQUIRE(e_plain, "blend_emb: null pointer");
  blend_emb_kernel<<<grid_for((long long)rows * dim, 256), 256, 0, (cudaStream_t)stream>>>(
      e_plain, e_cond, label, mask, emb_f32, (__half*)silu_emb_f16, rows, dim);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_sampler_prepare(float* x, const float* cond_frame, const float* mask, const float* concat_u,
                                     const float* concat_c, const float* sigmas, const int32_t* step_idx, void* unet_in_f16,
                                     int64_t ld_in, float* c_noise, int32_t T, int32_t h, int32_t w, void* stream) {
  VB_REQUIRE(x && sigmas && step_idx && unet_in_f16, "sampler_prepare: null pointer");
  VB_REQUIRE(ld_in >= 8 && ld_in % 8 == 0, "sampler_prepare: ld_in must be a multiple of 8");
  const long long total = (long long)T * h * w;
  sampler_prepare_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      x, cond_frame, mask, concat_u, concat_c, sigmas, step_idx, (__half*)unet_in_f16, ld_in, c_noise, T, h, w);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_sampler_update(float* x, const float* net_out, int64_t ld_net, const float* cond_frame,
                                    const float* mask, const float* scales, const float* sigmas, int32_t* step_idx,
                                    int32_t num_steps, int32_t T, int32_t h, int32_t w, void* stream) {
  VB_REQUIRE(x && net_out && scales && sigmas && step_idx, "sampler_update: null pointer");
  VB_REQUIRE(ld_net >= 4 && ld_net % 4 == 0, "sampler_update: ld_net must be a multiple of 4");
  const long long total = (long long)T * h * w;
  sampler_update_kernel<false, false><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      x, net_out, cond_frame, mask, scales, sigmas, step_idx, num_steps, T, h, w, ld_net, nullptr, nullptr, nullptr, 0,
      nullptr);
  step_inc_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_idx);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_sampler_update_2m(float* x, const float* net_out, int64_t ld_net, const float* cond_frame,
                                       const float* mask, const float* scales, const float* coefs, float* d_prev,
                                       const float* sigmas, int32_t* step_idx, int32_t num_steps, int32_t T, int32_t h,
                                       int32_t w, void* stream) {
  VB_REQUIRE(x && net_out && scales && coefs && d_prev && sigmas && step_idx, "sampler_update_2m: null pointer");
  VB_REQUIRE(ld_net >= 4 && ld_net % 4 == 0, "sampler_update_2m: ld_net must be a multiple of 4");
  VB_REQUIRE(((uintptr_t)coefs & 15) == 0, "sampler_update_2m: coefs must be 16-byte aligned");
  const long long total = (long long)T * h * w;
  sampler_update_kernel<true, false><<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      x, net_out, cond_frame, mask, scales, sigmas, step_idx, num_steps, T, h, w, ld_net,
      reinterpret_cast<const float4*>(coefs), d_prev, nullptr, 0, nullptr);
  step_inc_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_idx);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_sampler_update_action(float* x, const float* net_out, int64_t ld_net, const float* net_img,
                                           int64_t ld_img, const float* cond_frame, const float* mask, const float* scales,
                                           const float* action_scales, const float* coefs, float* d_prev,
                                           const float* sigmas, int32_t* step_idx, int32_t num_steps, int32_t T,
                                           int32_t h, int32_t w, void* stream) {
  VB_REQUIRE(x && net_out && net_img && scales && action_scales && sigmas && step_idx,
             "sampler_update_action: null pointer");
  VB_REQUIRE(ld_net >= 4 && ld_net % 4 == 0, "sampler_update_action: ld_net must be a multiple of 4");
  VB_REQUIRE(ld_img >= 4 && ld_img % 4 == 0, "sampler_update_action: ld_img must be a multiple of 4");
  VB_REQUIRE((coefs == nullptr) == (d_prev == nullptr),
             "sampler_update_action: coefs and d_prev are both NULL (Euler) or both given (2M)");
  VB_REQUIRE(((uintptr_t)coefs & 15) == 0, "sampler_update_action: coefs must be 16-byte aligned");
  const long long total = (long long)T * h * w;
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (coefs)
    sampler_update_kernel<true, true><<<grid, 256, 0, (cudaStream_t)stream>>>(
        x, net_out, cond_frame, mask, scales, sigmas, step_idx, num_steps, T, h, w, ld_net,
        reinterpret_cast<const float4*>(coefs), d_prev, net_img, ld_img, action_scales);
  else
    sampler_update_kernel<false, true><<<grid, 256, 0, (cudaStream_t)stream>>>(
        x, net_out, cond_frame, mask, scales, sigmas, step_idx, num_steps, T, h, w, ld_net, nullptr, nullptr, net_img,
        ld_img, action_scales);
  step_inc_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_idx);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_nchw_to_tokens(const float* x, void* out_f16, int64_t ldo, int32_t NB, int32_t C, int32_t H,
                                    int32_t W, void* stream) {
  VB_REQUIRE(x && out_f16, "nchw_to_tokens: null pointer");
  nchw_to_tokens_kernel<<<grid_for((long long)NB * C * H * W, 256), 256, 0, (cudaStream_t)stream>>>(
      x, (__half*)out_f16, ldo, NB, C, H, W);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_tokens_to_nchw(const void* x, int32_t x_is_f32, int64_t ldx, float* out, int32_t NB, int32_t C,
                                    int32_t H, int32_t W, void* stream) {
  VB_REQUIRE(x && out, "tokens_to_nchw: null pointer");
  tokens_to_nchw_kernel<<<grid_for((long long)NB * C * H * W, 256), 256, 0, (cudaStream_t)stream>>>(x, x_is_f32, ldx,
                                                                                                    out, NB, C, H, W);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// VAE decoder helpers
// ------------------------------------------------------------------------------------------
namespace vb {

// Row softmax: fp32 scores [rows, cols] (row stride ld_in) -> fp16 probabilities.  One block per row.
__global__ void __launch_bounds__(256)
softmax_rows_kernel(const float* __restrict__ x, long long ld_in, __half* __restrict__ y, long long ld_out, int cols) {
  __shared__ float red[32];
  const float* xr = x + (long long)blockIdx.x * ld_in;
  __half* yr = y + (long long)blockIdx.x * ld_out;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float mx = -INFINITY;
  for (int i = threadIdx.x * 4; i < cols; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(xr + i);
    mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < nw; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x * 4; i < cols; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(xr + i);
    sum += __expf(v.x - mx) + __expf(v.y - mx) + __expf(v.z - mx) + __expf(v.w - mx);
  }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < nw; ++i) sum += red[i];
  const float inv = 1.0f / sum;
  for (int i = threadIdx.x * 4; i < cols; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(xr + i);
    __half2 a = __floats2half2_rn(__expf(v.x - mx) * inv, __expf(v.y - mx) * inv);
    __half2 b = __floats2half2_rn(__expf(v.z - mx) * inv, __expf(v.w - mx) * inv);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&a);
    u.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(yr + i) = u;
  }
}

// AE3DConv's time_mix_conv (3 -> 3 channels, kernel (3,1,1), zero padded over frames) fused with the
// chunk-overlap rule of decode_first_stage: frames with blend[t] != 0 are averaged with what `out`
// already holds.  x: token-major fp32 [T*HW, C]; out: NCHW fp32 frames starting at out_frame0.
__global__ void time_mix_small_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                      const float* __restrict__ bias, float* __restrict__ out, const int* __restrict__ blend,
                                      int T, int HW, int C, int out_frame0, int skip_frames, long long ldx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)T * HW) return;
  const int t = (int)(i / HW), pix = (int)(i % HW);
  if (t < skip_frames) return;
  float acc[4];
  for (int co = 0; co < C; ++co) acc[co] = bias ? bias[co] : 0.f;
  for (int kt = 0; kt < 3; ++kt) {
    const int tt = t + kt - 1;
    if (tt < 0 || tt >= T) continue;
    const float* xp = x + ((long long)tt * HW + pix) * ldx;
    for (int ci = 0; ci < C; ++ci) {
      const float xv = xp[ci];
      for (int co = 0; co < C; ++co) acc[co] = fmaf(xv, w[(co * C + ci) * 3 + kt], acc[co]);
    }
  }
  const int mode = blend ? blend[t] : 0;
  for (int co = 0; co < C; ++co) {
    float* op = out + ((long long)(out_frame0 + t) * C + co) * HW + pix;
    *op = mode ? 0.5f * (*op + acc[co]) : acc[co];
  }
}

}  // namespace vb

extern "C" int b200v_softmax_rows(const float* x, int64_t ld_in, void* y_f16, int64_t ld_out, int64_t rows, int32_t cols,
                                  void* stream) {
  VB_REQUIRE(x && y_f16 && cols % 4 == 0 && ld_in % 4 == 0 && ld_out % 4 == 0, "softmax_rows: bad args");
  vb::softmax_rows_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(x, ld_in, (__half*)y_f16, ld_out, cols);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int b200v_time_mix_small(const float* x, int64_t ldx, const float* w, const float* bias, float* out,
                                    const int32_t* blend, int32_t T, int32_t HW, int32_t C, int32_t out_frame0,
                                    int32_t skip_frames, void* stream) {
  VB_REQUIRE(x && w && out && C >= 1 && C <= 4, "time_mix_small: bad args");
  const long long total = (long long)T * HW;
  vb::time_mix_small_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      x, w, bias, out, blend, T, HW, C, out_frame0, skip_frames, ldx);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
