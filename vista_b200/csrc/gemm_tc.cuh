// Tap-GEMM: persistent, warp-specialised wgmma kernel (template tapgemm_kernel<TN, ACT, RV, NRES, GEN, STATS>).
//   warpgroups 0, 1 : consumers; warpgroup g owns rows 64 g .. 64 g + 63 of the 128-token tile and issues one
//                     wgmma.m64n{TN}k16 per 16-wide K step over the TN (= tile_n) columns, accumulating in registers;
//                     then the epilogue (fragment -> smem transpose -> fused bias / row-vector / SiLU / GEGLU / GELU / residuals /
//                     GroupNorm statistics -> coalesced stores)
//   warpgroup 2     : producer; one thread issues the TMA loads (A tile 128 tokens x 64 ch per tap / K-chunk, B tile
//                     tile_n x 64).  setmaxnreg moves its registers to the consumers (40 / 232 per thread).
// The shared-memory ring (up to 8 stages) runs ahead of the consumers across tile boundaries, so the loads of tile i+1
// overlap the epilogue of tile i.  The 3x3 / (3,1,1) convolutions are implicit GEMMs: the A tile of every tap is a
// shifted 4-D TMA box of the token-major activation, zero padding comes from TMA OOB fill.  a_mode 2 convolves the
// nearest-2x upsampled view of a low-resolution tensor without materialising it: a tile is one low-resolution box and
// one output parity (py, px); within it upsampling is a shift, so every tap is again one shifted box of the low tensor.
// gemm_tn_*.cu instantiate the kernels of two tile widths each (so that they compile in parallel); gemm_tc.cu holds
// the launcher.
#pragma once
#include "../../include/vista_b200.h"
#include "host.cuh"
#include "ptx.cuh"

namespace vb {

constexpr int kMaxStages = 8;
constexpr int kABytes = 128 * 64 * 2;                 // 16 KB
constexpr int kStageBufBytes = 64 * 32 * 4;           // epilogue staging of one warpgroup: 64 rows x 32 fp32
constexpr int kStagingBytes = 2 * 2 * kStageBufBytes; // 2 warpgroups, double buffered
constexpr int kGemmThreads = 384;                     // 2 consumer warpgroups + 1 producer warpgroup

struct TGParams {
  int a_mode;
  int W, H, NB;
  int BW, BH, BB;
  int bw_sh, bh_sh;             // log2(BW), log2(BH): the box extents are powers of two (product 128)
  int tiles_w, tiles_h;
  int m_tiles, n_tiles;
  int ntaps, kc_per_tap;
  int dh[9], dw[9];
  int N;
  int nstages, stage_bytes;
  long long tokens;
  void* out;
  int ldo_b;                    // row strides in BYTES (int: one IMAD.WIDE per address)
  int out_f32, act;
  const float* bias;
  const float* rowvec;
  int ld_rowvec_b;
  int rv_div, rv_mod;
  const void* res1;
  int ld_res1_b;
  float s_res1;
  const void* res2;
  int ld_res2_b;
  float s_res2;
  float s_acc;
  // GroupNorm statistics of the OUTPUT, fused (STATS variants): per (128-token tile, 32-row quarter) column sums and sums
  // of squares of the stored values, fp32, at stats[((tile * 4 + quarter) * stats_ld + stats_col0 + n) * 2 + {0,1}];
  // the host guarantees that a tile is 128 consecutive tokens (b200v_gemm checks the box)
  float* stats;
  int stats_ld, stats_col0;
};

__device__ __forceinline__ float2 unpack2(uint32_t w, int bf16) {
  if (bf16) return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xFFFF0000u));
  return __half22float2(*reinterpret_cast<const __half2*>(&w));
}
__device__ __forceinline__ uint32_t pack2(float a, float b, int bf16) {
  if (bf16) {
    __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&t);
  }
  __half2 t = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// One 64-wide K chunk of the warpgroup's 64 x TN tile: 4 K steps of one m64nTNk16 each; a K step is 32 B (>> 4 = 2) in
// both descriptors.
template <int TN, bool BF16>
__device__ __forceinline__ void issue_kchunk(float (&acc)[TN / 2], uint64_t adesc, uint64_t bdesc, bool overwrite) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
    wgmma_ss<TN, BF16>(acc, adesc + (uint64_t)(2 * kk), bdesc + (uint64_t)(2 * kk), (overwrite && kk == 0) ? 0 : 1);
}

// TN: tile width (columns of N per tile), a multiple of 32 up to 256; BF16: bf16 operands and residuals (GEN only)
template <int TN, int ACT_, bool RV_, int NRES_, bool GEN, bool STATS = false, bool BF16 = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
tapgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const TGParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);  // 1024 B aligned (SWIZZLE_128B requirement)
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);           // [kMaxStages]
  uint64_t* empty = full + kMaxStages;                          // [kMaxStages]
  uint8_t* stages = smem + 1024;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KC = p.ntaps * p.kc_per_tap;
  // Tile schedule: CTA b walks tiles b, b + grid, ...; tile -> (m_blk, n_blk) = (tile / n_tiles, tile % n_tiles).
  const int total_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    for (int i = 0; i < p.nstages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);     // one arrival per consumer warp
    }
    fence_barrier_init();
  }
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  __syncthreads();

  if (warp >= 8) {
    // ------------------------------------------------------------ TMA producer
    setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const uint32_t tx = (uint32_t)(kABytes + TN * 128);
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m_blk = tile / p.n_tiles, n_blk = tile - m_blk * p.n_tiles;
        const int up = p.a_mode == 2;
        const int box = up ? (m_blk >> 2) : m_blk;     // a_mode 2: four output parities per low-resolution box
        const int px = up ? (m_blk & 1) : 0, py = up ? ((m_blk >> 1) & 1) : 0;
        const int tw = box % p.tiles_w;
        const int th = (box / p.tiles_w) % p.tiles_h;
        const int tb = box / (p.tiles_w * p.tiles_h);
        const int w0 = tw * p.BW, h0 = th * p.BH, b0 = tb * p.BB;
        const int n0 = n_blk * TN;
        for (int kc = 0; kc < KC; ++kc) {
          mbar_wait_relaxed(&empty[stage], phase ^ 1, 1);
          uint8_t* sA = stages + stage * p.stage_bytes;
          uint8_t* sB = sA + kABytes;
          const int tap = kc / p.kc_per_tap;
          const int c0 = (kc - tap * p.kc_per_tap) * 64;
          mbar_expect_tx(&full[stage], tx);
          // a_mode 2: upsampled pixel 2 j + px shifted by d reads low-resolution pixel j + floor((px + d) / 2)
          const int dw = up ? ((px + p.dw[tap]) >> 1) : p.dw[tap];
          const int dh = up ? ((py + p.dh[tap]) >> 1) : p.dh[tap];
          if (p.a_mode == 0)
            tma_load_2d(sA, &tmA, &full[stage], c0, w0);
          else
            tma_load_4d(sA, &tmA, &full[stage], c0, w0 + dw, h0 + dh, b0);
          tma_load_2d(sB, &tmB, &full[stage], kc * 64, n0);
          if (++stage == p.nstages) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
    return;
  }

  // ------------------------------------------------------------ consumers (warps 0 .. 7)
  setmaxnreg_inc<232>();
  const int wg = warp >> 2, wq = warp & 3;
  const int act = GEN ? p.act : ACT_;
  const bool has_rv = GEN ? (p.rowvec != nullptr) : RV_;
  const bool has_r1 = GEN ? (p.res1 != nullptr) : (NRES_ >= 1);
  const bool has_r2 = GEN ? (p.res2 != nullptr) : (NRES_ >= 2);
  constexpr bool bf16 = BF16;
  const bool f32o = GEN ? (p.out_f32 != 0) : false;
  const bool has_bias = p.bias != nullptr;
  constexpr int half = TN >> 1;
  const int tile_out_cols = (act == 2) ? half : TN;
  const int n_out_total = (act == 2) ? (p.N >> 1) : p.N;
  const int G = tile_out_cols >> 5;       // 32-column output groups per tile
  const int out_es = f32o ? 4 : 2;
  const char* r1p = reinterpret_cast<const char*>(p.res1);
  const char* r2p = reinterpret_cast<const char*>(p.res2);
  // descriptors: only the start address changes (per stage); A of this warpgroup is 64 rows (8 KB) into the A tile
  const uint64_t desc0 = make_desc_sw128(smem_u32(stages), 16, 1024);
  const uint32_t stage_step = (uint32_t)p.stage_bytes >> 4;
  const uint32_t stg0 = smem_u32(stages + p.nstages * p.stage_bytes) + wg * 2 * kStageBufBytes;
  // phase-A fragment coordinates (rows of this warp: 16 wq + g, + 8) and phase-B coordinates (32 rows x 16 columns)
  const int g = lane >> 2, c = lane & 3;
  const int rh = wq & 1, chh = wq >> 1;
  const int ch = lane & 3, rsub = lane >> 2;
  int stage = 0;
  uint32_t phase = 0;
  uint32_t gcount = 0;                   // epilogue groups done by this warpgroup: selects the staging buffer

  float acc[TN / 2];
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int m_blk = tile / p.n_tiles, n_blk = tile - m_blk * p.n_tiles;
    // ---------------- main loop
    int prev = -1;
    for (int kc = 0; kc < KC; ++kc) {
      mbar_wait(&full[stage], phase, 3);
      const uint64_t ad = desc0 + (uint64_t)(stage * stage_step + wg * 512);
      const uint64_t bd = desc0 + (uint64_t)(stage * stage_step + (kABytes >> 4));
      wgmma_fence();
      issue_kchunk<TN, BF16>(acc, ad, bd, kc == 0);
      wgmma_commit();
      if (prev >= 0) {                   // the chunk before this one has been read: free its slot
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = stage;
      if (++stage == p.nstages) {
        stage = 0;
        phase ^= 1;
      }
    }
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&empty[prev]);
    fence_regs(acc);

    // ---------------- epilogue: rows of phase B (32 per warp) -> tokens
    const int r_own = wg * 64 + rh * 32 + lane;   // tile row this lane resolves
    int token_own, valid_own;
    if (p.a_mode == 0) {
      token_own = m_blk * 128 + r_own;
      valid_own = token_own < p.tokens;
    } else {
      const int up = p.a_mode == 2;
      const int box = up ? (m_blk >> 2) : m_blk;
      const int tw = box % p.tiles_w;
      const int t2 = box / p.tiles_w;
      const int th = t2 % p.tiles_h;
      const int tb = t2 / p.tiles_h;
      const int ww = r_own & (p.BW - 1), hh = (r_own >> p.bw_sh) & (p.BH - 1), bb = r_own >> (p.bw_sh + p.bh_sh);
      const int w = tw * p.BW + ww, h = th * p.BH + hh, b = tb * p.BB + bb;
      valid_own = (w < p.W) && (h < p.H) && (b < p.NB);
      // a_mode 2: output pixel (2 h + py, 2 w + px) of the (2 H) x (2 W) frame
      token_own = up ? ((2 * (b * p.H + h) + ((m_blk >> 1) & 1)) * 2 * p.W + 2 * w + (m_blk & 1))
                     : (b * p.H + h) * p.W + w;
    }
    if (!valid_own) token_own = 0;
    // phase-B row i of this lane = 8 i + rsub (of the warp's 32)
    const uint32_t vrows = __ballot_sync(0xffffffffu, valid_own) >> rsub;   // bit 8 i <-> row i
    int tok[4], rvrow[4];
    {
      const int rv_own = has_rv ? (token_own / p.rv_div) % p.rv_mod : 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        tok[i] = __shfl_sync(0xffffffffu, token_own, i * 8 + rsub);
        rvrow[i] = has_rv ? __shfl_sync(0xffffffffu, rv_own, i * 8 + rsub) : 0;
      }
    }
    const int n_out_base = n_blk * tile_out_cols;
#pragma unroll
    for (int k = 0; k < TN / 32; ++k) {
      if (k >= G) break;
      const int c0 = k * 32;
      if (n_out_base + c0 >= n_out_total) break;   // groups entirely beyond N (last n-tile of a padded N)
      const uint32_t stg = stg0 + (gcount & 1) * kStageBufBytes;
      ++gcount;
      // ---------------- phase A: the warp's 16 rows x 32 columns of the fragment -> staging (16-byte chunks XOR-swizzled
      // by row).  GEGLU is evaluated here (value * gelu(gate)); every other epilogue moves the raw accumulator.
      float f[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) f[j] = acc[16 * k + j];
      if (act == 2) {
        float gt[16];                     // gate columns half + c0 .. : group half / 32 + k of the accumulator
        const int kg = (half >> 5) + k;
#pragma unroll
        for (int j = 0; j < 16; ++j) gt[j] = 0.f;
#pragma unroll
        for (int q = 0; q < TN / 32; ++q)
          if (q == kg) {
#pragma unroll
            for (int j = 0; j < 16; ++j) gt[j] = acc[16 * q + j];
          }
        const int nb = n_blk * TN + c0;    // bias index of the value columns (gate: + half)
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
          float2 bv = make_float2(0.f, 0.f), bg = make_float2(0.f, 0.f);
          if (has_bias) {
            bv = __ldg(reinterpret_cast<const float2*>(p.bias + nb + 8 * ii + 2 * c));
            bg = __ldg(reinterpret_cast<const float2*>(p.bias + nb + half + 8 * ii + 2 * c));
          }
          f[4 * ii + 0] = geglu_fast(f[4 * ii + 0] + bv.x, gt[4 * ii + 0] + bg.x);
          f[4 * ii + 1] = geglu_fast(f[4 * ii + 1] + bv.y, gt[4 * ii + 1] + bg.y);
          f[4 * ii + 2] = geglu_fast(f[4 * ii + 2] + bv.x, gt[4 * ii + 2] + bg.x);
          f[4 * ii + 3] = geglu_fast(f[4 * ii + 3] + bv.y, gt[4 * ii + 3] + bg.y);
        }
      }
#pragma unroll
      for (int ii = 0; ii < 4; ++ii) {
        const int chunk = 2 * ii + (c >> 1), sub = (c & 1) * 8;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int row = wq * 16 + g + 8 * hr;
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stg + row * 128 + ((chunk ^ (row & 7)) << 4) + sub),
                       "f"(f[4 * ii + 2 * hr]), "f"(f[4 * ii + 2 * hr + 1])
                       : "memory");
        }
      }
      asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
      // ---------------- phase B (lane = 4 fixed columns, 8 rows per instruction): bias / s_acc / row-vector / SiLU /
      // residuals / pack / store; every global access covers a contiguous row segment of 16 output elements
      {
        const int n = n_out_base + c0 + chh * 16 + ch * 4;
        const bool n_ok = n + 4 <= n_out_total;
        float4 bs = make_float4(0.f, 0.f, 0.f, 0.f);
        float sa = 1.0f;
        if (act != 2) {
          sa = p.s_acc;
          if (has_bias && n_ok) {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + n));
            bs = make_float4(b4.x * sa, b4.y * sa, b4.z * sa, b4.w * sa);
          }
        }
        char* obase = reinterpret_cast<char*>(p.out) + (long long)n * out_es;
        const char* r1base = r1p + (long long)n * 2;
        const char* r2base = r2p + (long long)n * 2;
        const char* rvbase = reinterpret_cast<const char*>(p.rowvec) + (long long)n * 4;
        float cs[4] = {0.f, 0.f, 0.f, 0.f}, cq[4] = {0.f, 0.f, 0.f, 0.f};   // STATS: column sums over this lane's rows
        float4 v[4], rv[4];
        uint2 u1[4], u2[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int row = rh * 32 + i * 8 + rsub;
          const int chunk = chh * 4 + ch;
          asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                       : "=f"(v[i].x), "=f"(v[i].y), "=f"(v[i].z), "=f"(v[i].w)
                       : "r"(stg + row * 128 + ((chunk ^ (row & 7)) << 4)));
          const bool ok = n_ok && ((vrows >> (8 * i)) & 1u);
          rv[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          u1[i] = make_uint2(0, 0);
          u2[i] = make_uint2(0, 0);
          if (has_rv && ok) rv[i] = __ldg(reinterpret_cast<const float4*>(rvbase + (long long)rvrow[i] * p.ld_rowvec_b));
          if (has_r1 && ok) u1[i] = __ldg(reinterpret_cast<const uint2*>(r1base + (long long)tok[i] * p.ld_res1_b));
          if (has_r2 && ok) u2[i] = __ldg(reinterpret_cast<const uint2*>(r2base + (long long)tok[i] * p.ld_res2_b));
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const bool ok = n_ok && ((vrows >> (8 * i)) & 1u);   // straight-line code, predicated store
          float4 o = v[i];
          if (act != 2) {
            o.x = fmaf(o.x, sa, bs.x); o.y = fmaf(o.y, sa, bs.y); o.z = fmaf(o.z, sa, bs.z); o.w = fmaf(o.w, sa, bs.w);
            if (has_rv) { o.x += rv[i].x; o.y += rv[i].y; o.z += rv[i].z; o.w += rv[i].w; }
            if (act == 1) { o.x = silu_f(o.x); o.y = silu_f(o.y); o.z = silu_f(o.z); o.w = silu_f(o.w); }
            if (!GEN && act == 3) { o.x = gelu_erf_fast(o.x); o.y = gelu_erf_fast(o.y); o.z = gelu_erf_fast(o.z); o.w = gelu_erf_fast(o.w); }
            if (has_r1) {
              const float2 a = unpack2(u1[i].x, bf16), b = unpack2(u1[i].y, bf16);
              o.x = fmaf(p.s_res1, a.x, o.x); o.y = fmaf(p.s_res1, a.y, o.y);
              o.z = fmaf(p.s_res1, b.x, o.z); o.w = fmaf(p.s_res1, b.y, o.w);
            }
            if (has_r2) {
              const float2 a = unpack2(u2[i].x, bf16), b = unpack2(u2[i].y, bf16);
              o.x = fmaf(p.s_res2, a.x, o.x); o.y = fmaf(p.s_res2, a.y, o.y);
              o.z = fmaf(p.s_res2, b.x, o.z); o.w = fmaf(p.s_res2, b.y, o.w);
            }
          }
          if (STATS && ok) {
            cs[0] += o.x; cs[1] += o.y; cs[2] += o.z; cs[3] += o.w;
            cq[0] = fmaf(o.x, o.x, cq[0]); cq[1] = fmaf(o.y, o.y, cq[1]);
            cq[2] = fmaf(o.z, o.z, cq[2]); cq[3] = fmaf(o.w, o.w, cq[3]);
          }
          char* optr = obase + (long long)tok[i] * p.ldo_b;
          if (f32o) {
            if (ok) *reinterpret_cast<float4*>(optr) = o;
          } else {
            const uint2 pk = make_uint2(pack2(o.x, o.y, bf16), pack2(o.z, o.w, bf16));
            if (ok) *reinterpret_cast<uint2*>(optr) = pk;
          }
        }
        if (STATS) {
          // rows of one column live in lanes ch, ch + 4, ...: fixed-order butterfly, then lane rsub == 0 holds the sums
          // over the warp's 32 rows (quarter 2 wg + rh of the tile) and writes them: bit-reproducible
#pragma unroll
          for (int off = 4; off < 32; off <<= 1) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              cs[q] += __shfl_xor_sync(0xffffffffu, cs[q], off);
              cq[q] += __shfl_xor_sync(0xffffffffu, cq[q], off);
            }
          }
          if (rsub == 0 && n_ok) {
            float* dst = p.stats + (((long long)m_blk * 4 + wg * 2 + rh) * p.stats_ld + p.stats_col0 + n) * 2;
            *reinterpret_cast<float4*>(dst) = make_float4(cs[0], cq[0], cs[1], cq[1]);
            *reinterpret_cast<float4*>(dst + 4) = make_float4(cs[2], cq[2], cs[3], cq[3]);
          }
        }
      }
    }
  }
}

using GemmKern = void (*)(const CUtensorMap, const CUtensorMap, const TGParams);
constexpr int kGemmVariants = 13;

// The instantiations of one tile width, indexed by epilogue variant: 0-2 plain with 0 / 1 / 2 residuals, 3-4 row vector
// with 0 / 1 residual, 5 SiLU, 6 GEGLU, 7 generic fp16 (every feature a runtime test), 8 erf-GELU, 9-11 fused
// statistics (plain, one residual, row vector), 12 generic bf16.
template <int TN>
const GemmKern* gemm_variants() {
  static const GemmKern v[kGemmVariants] = {
      tapgemm_kernel<TN, 0, false, 0, false>,       tapgemm_kernel<TN, 0, false, 1, false>,
      tapgemm_kernel<TN, 0, false, 2, false>,       tapgemm_kernel<TN, 0, true, 0, false>,
      tapgemm_kernel<TN, 0, true, 1, false>,        tapgemm_kernel<TN, 1, false, 0, false>,
      tapgemm_kernel<TN, 2, false, 0, false>,       tapgemm_kernel<TN, 0, true, 2, true>,
      tapgemm_kernel<TN, 3, false, 0, false>,       tapgemm_kernel<TN, 0, false, 0, false, true>,
      tapgemm_kernel<TN, 0, false, 1, false, true>, tapgemm_kernel<TN, 0, true, 0, false, true>,
      tapgemm_kernel<TN, 0, true, 2, true, false, true>};
  return v;
}

}  // namespace vb
