// Tap-GEMM: persistent, warp-specialised wgmma kernel (template tapgemm_kernel<ACT, RV, NRES, GEN, STATS>).
//   warpgroups 0, 1 : consumers; warpgroup g owns rows 64 g .. 64 g + 63 of the 128-token tile and issues
//                     wgmma.m64n64k16 (m64n32k16 for a 32-column tail) over the tile_n columns, accumulating in registers;
//                     then the epilogue (fragment -> smem transpose -> fused bias / row-vector / SiLU / GEGLU / GELU / residuals /
//                     GroupNorm statistics -> coalesced stores)
//   warpgroup 2     : producer; one thread issues the TMA loads (A tile 128 tokens x 64 ch per tap / K-chunk, B tile
//                     tile_n x 64).  setmaxnreg moves its registers to the consumers (40 / 232 per thread).
// The shared-memory ring (up to 8 stages) runs ahead of the consumers across tile boundaries, so the loads of tile i+1
// overlap the epilogue of tile i.  The 3x3 / (3,1,1) convolutions are implicit GEMMs: the A tile of every tap is a
// shifted 4-D TMA box of the token-major activation, zero padding comes from TMA OOB fill.
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
  int N, TN;
  int bf16;
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

// One 64-wide K chunk of the warpgroup's 64 x TN tile: 4 K steps x (nfull 64-column slices + an optional 32-column tail).
// B slice s starts 64 rows (8 KB, >> 4 = 512) after slice s - 1; a K step is 32 B (>> 4 = 2) in both descriptors.
template <bool BF16>
__device__ __forceinline__ void issue_kchunk(float (&acc)[4][32], uint64_t adesc, uint64_t bdesc, int nfull, bool tail,
                                             bool overwrite) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const int sc = (overwrite && kk == 0) ? 0 : 1;
    const uint64_t ad = adesc + (uint64_t)(2 * kk);
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const uint64_t bd = bdesc + (uint64_t)(512 * s + 2 * kk);
      if (s < nfull) {
        if (BF16) wgmma_m64n64_bf16(acc[s], ad, bd, sc); else wgmma_m64n64_f16(acc[s], ad, bd, sc);
      } else if (s == nfull && tail) {
        float(&t)[16] = *reinterpret_cast<float(*)[16]>(&acc[s][0]);
        if (BF16) wgmma_m64n32_bf16(t, ad, bd, sc); else wgmma_m64n32_f16(t, ad, bd, sc);
      }
    }
  }
}

template <int ACT_, bool RV_, int NRES_, bool GEN, bool STATS = false>
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
      const uint32_t tx = (uint32_t)(kABytes + p.TN * 128);
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m_blk = tile / p.n_tiles, n_blk = tile - m_blk * p.n_tiles;
        const int tw = m_blk % p.tiles_w;
        const int th = (m_blk / p.tiles_w) % p.tiles_h;
        const int tb = m_blk / (p.tiles_w * p.tiles_h);
        const int w0 = tw * p.BW, h0 = th * p.BH, b0 = tb * p.BB;
        const int n0 = n_blk * p.TN;
        for (int kc = 0; kc < KC; ++kc) {
          mbar_wait_relaxed(&empty[stage], phase ^ 1, 1);
          uint8_t* sA = stages + stage * p.stage_bytes;
          uint8_t* sB = sA + kABytes;
          const int tap = kc / p.kc_per_tap;
          const int c0 = (kc - tap * p.kc_per_tap) * 64;
          mbar_expect_tx(&full[stage], tx);
          if (p.a_mode == 0)
            tma_load_2d(sA, &tmA, &full[stage], c0, w0);
          else
            tma_load_4d(sA, &tmA, &full[stage], c0, w0 + p.dw[tap], h0 + p.dh[tap], b0);
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
  const bool bf16 = GEN ? (p.bf16 != 0) : false;
  const bool f32o = GEN ? (p.out_f32 != 0) : false;
  const bool has_bias = p.bias != nullptr;
  const int nfull = p.TN >> 6;
  const bool tail = (p.TN & 32) != 0;
  const int half = p.TN >> 1;
  const int tile_out_cols = (act == 2) ? half : p.TN;
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

  float acc[4][32];
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int m_blk = tile / p.n_tiles, n_blk = tile - m_blk * p.n_tiles;
    // ---------------- main loop
    int prev = -1;
    for (int kc = 0; kc < KC; ++kc) {
      mbar_wait(&full[stage], phase, 3);
      const uint64_t ad = desc0 + (uint64_t)(stage * stage_step + wg * 512);
      const uint64_t bd = desc0 + (uint64_t)(stage * stage_step + (kABytes >> 4));
      wgmma_fence();
      if (GEN && bf16) issue_kchunk<true>(acc, ad, bd, nfull, tail, kc == 0);
      else issue_kchunk<false>(acc, ad, bd, nfull, tail, kc == 0);
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
#pragma unroll
    for (int s = 0; s < 4; ++s) fence_regs(acc[s]);

    // ---------------- epilogue: rows of phase B (32 per warp) -> tokens
    const int r_own = wg * 64 + rh * 32 + lane;   // tile row this lane resolves
    int token_own, valid_own;
    if (p.a_mode == 0) {
      token_own = m_blk * 128 + r_own;
      valid_own = token_own < p.tokens;
    } else {
      const int tw = m_blk % p.tiles_w;
      const int t2 = m_blk / p.tiles_w;
      const int th = t2 % p.tiles_h;
      const int tb = t2 / p.tiles_h;
      const int ww = r_own & (p.BW - 1), hh = (r_own >> p.bw_sh) & (p.BH - 1), bb = r_own >> (p.bw_sh + p.bh_sh);
      const int w = tw * p.BW + ww, h = th * p.BH + hh, b = tb * p.BB + bb;
      valid_own = (w < p.W) && (h < p.H) && (b < p.NB);
      token_own = (b * p.H + h) * p.W + w;
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
    for (int k = 0; k < 8; ++k) {
      if (k >= G) break;
      const int c0 = k * 32;
      if (n_out_base + c0 >= n_out_total) break;   // groups entirely beyond N (last n-tile of a padded N)
      const uint32_t stg = stg0 + (gcount & 1) * kStageBufBytes;
      ++gcount;
      // ---------------- phase A: the warp's 16 rows x 32 columns of the fragment -> staging (16-byte chunks XOR-swizzled
      // by row).  GEGLU is evaluated here (value * gelu(gate)); every other epilogue moves the raw accumulator.
      float f[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) f[j] = acc[k >> 1][(k & 1) * 16 + j];
      if (act == 2) {
        float gt[16];                     // gate columns half + c0 .. : group half / 32 + k of the accumulator
        const int kg = (half >> 5) + k;
#pragma unroll
        for (int j = 0; j < 16; ++j) gt[j] = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q)
          if (q == kg) {
#pragma unroll
            for (int j = 0; j < 16; ++j) gt[j] = acc[q >> 1][(q & 1) * 16 + j];
          }
        const int nb = n_blk * p.TN + c0;  // bias index of the value columns (gate: + half)
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

}  // namespace vb

extern "C" int b200v_gemm(const b200v_gemm_desc* d, void* stream_) {
  using namespace vb;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  VB_REQUIRE(d && d->a && d->b && d->out, "b200v_gemm: null pointer");
  VB_REQUIRE(d->cin > 0 && d->cin % 64 == 0, "b200v_gemm: cin=%d must be a positive multiple of 64", d->cin);
  VB_REQUIRE(d->ntaps >= 1 && d->ntaps <= 9, "b200v_gemm: ntaps=%d out of range", d->ntaps);
  VB_REQUIRE(d->N > 0 && d->N % 8 == 0, "b200v_gemm: N=%d must be a multiple of 8", d->N);
  VB_REQUIRE(d->tile_n >= 32 && d->tile_n <= 256 && d->tile_n % 32 == 0, "b200v_gemm: tile_n=%d invalid", d->tile_n);
  VB_REQUIRE(d->lda % 8 == 0 && d->ldo % 8 == 0, "b200v_gemm: lda/ldo must be multiples of 8");
  VB_REQUIRE(d->act >= 0 && d->act <= 3, "b200v_gemm: act=%d invalid", d->act);
  VB_REQUIRE(!(d->act == 2 && (d->tile_n % 64 != 0 || d->N % d->tile_n != 0 || d->out_f32)),
             "b200v_gemm: GEGLU needs tile_n %% 64 == 0, N %% tile_n == 0, 16-bit output");
  VB_REQUIRE(!(d->act == 2 && (d->rowvec || d->res1 || d->res2)), "b200v_gemm: GEGLU epilogue takes bias only");
  VB_REQUIRE(!(d->act == 3 && (d->rowvec || d->res1 || d->res2 || d->bf16 || d->out_f32 || d->stats || getenv("VB_GEMM_GENERIC"))),
             "b200v_gemm: the GELU epilogue takes bias only, fp16 operands and output (compiled variant)");
  VB_REQUIRE(!d->res1 || d->ld_res1 % 8 == 0, "b200v_gemm: ld_res1 must be a multiple of 8");
  VB_REQUIRE(!d->res2 || d->ld_res2 % 8 == 0, "b200v_gemm: ld_res2 must be a multiple of 8");
  VB_REQUIRE(!d->rowvec || (d->ld_rowvec % 4 == 0 && d->rv_div > 0 && d->rv_mod > 0), "b200v_gemm: bad rowvec args");
  VB_REQUIRE((reinterpret_cast<uintptr_t>(d->a) & 15) == 0 && (reinterpret_cast<uintptr_t>(d->b) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(d->out) & 15) == 0,
             "b200v_gemm: a/b/out must be 16-byte aligned");

  TGParams p;
  memset(&p, 0, sizeof(p));
  p.a_mode = d->a_mode;
  p.tokens = d->tokens;
  const long long K = (long long)d->ntaps * d->cin;
  CUtensorMap tmA, tmB;
  if (d->a_mode == 0) {
    VB_REQUIRE(d->ntaps == 1 && d->h_pad == 0, "b200v_gemm: linear mode takes one tap and no halo rows");
    VB_REQUIRE(d->tokens > 0 && d->tokens < (1ll << 31) - 256, "b200v_gemm: tokens out of range");
    p.W = (int)d->tokens; p.H = 1; p.NB = 1;
    p.BW = 128; p.BH = 1; p.BB = 1;
    p.tiles_w = (int)((d->tokens + 127) / 128); p.tiles_h = 1;
    p.m_tiles = p.tiles_w;
    uint64_t dims[2] = {(uint64_t)d->cin, (uint64_t)d->tokens};
    uint64_t strides[1] = {(uint64_t)d->lda * 2};
    uint32_t box[2] = {64, 128};
    uint32_t es[2] = {1, 1};
    if (encode_tmap_16bit(&tmA, d->a, 2, dims, strides, box, es, d->bf16)) return 3;
  } else {
    VB_REQUIRE(d->W > 0 && d->H > 0 && d->NB > 0 && (long long)d->W * d->H * d->NB == d->tokens &&
                   d->tokens < (1ll << 31) - 256,
               "b200v_gemm: W*H*NB != tokens (or >= 2^31)");
    VB_REQUIRE(d->box_w > 0 && d->box_h > 0 && d->box_b > 0 && d->box_w * d->box_h * d->box_b == 128,
               "b200v_gemm: box_w*box_h*box_b must be 128");
    p.W = d->W; p.H = d->H; p.NB = d->NB;
    p.BW = d->box_w; p.BH = d->box_h; p.BB = d->box_b;
    p.tiles_w = (d->W + p.BW - 1) / p.BW;
    p.tiles_h = (d->H + p.BH - 1) / p.BH;
    const int tiles_b = (d->NB + p.BB - 1) / p.BB;
    p.m_tiles = p.tiles_w * p.tiles_h * tiles_b;
    VB_REQUIRE(d->h_pad >= 0 && d->h_pad <= 4, "b200v_gemm: h_pad=%d out of range", d->h_pad);
    const uint64_t He = (uint64_t)d->H + 2ull * d->h_pad;     // rows of H in memory (halo rows before and after)
    uint64_t dims[4] = {(uint64_t)d->cin, (uint64_t)d->W, He, (uint64_t)d->NB};
    uint64_t strides[3] = {(uint64_t)d->lda * 2, (uint64_t)d->lda * 2 * d->W, (uint64_t)d->lda * 2 * d->W * He};
    uint32_t box[4] = {64, (uint32_t)p.BW, (uint32_t)p.BH, (uint32_t)p.BB};
    uint32_t es[4] = {1, 1, 1, 1};
    if (encode_tmap_16bit(&tmA, d->a, 4, dims, strides, box, es, d->bf16)) return 3;
  }
  {
    uint64_t dims[2] = {(uint64_t)K, (uint64_t)d->N};
    uint64_t strides[1] = {(uint64_t)K * 2};
    uint32_t box[2] = {64, (uint32_t)d->tile_n};
    uint32_t es[2] = {1, 1};
    if (encode_tmap_16bit(&tmB, d->b, 2, dims, strides, box, es, d->bf16)) return 3;
  }
  p.ntaps = d->ntaps;
  p.kc_per_tap = d->cin / 64;
  for (int i = 0; i < 9; ++i) {
    p.dh[i] = d->dh[i] + (d->a_mode == 1 ? d->h_pad : 0);   // TMA coordinates count from the first halo row
    p.dw[i] = d->dw[i];
  }
  p.N = d->N;
  p.TN = d->tile_n;
  p.n_tiles = (d->N + d->tile_n - 1) / d->tile_n;
  p.bf16 = d->bf16;
  p.stage_bytes = kABytes + ((d->tile_n * 128 + 1023) / 1024) * 1024;
  constexpr int kMaxSmem = 227 * 1024;         // opt-in dynamic shared memory per block on sm_90
  p.nstages = (kMaxSmem - 2048 - kStagingBytes) / p.stage_bytes;
  if (p.nstages > kMaxStages) p.nstages = kMaxStages;
  const long long kMaxLd = (1ll << 31) - 1;
  VB_REQUIRE(d->ldo * (d->out_f32 ? 4 : 2) <= kMaxLd && d->ld_rowvec * 4 <= kMaxLd && d->ld_res1 * 2 <= kMaxLd &&
                 d->ld_res2 * 2 <= kMaxLd,
             "b200v_gemm: row stride too large");
  for (p.bw_sh = 0; (1 << p.bw_sh) < p.BW; ++p.bw_sh) {}
  for (p.bh_sh = 0; (1 << p.bh_sh) < p.BH; ++p.bh_sh) {}
  p.out = d->out; p.ldo_b = (int)(d->ldo * (d->out_f32 ? 4 : 2)); p.out_f32 = d->out_f32; p.act = d->act;
  p.bias = d->bias;
  p.rowvec = d->rowvec; p.ld_rowvec_b = (int)(d->ld_rowvec * 4); p.rv_div = d->rv_div > 0 ? d->rv_div : 1;
  p.rv_mod = d->rv_mod > 0 ? d->rv_mod : 1;
  p.res1 = d->res1; p.ld_res1_b = (int)(d->ld_res1 * 2); p.s_res1 = d->s_res1;
  p.res2 = d->res2; p.ld_res2_b = (int)(d->ld_res2 * 2); p.s_res2 = d->s_res2;
  p.s_acc = d->s_acc;
  VB_REQUIRE(!(d->res2 && !d->res1), "b200v_gemm: res2 without res1");
  p.stats = d->stats; p.stats_ld = (int)d->stats_ld; p.stats_col0 = d->stats_col0;
  if (d->stats) {
    VB_REQUIRE(!d->bf16 && !d->out_f32 && d->act == 0 && !d->res2 && !(d->rowvec && d->res1),
               "b200v_gemm: fused statistics need fp16 output, act 0, <= 1 residual and no rowvec + residual");
    VB_REQUIRE(d->stats_ld >= d->stats_col0 + d->N && d->stats_col0 % 4 == 0 && d->stats_ld % 4 == 0 &&
                   (reinterpret_cast<uintptr_t>(d->stats) & 15) == 0,
               "b200v_gemm: bad stats_ld / stats_col0 / alignment");
    VB_REQUIRE(d->a_mode == 0 || (p.BB == 1 && d->W % p.BW == 0 && d->H % p.BH == 0 && (p.BW == d->W || p.BH == 1)),
               "b200v_gemm: fused statistics need token tiles of 128 consecutive tokens (box %d x %d x %d on %d x %d)",
               p.BW, p.BH, p.BB, d->W, d->H);
  }

  const int smem_bytes = 1024 + 1024 + p.nstages * p.stage_bytes + kStagingBytes;
  // Epilogue variant: the common fp16 feature sets are compiled in (no per-element feature tests), everything
  // else (bf16 operands, fp32 output, unusual combinations) takes the generic instantiation.
  using Kern = void (*)(const CUtensorMap, const CUtensorMap, const TGParams);
  static const Kern kVariants[9] = {tapgemm_kernel<0, false, 0, false>, tapgemm_kernel<0, false, 1, false>,
                                    tapgemm_kernel<0, false, 2, false>, tapgemm_kernel<0, true, 0, false>,
                                    tapgemm_kernel<0, true, 1, false>,  tapgemm_kernel<1, false, 0, false>,
                                    tapgemm_kernel<2, false, 0, false>, tapgemm_kernel<0, true, 2, true>,
                                    tapgemm_kernel<3, false, 0, false>};
  int variant = 7;
  if (!d->bf16 && !d->out_f32 && !getenv("VB_GEMM_GENERIC")) {
    const int nres = (d->res1 ? 1 : 0) + (d->res2 ? 1 : 0);
    if (d->act == 0 && !d->rowvec) variant = nres;
    else if (d->act == 0 && nres <= 1) variant = 3 + nres;
    else if (d->act == 1 && !d->rowvec && nres == 0) variant = 5;
    else if (d->act == 2) variant = 6;
    else if (d->act == 3) variant = 8;
  }
  // fused-statistics instantiations: plain, one residual, row vector
  static const Kern kStats[3] = {tapgemm_kernel<0, false, 0, false, true>, tapgemm_kernel<0, false, 1, false, true>,
                                 tapgemm_kernel<0, true, 0, false, true>};
  static bool attr_set[64] = {false};
  if (vb::first_use_on_device(attr_set)) {
    for (int i = 0; i < 3; ++i)
      VB_CHECK_CUDA(cudaFuncSetAttribute(kStats[i], cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
    for (int i = 0; i < 9; ++i)
      VB_CHECK_CUDA(cudaFuncSetAttribute(kVariants[i], cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
  }
  const long long total = (long long)p.m_tiles * p.n_tiles;
  int grid = device_sm_count();
  if (total < grid) grid = (int)total;
  const Kern k = d->stats ? kStats[d->rowvec ? 2 : (d->res1 ? 1 : 0)] : kVariants[variant];
  k<<<grid, kGemmThreads, smem_bytes, stream>>>(tmA, tmB, p);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
