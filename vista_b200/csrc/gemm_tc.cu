// Tap-GEMM launcher (b200v_gemm): validates the descriptor, encodes the tensor maps and launches the instantiation of
// tapgemm_kernel (gemm_tc.cuh) for the tile width and epilogue.
#include "gemm_tc.cuh"

namespace vb {
extern template const GemmKern* gemm_variants<32>();
extern template const GemmKern* gemm_variants<64>();
extern template const GemmKern* gemm_variants<96>();
extern template const GemmKern* gemm_variants<128>();
extern template const GemmKern* gemm_variants<160>();
extern template const GemmKern* gemm_variants<192>();
extern template const GemmKern* gemm_variants<224>();
extern template const GemmKern* gemm_variants<256>();
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
  VB_REQUIRE(!(d->act == 3 && (d->rowvec || d->res1 || d->res2 || d->bf16 || d->out_f32 || d->stats)),
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
    VB_REQUIRE(d->a_mode == 1 || d->a_mode == 2, "b200v_gemm: a_mode=%d invalid", d->a_mode);
    const long long out_tokens = d->a_mode == 2 ? 4ll * d->tokens : d->tokens;
    VB_REQUIRE(d->W > 0 && d->H > 0 && d->NB > 0 && (long long)d->W * d->H * d->NB == d->tokens &&
                   out_tokens < (1ll << 31) - 256,
               "b200v_gemm: W*H*NB != tokens (or output tokens >= 2^31)");
    VB_REQUIRE(d->a_mode == 1 || (d->h_pad == 0 && d->act == 0 && !d->rowvec && !d->res1 && !d->res2 && !d->bf16 &&
                                  !d->out_f32 && d->s_acc == 1.0f),
               "b200v_gemm: the upsampling mode (a_mode 2) takes bias and fused statistics only, fp16 in and out");
    VB_REQUIRE(d->box_w > 0 && d->box_h > 0 && d->box_b > 0 && d->box_w * d->box_h * d->box_b == 128,
               "b200v_gemm: box_w*box_h*box_b must be 128");
    p.W = d->W; p.H = d->H; p.NB = d->NB;
    p.BW = d->box_w; p.BH = d->box_h; p.BB = d->box_b;
    p.tiles_w = (d->W + p.BW - 1) / p.BW;
    p.tiles_h = (d->H + p.BH - 1) / p.BH;
    const int tiles_b = (d->NB + p.BB - 1) / p.BB;
    p.m_tiles = p.tiles_w * p.tiles_h * tiles_b * (d->a_mode == 2 ? 4 : 1);
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
  p.n_tiles = (d->N + d->tile_n - 1) / d->tile_n;
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
    // a_mode 2: a tile is one parity of one low-resolution box, and the tiles of a frame (4 H W / 128 of them) are
    // consecutive when boxes tile the frame exactly: groupnorm_from_partials reads a frame's partials as one block
    VB_REQUIRE(d->a_mode == 0 || (p.BB == 1 && d->W % p.BW == 0 && d->H % p.BH == 0 &&
                                  (d->a_mode == 2 || p.BW == d->W || p.BH == 1)),
               "b200v_gemm: fused statistics need token tiles of 128 consecutive tokens, or boxes that tile each frame "
               "in upsampling mode (box %d x %d x %d on %d x %d)",
               p.BW, p.BH, p.BB, d->W, d->H);
  }

  const int smem_bytes = 1024 + 1024 + p.nstages * p.stage_bytes + kStagingBytes;
  // Epilogue variant: the common fp16 feature sets are compiled in (no per-element feature tests), everything
  // else (fp32 output, unusual combinations) takes the generic instantiation of its operand type (7 fp16, 12 bf16).
  int variant = d->bf16 ? 12 : 7;
  if (d->stats) {
    variant = 9 + (d->rowvec ? 2 : (d->res1 ? 1 : 0));
  } else if (!d->bf16 && !d->out_f32) {
    const int nres = (d->res1 ? 1 : 0) + (d->res2 ? 1 : 0);
    if (d->act == 0 && !d->rowvec) variant = nres;
    else if (d->act == 0 && nres <= 1) variant = 3 + nres;
    else if (d->act == 1 && !d->rowvec && nres == 0) variant = 5;
    else if (d->act == 2) variant = 6;
    else if (d->act == 3) variant = 8;
  }
  static const GemmKern* const kByWidth[8] = {gemm_variants<32>(),  gemm_variants<64>(),  gemm_variants<96>(),
                                              gemm_variants<128>(), gemm_variants<160>(), gemm_variants<192>(),
                                              gemm_variants<224>(), gemm_variants<256>()};
  static bool attr_set[64] = {false};
  if (vb::first_use_on_device(attr_set)) {
    for (int w = 0; w < 8; ++w)
      for (int i = 0; i < kGemmVariants; ++i)
        VB_CHECK_CUDA(cudaFuncSetAttribute(kByWidth[w][i], cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem));
  }
  const long long total = (long long)p.m_tiles * p.n_tiles;
  int grid = device_sm_count();
  if (total < grid) grid = (int)total;
  const GemmKern k = kByWidth[d->tile_n / 32 - 1][variant];
  k<<<grid, kGemmThreads, smem_bytes, stream>>>(tmA, tmB, p);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
