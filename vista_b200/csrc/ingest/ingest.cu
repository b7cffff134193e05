// Camera frames in (sample.py:174-201, load_img): uint8 RGB frames, cropped and Lanczos-resized exactly as Pillow's 8-bit
// resampler does it (Resample.c, ImagingResampleHorizontal_8bpc / ImagingResampleVertical_8bpc), then ToTensor and
// x * 2 - 1 into fp32 (T, 3, H, W).
//
// Pillow's resampler is integer arithmetic once its coefficient tables exist: per output index an input window
// (xmin, n) and n int32 weights in 22-bit fixed point.  The tables are built on the host in double (vista_b200/ingest.py)
// and uploaded once per geometry, so the kernels only multiply and add integers and the bytes match Pillow's.
//   resize_h_kernel : horizontal pass over the cropped frame's rows [y_first, y_first + y_rows) -> uint8 scratch
//                     (T, y_rows, W, 3); only the rows the vertical pass reads are computed (Pillow's ybox_first/last).
//   resize_v_kernel : vertical pass (or none, when the height is unchanged) over the scratch or, when the width is
//                     unchanged, straight over the cropped frame, then u8 / 255 * 2 - 1 into fp32 (T, 3, H, W).
#include "../../../include/vista_b200.h"
#include "../host.cuh"

namespace vb {

constexpr int kIngestThreads = 256;
constexpr int kIngestMaxTaps = 1024;      // input window per output pixel: a shrink by up to 170x per axis
constexpr int kPrecisionBits = 22;        // Resample.c PRECISION_BITS

__device__ __forceinline__ uint8_t clip8(int acc) {
  const int v = acc >> kPrecisionBits;    // arithmetic shift, as Pillow's clip8 lookup index
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// one thread per intermediate pixel (t, r, x), 3 channels
__global__ void __launch_bounds__(kIngestThreads) resize_h_kernel(
    const uint8_t* __restrict__ src, long long frame_stride, long long row_stride, const int* __restrict__ bounds,
    const int* __restrict__ weights, int ksize, int T, int y_rows, int W, uint8_t* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long per_frame = (long long)y_rows * W;
  if (i >= (long long)T * per_frame) return;
  const int t = (int)(i / per_frame);
  const int rem = (int)(i - (long long)t * per_frame);
  const int r = rem / W, x = rem - r * W;
  const int xmin = __ldg(bounds + 2 * x), n = __ldg(bounds + 2 * x + 1);
  const uint8_t* p = src + (long long)t * frame_stride + (long long)r * row_stride + 3LL * xmin;
  const int* k = weights + (long long)x * ksize;
  int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
  for (int j = 0; j < n; ++j) {
    const int w = __ldg(k + j);
    a0 += (int)__ldg(p + 3 * j) * w;
    a1 += (int)__ldg(p + 3 * j + 1) * w;
    a2 += (int)__ldg(p + 3 * j + 2) * w;
  }
  uint8_t* o = dst + 3 * i;
  o[0] = clip8(a0);
  o[1] = clip8(a1);
  o[2] = clip8(a2);
}

// torchvision to_tensor (uint8 -> fp32, div(255), correctly rounded) followed by x * 2.0 - 1.0, one rounding per op
__device__ __forceinline__ float to_unit(uint8_t u) {
  return __fsub_rn(__fmul_rn(__fdiv_rn((float)u, 255.0f), 2.0f), 1.0f);
}

// one thread per output pixel (t, y, x), 3 channels; kVertical = false: the height is unchanged, row y is read as is
template <bool kVertical>
__global__ void __launch_bounds__(kIngestThreads) resize_v_kernel(
    const uint8_t* __restrict__ src, long long frame_stride, long long row_stride, int row_offset,
    const int* __restrict__ bounds, const int* __restrict__ weights, int ksize, int T, int H, int W,
    float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long hw = (long long)H * W;
  if (i >= (long long)T * hw) return;
  const int t = (int)(i / hw);
  const int pix = (int)(i - (long long)t * hw);
  const int y = pix / W, x = pix - y * W;
  const uint8_t* col = src + (long long)t * frame_stride + 3LL * x;
  uint8_t v0, v1, v2;
  if (kVertical) {
    const int ymin = __ldg(bounds + 2 * y), n = __ldg(bounds + 2 * y + 1);
    const uint8_t* p = col + (long long)(ymin - row_offset) * row_stride;
    const int* k = weights + (long long)y * ksize;
    int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
    for (int j = 0; j < n; ++j) {
      const int w = __ldg(k + j);
      const uint8_t* q = p + (long long)j * row_stride;
      a0 += (int)__ldg(q) * w;
      a1 += (int)__ldg(q + 1) * w;
      a2 += (int)__ldg(q + 2) * w;
    }
    v0 = clip8(a0);
    v1 = clip8(a1);
    v2 = clip8(a2);
  } else {
    const uint8_t* q = col + (long long)(y - row_offset) * row_stride;
    v0 = __ldg(q);
    v1 = __ldg(q + 1);
    v2 = __ldg(q + 2);
  }
  float* o = out + (long long)t * 3 * hw + pix;
  o[0] = to_unit(v0);
  o[hw] = to_unit(v1);
  o[2 * hw] = to_unit(v2);
}

static unsigned ingest_blocks(long long n) { return (unsigned)((n + kIngestThreads - 1) / kIngestThreads); }

}  // namespace vb

extern "C" int b200v_frames_u8_resize(const uint8_t* src, int64_t frame_stride, int64_t row_stride, int32_t T,
                                      int32_t src_h, int32_t src_w, int32_t crop_x, int32_t crop_y, int32_t crop_w,
                                      int32_t crop_h, int32_t out_h, int32_t out_w, const int32_t* xbounds,
                                      const int32_t* xweights, int32_t xksize, const int32_t* ybounds,
                                      const int32_t* yweights, int32_t yksize, int32_t y_first, int32_t y_rows,
                                      uint8_t* scratch, float* out, void* stream) {
  using namespace vb;
  VB_REQUIRE(src && out, "frames_u8_resize: null pointer");
  VB_REQUIRE(T > 0 && src_h > 0 && src_w > 0 && crop_w > 0 && crop_h > 0 && out_h > 0 && out_w > 0,
             "frames_u8_resize: sizes must be positive (T=%d src %dx%d crop %dx%d out %dx%d)", T, src_w, src_h, crop_w,
             crop_h, out_w, out_h);
  VB_REQUIRE(crop_x >= 0 && crop_y >= 0 && (int64_t)crop_x + crop_w <= src_w && (int64_t)crop_y + crop_h <= src_h,
             "frames_u8_resize: crop (%d, %d) + %dx%d is not inside the %dx%d frame", crop_x, crop_y, crop_w, crop_h,
             src_w, src_h);
  VB_REQUIRE(row_stride >= 3LL * src_w && frame_stride >= (int64_t)(src_h - 1) * row_stride + 3LL * src_w,
             "frames_u8_resize: strides (frame %lld, row %lld) do not hold a %dx%d RGB frame", (long long)frame_stride,
             (long long)row_stride, src_w, src_h);
  const bool need_h = crop_w != out_w, need_v = crop_h != out_h;     // Pillow skips a pass whose size is unchanged
  VB_REQUIRE(!need_h || (xbounds && xweights && xksize > 0 && xksize <= kIngestMaxTaps),
             "frames_u8_resize: the horizontal pass needs tables with 0 < ksize <= %d (ksize %d)", kIngestMaxTaps, xksize);
  VB_REQUIRE(!need_v || (ybounds && yweights && yksize > 0 && yksize <= kIngestMaxTaps),
             "frames_u8_resize: the vertical pass needs tables with 0 < ksize <= %d (ksize %d)", kIngestMaxTaps, yksize);
  VB_REQUIRE(y_first >= 0 && y_rows > 0 && (int64_t)y_first + y_rows <= crop_h && (need_v || y_rows == crop_h),
             "frames_u8_resize: rows [%d, %d + %d) are not inside the %d cropped rows", y_first, y_first, y_rows, crop_h);
  VB_REQUIRE(!need_h || scratch, "frames_u8_resize: the horizontal pass needs scratch of T * y_rows * out_w * 3 bytes");
  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t* crop = src + (int64_t)crop_y * row_stride + 3LL * crop_x;
  // the vertical pass's input: the horizontal pass's rows, or the cropped frame itself
  const uint8_t* vin = crop;
  int64_t vfs = frame_stride, vrs = row_stride;
  int row_offset = 0;
  if (need_h) {
    resize_h_kernel<<<ingest_blocks((long long)T * y_rows * out_w), kIngestThreads, 0, st>>>(
        crop + (int64_t)y_first * row_stride, frame_stride, row_stride, xbounds, xweights, xksize, T, y_rows, out_w,
        scratch);
    VB_CHECK_CUDA(cudaGetLastError());
    vin = scratch;
    vrs = 3LL * out_w;
    vfs = (int64_t)y_rows * vrs;
    row_offset = y_first;
  }
  const unsigned blocks = ingest_blocks((long long)T * out_h * out_w);
  if (need_v)
    resize_v_kernel<true><<<blocks, kIngestThreads, 0, st>>>(vin, vfs, vrs, row_offset, ybounds, yweights, yksize, T,
                                                              out_h, out_w, out);
  else
    resize_v_kernel<false><<<blocks, kIngestThreads, 0, st>>>(vin, vfs, vrs, row_offset, nullptr, nullptr, 0, T, out_h,
                                                               out_w, out);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
