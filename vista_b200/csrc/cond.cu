// The conditioner's sinusoidal scalar embedders (ConcatTimestepEmbedderND, vwm/modules/encoders/modules.py:402-425):
// every such slot of one conditioning tensor (`vector`, or the action columns of `crossattn`) in one launch.
//   out[r, dst_col + j * outdim + k]        = cos(v[r, value_col + j] * f_k)     k < outdim / 2
//   out[r, dst_col + j * outdim + half + k] = sin(v[r, value_col + j] * f_k)
// with f_k = freqs[freq_off + k] computed on the host by timestep_embedding's own expression (util.py:156-160), so the
// only arithmetic here is one fp32 multiply and a full-precision sincosf (arguments reach several hundred radians, far
// outside the range where __sinf / __cosf are accurate).  An odd outdim gets a zero last column (util.py:163-164).
#include <math.h>

#include "../../include/vista_b200.h"
#include "host.cuh"

namespace vb {

__global__ void sinusoid_embed_kernel(const float* __restrict__ values, long long ldv, b200v_sinusoid_table table,
                                      const float* __restrict__ freqs, float* __restrict__ out, long long ldo) {
  const b200v_sinusoid_slot s = table.slot[blockIdx.x];
  const long long r = blockIdx.y;
  const int half = s.outdim >> 1;
  float* o = out + r * ldo + s.dst_col;
  const int work = s.num_features * half;
  for (int i = threadIdx.x; i < work; i += blockDim.x) {
    const int j = i / half, k = i - j * half;
    float c = 0.f, sn = 0.f;
    if (!s.zero) {
      const float a = values[r * ldv + s.value_col + j] * freqs[s.freq_off + k];
      sincosf(a, &sn, &c);
    }
    o[j * s.outdim + k] = c;
    o[j * s.outdim + half + k] = sn;
  }
  if (s.outdim & 1)
    for (int j = threadIdx.x; j < s.num_features; j += blockDim.x) o[j * s.outdim + s.outdim - 1] = 0.f;
}

}  // namespace vb

extern "C" int b200v_sinusoid_embed(const float* values, int64_t ld_values, int32_t rows, const b200v_sinusoid_table* table,
                                    const float* freqs, float* out, int64_t ldo, void* stream) {
  using namespace vb;
  VB_REQUIRE(table && out, "sinusoid_embed: null pointer");
  VB_REQUIRE(rows > 0 && rows <= 65535, "sinusoid_embed: rows=%d out of range", rows);
  VB_REQUIRE(table->n_slots > 0 && table->n_slots <= B200V_SINUSOID_MAX_SLOTS, "sinusoid_embed: n_slots=%d out of range",
             table->n_slots);
  for (int i = 0; i < table->n_slots; ++i) {
    const b200v_sinusoid_slot& s = table->slot[i];
    VB_REQUIRE(s.num_features > 0 && s.outdim > 0 && s.dst_col >= 0 &&
                   s.dst_col + (long long)s.num_features * s.outdim <= ldo,
               "sinusoid_embed: slot %d (num_features %d, outdim %d, dst_col %d) does not fit a row of %lld", i,
               s.num_features, s.outdim, s.dst_col, (long long)ldo);
    VB_REQUIRE(s.zero || (values && freqs && s.value_col >= 0 && s.value_col + s.num_features <= ld_values &&
                          s.freq_off >= 0),
               "sinusoid_embed: slot %d reads outside the value / frequency tables", i);
  }
  dim3 grid(table->n_slots, rows);
  sinusoid_embed_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(values, ld_values, *table, freqs, out, ldo);
  VB_CHECK_CUDA(cudaGetLastError());
  return 0;
}
