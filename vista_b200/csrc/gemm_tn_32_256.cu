// Tap-GEMM instantiations of tile widths 32 and 256.
#include "gemm_tc.cuh"

namespace vb {
template const GemmKern* gemm_variants<32>();
template const GemmKern* gemm_variants<256>();
}  // namespace vb
