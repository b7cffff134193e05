// Tap-GEMM instantiations of tile widths 64 and 224.
#include "gemm_tc.cuh"

namespace vb {
template const GemmKern* gemm_variants<64>();
template const GemmKern* gemm_variants<224>();
}  // namespace vb
