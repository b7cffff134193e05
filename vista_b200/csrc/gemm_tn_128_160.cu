// Tap-GEMM instantiations of tile widths 128 and 160.
#include "gemm_tc.cuh"

namespace vb {
template const GemmKern* gemm_variants<128>();
template const GemmKern* gemm_variants<160>();
}  // namespace vb
