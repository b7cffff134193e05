// Tap-GEMM instantiations of tile widths 96 and 192.
#include "gemm_tc.cuh"

namespace vb {
template const GemmKern* gemm_variants<96>();
template const GemmKern* gemm_variants<192>();
}  // namespace vb
