// Explicit instantiations of the tensor-core conv kernel, split over 8 x 2 translation units (-DCDS_TC_PART=k selects the
// shapes, -DCDS_TC_TF32=0|1 the operand type) so that the build runs in parallel.  Every entry of CDS_TC_VARIANTS
// (conv_tc.cuh) must appear in exactly one part below.
#define CDS_TC_INSTANTIATE
#include "conv_tc.cuh"

#ifndef CDS_TC_PART
#error "compile with -DCDS_TC_PART=<0..7>"
#endif
#ifndef CDS_TC_TF32
#error "compile with -DCDS_TC_TF32=<0|1>"
#endif

namespace cds {
#define CDS_TC_INST(KC_, N_, S_)                                                                                \
  template cudaError_t conv_tc_launch_t<KC_, N_, false, S_, (CDS_TC_TF32 != 0)>(const ConvTcLaunch&, const int*, cudaStream_t);  \
  template cudaError_t conv_tc_launch_t<KC_, N_, true, S_, (CDS_TC_TF32 != 0)>(const ConvTcLaunch&, const int*, cudaStream_t);   \
  template cudaError_t conv_tc_preload_t<KC_, N_, false, S_, (CDS_TC_TF32 != 0)>();                                              \
  template cudaError_t conv_tc_preload_t<KC_, N_, true, S_, (CDS_TC_TF32 != 0)>();

#if CDS_TC_PART == 0
CDS_TC_INST(64, 16, 1) CDS_TC_INST(32, 16, 1) CDS_TC_INST(64, 256, 2) CDS_TC_INST(64, 128, 8)
#elif CDS_TC_PART == 1
CDS_TC_INST(64, 32, 1) CDS_TC_INST(32, 32, 1) CDS_TC_INST(64, 256, 4) CDS_TC_INST(64, 128, 4)
#elif CDS_TC_PART == 2
CDS_TC_INST(64, 64, 1) CDS_TC_INST(32, 64, 1) CDS_TC_INST(64, 160, 1)
#elif CDS_TC_PART == 3
CDS_TC_INST(64, 128, 1) CDS_TC_INST(32, 128, 1) CDS_TC_INST(64, 192, 1)
#elif CDS_TC_PART == 4
CDS_TC_INST(64, 256, 1) CDS_TC_INST(32, 32, 2)
#elif CDS_TC_PART == 5
CDS_TC_INST(64, 32, 2) CDS_TC_INST(32, 256, 1)
#elif CDS_TC_PART == 6
CDS_TC_INST(64, 64, 2) CDS_TC_INST(32, 64, 2)
#elif CDS_TC_PART == 7
CDS_TC_INST(64, 128, 2) CDS_TC_INST(32, 128, 2)
#else
#error "CDS_TC_PART out of range"
#endif
}  // namespace cds
