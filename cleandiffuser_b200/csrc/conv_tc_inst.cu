// Explicit instantiations of the tensor-core conv kernel, split over 8 translation units (-DCDS_TC_PART=k selects the
// instantiations) so that the build runs in parallel; the parts take about equally long to compile.  Every entry of
// CDS_TC_VARIANTS (conv_tc.cuh) must appear in exactly one part below.
#define CDS_TC_INSTANTIATE
#include "conv_tc.cuh"

#ifndef CDS_TC_PART
#error "compile with -DCDS_TC_PART=<0..7>"
#endif

namespace cds {
#define CDS_TC_INST(KC_, N_, S_, R_, T_)                                                                                  \
  template cudaError_t conv_tc_launch_t<KC_, N_, R_ != 0, S_, T_ != 0>(const ConvTcLaunch&, const int*, cudaStream_t);  \
  template cudaError_t conv_tc_preload_t<KC_, N_, R_ != 0, S_, T_ != 0>();

#if CDS_TC_PART == 0
CDS_TC_INST(64, 16, 1, 0, 0) CDS_TC_INST(64, 32, 1, 0, 0) CDS_TC_INST(64, 32, 1, 1, 0) CDS_TC_INST(64, 32, 2, 0, 0)
CDS_TC_INST(64, 32, 2, 1, 0) CDS_TC_INST(64, 64, 1, 0, 0) CDS_TC_INST(64, 64, 1, 1, 0) CDS_TC_INST(64, 64, 2, 0, 0)
#elif CDS_TC_PART == 1
CDS_TC_INST(64, 64, 2, 1, 0) CDS_TC_INST(64, 128, 1, 0, 0) CDS_TC_INST(64, 128, 1, 1, 0) CDS_TC_INST(64, 128, 2, 0, 0)
CDS_TC_INST(64, 128, 2, 1, 0) CDS_TC_INST(64, 128, 4, 1, 0) CDS_TC_INST(64, 128, 8, 1, 0) CDS_TC_INST(64, 160, 1, 0, 0)
CDS_TC_INST(64, 192, 1, 0, 0)
#elif CDS_TC_PART == 2
CDS_TC_INST(64, 256, 1, 0, 0) CDS_TC_INST(64, 256, 2, 0, 0) CDS_TC_INST(64, 256, 4, 0, 0)
#elif CDS_TC_PART == 3
CDS_TC_INST(32, 16, 1, 0, 0) CDS_TC_INST(32, 32, 1, 0, 0) CDS_TC_INST(32, 32, 1, 1, 0) CDS_TC_INST(32, 32, 2, 0, 0)
CDS_TC_INST(32, 32, 2, 1, 0) CDS_TC_INST(32, 64, 1, 0, 0) CDS_TC_INST(32, 64, 1, 1, 0) CDS_TC_INST(32, 64, 2, 0, 0)
CDS_TC_INST(32, 64, 2, 1, 0) CDS_TC_INST(32, 128, 1, 0, 0)
#elif CDS_TC_PART == 4
CDS_TC_INST(32, 128, 1, 1, 0) CDS_TC_INST(32, 128, 2, 0, 0) CDS_TC_INST(32, 128, 2, 1, 0) CDS_TC_INST(32, 256, 1, 0, 0)
CDS_TC_INST(64, 16, 1, 0, 1) CDS_TC_INST(64, 32, 1, 0, 1) CDS_TC_INST(64, 32, 1, 1, 1) CDS_TC_INST(64, 64, 1, 0, 1)
CDS_TC_INST(64, 64, 1, 1, 1)
#elif CDS_TC_PART == 5
CDS_TC_INST(64, 64, 2, 0, 1) CDS_TC_INST(64, 64, 2, 1, 1) CDS_TC_INST(64, 128, 1, 0, 1) CDS_TC_INST(64, 128, 1, 1, 1)
CDS_TC_INST(64, 128, 2, 0, 1) CDS_TC_INST(64, 128, 2, 1, 1) CDS_TC_INST(64, 128, 4, 1, 1) CDS_TC_INST(64, 128, 8, 1, 1)
CDS_TC_INST(64, 160, 1, 0, 1) CDS_TC_INST(64, 192, 1, 0, 1)
#elif CDS_TC_PART == 6
CDS_TC_INST(64, 256, 1, 0, 1) CDS_TC_INST(64, 256, 2, 0, 1) CDS_TC_INST(64, 256, 4, 0, 1) CDS_TC_INST(32, 16, 1, 0, 1)
CDS_TC_INST(32, 32, 1, 0, 1)
#elif CDS_TC_PART == 7
CDS_TC_INST(32, 32, 1, 1, 1) CDS_TC_INST(32, 64, 1, 0, 1) CDS_TC_INST(32, 64, 1, 1, 1) CDS_TC_INST(32, 64, 2, 0, 1)
CDS_TC_INST(32, 64, 2, 1, 1) CDS_TC_INST(32, 128, 1, 0, 1) CDS_TC_INST(32, 128, 1, 1, 1) CDS_TC_INST(32, 128, 2, 0, 1)
CDS_TC_INST(32, 128, 2, 1, 1) CDS_TC_INST(32, 256, 1, 0, 1)
#else
#error "CDS_TC_PART out of range"
#endif
}  // namespace cds
