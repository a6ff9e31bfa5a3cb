// Stride-1 3x3 SAME convolution entry point (serl_conv3x3s1_tc_h16).  The shifted-window kernel of the sm_100 build addressed the
// nine taps as row-shifted MMA descriptors over one staged input patch; a shift that is not a multiple of eight rows moves the
// operand off the 128-byte swizzle atom, which tcgen05 descriptors absorb through their base-offset field.  On sm_90a the
// convolution runs on the implicit-GEMM wgmma kernel of conv_tcgen05.cu, which produces the same output and GroupNorm sums.
#include "common.cuh"
#include "serl_b200.h"

using namespace serl;

extern "C" int serl_conv3x3s1_tc_h16(const serl_conv_tc_desc* d, int base_offset_mode, void* stream) {
  (void)base_offset_mode;
  if (!d || !d->x || !d->w || !d->y || !d->stats || !d->error) { set_last_error("serl_conv3x3s1_tc_h16: invalid descriptor"); return SERL_ERR_INVALID; }
  if (d->kh != 3 || d->kw != 3 || d->stride != 1 || d->pad_lo != 1 || d->Ho != d->Hi || d->Wo != d->Wi || d->Ci % 64 || d->Co % 64 || d->Wi > 32 || d->in_a) {
    set_last_error("serl_conv3x3s1_tc_h16: needs a 3x3 stride-1 SAME conv, Ci,Co %% 64 == 0, W <= 32, no operand transform"); return SERL_ERR_UNSUPPORTED;
  }
  return serl_conv2d_tc_h16(d, stream);
}
