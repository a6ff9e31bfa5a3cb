// Stride-1 3x3 convolution + GroupNorm (+ residual) (+ ReLU) in one kernel, and the stride-2 head of ResNetBlock_1..3
// (3x3/2 conv + GroupNorm + ReLU, 1x1/2 projection + GroupNorm).
//
// GroupNorm needs the statistics of a whole image before any of its outputs can be normalised, so the fusion keeps every fp32
// accumulator of an image on chip until its last tile is done and normalises from those values (the raw conv output is never
// rounded to 16 bits and never reaches HBM).  On sm_90a they stay in shared memory: conv_tc_kernel's fused GroupNorm epilogue
// (conv_tcgen05.cu, kFuse == 1) walks work items of whole images x one channel slice, at most 128 KB of accumulators each.
// Reference algebra: vision/resnet_v1.py:129-156 (ResNetBlock), :119-126 (MyGroupNorm).
#include "common.cuh"
#include "serl_b200.h"

// conv_tcgen05.cu
struct serl_fused_conv {
  const void* x; const void* w; void* y; float* out_f32; const void* res;
  const float* gamma; const float* beta; const float* res_stats; const float* res_gamma; const float* res_beta;
  int32_t* error; int N, Hi, Ci, Ho, Co, k, stride, pad, relu, fmt; float eps;
};
int serl_conv_fused_gn(const serl_fused_conv& f, void* stream);

using namespace serl;

extern "C" int serl_conv3x3s2_res_h16(const serl_conv3x3s2_res_desc* d, void* stream) {
  if (!d || !d->x || !d->w || !d->w_proj || !d->y || !d->r || !d->gamma || !d->beta || !d->gamma_proj || !d->beta_proj || !d->error || d->N < 1) {
    set_last_error("serl_conv3x3s2_res_h16: invalid descriptor"); return SERL_ERR_INVALID;
  }
  if (d->Co != 2 * d->Ci) { set_last_error("serl_conv3x3s2_res_h16: Co == 2 Ci only (ResNet-10 stage heads)"); return SERL_ERR_UNSUPPORTED; }
  if (!((d->Wo == 16 && d->Co == 128) || (d->Wo == 8 && d->Co == 256) || (d->Wo == 4 && d->Co == 512))) {
    set_last_error("serl_conv3x3s2_res_h16: unsupported shape (Wo=%d, Ci=%d, Co=%d)", d->Wo, d->Ci, d->Co); return SERL_ERR_UNSUPPORTED;
  }
  // y = relu(GN(conv3x3/2 SAME (x))): XLA SAME on an even size pads 0 low, 1 high
  serl_fused_conv f{d->x, d->w, d->y, nullptr, nullptr, d->gamma, d->beta, nullptr, nullptr, nullptr, d->error,
                    d->N, 2 * d->Wo, d->Ci, d->Wo, d->Co, 3, 2, 0, 1, d->fmt, d->eps};
  if (int e = serl_conv_fused_gn(f, stream)) return e;
  // r = GN(conv1x1/2 (x)) (the block's residual branch, normalised, no ReLU)
  serl_fused_conv p{d->x, d->w_proj, d->r, nullptr, nullptr, d->gamma_proj, d->beta_proj, nullptr, nullptr, nullptr, d->error,
                    d->N, 2 * d->Wo, d->Ci, d->Wo, d->Co, 1, 2, 0, 0, d->fmt, d->eps};
  return serl_conv_fused_gn(p, stream);
}

extern "C" int serl_conv3x3_res_h16(const serl_conv3x3_res_desc* d, void* stream) {
  if (!d || !d->x || !d->w || !d->gamma || !d->beta || !d->error || (!d->y && !d->out_f32) || d->N < 1) {
    set_last_error("serl_conv3x3_res_h16: invalid descriptor"); return SERL_ERR_INVALID;
  }
  if ((d->res_stats != nullptr) != (d->res_gamma != nullptr) || (d->res_stats != nullptr) != (d->res_beta != nullptr) || (d->res_stats && !d->res)) {
    set_last_error("serl_conv3x3_res_h16: res_stats / res_gamma / res_beta go together (and need res)"); return SERL_ERR_INVALID;
  }
  if (d->H != d->W || d->Co != d->Ci) { set_last_error("serl_conv3x3_res_h16: square maps with Ci == Co only"); return SERL_ERR_UNSUPPORTED; }
  if (!((d->W == 32 && d->Ci == 64) || (d->W == 16 && d->Ci == 128) || (d->W == 8 && d->Ci == 256) || (d->W == 4 && d->Ci == 512))) {
    set_last_error("serl_conv3x3_res_h16: unsupported shape (H=W=%d, Ci=%d, Co=%d): ResNet-10 block shapes at 128x128 input only", d->W, d->Ci, d->Co);
    return SERL_ERR_UNSUPPORTED;
  }
  serl_fused_conv f{d->x, d->w, d->out_f32 ? nullptr : d->y, d->out_f32, d->res, d->gamma, d->beta, d->res_stats, d->res_gamma, d->res_beta,
                    d->error, d->N, d->H, d->Ci, d->H, d->Co, 3, 1, 1, d->relu, d->fmt, d->eps};
  return serl_conv_fused_gn(f, stream);
}
