// Internal parameter blocks of the training-path (backward) kernels; see include/vmambair_b200.h for the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vmambair_b200.h"
#include "oss_params.h"

namespace vmb {
struct LnFwdParams {
    const void* x; const float* w; const float* b; void* y; float* stats;
    int B, C, L, mode;
    int64_t x_bs, x_cs, y_bs, y_cs;
};
struct LnBwdParams {
    const void* x; const void* g; const void* add; const float* w; void* dx; float* dw; float* db; float* stats;
    int B, C, L, mode;
    int64_t x_bs, x_cs, g_bs, g_cs, a_bs, a_cs, dx_bs, dx_cs;
};
struct MergeBwdParams {
    const float* merged; const float* stats; const void* z; const void* dy2; const float* dpooled;
    const float* w; const float* b; void* dm; void* dz; float* dw; float* db;
    int B, C, L;
    int64_t z_bs, z_cs, dz_bs, dz_cs;
};
struct DwBwdParams {
    const void* x; const float* w; const float* bias; const void* g; void* dv; float* dwgt; float* dbias;
    int B, Cout, H, W, mode;
    int64_t x_bs, x_cs, g_bs, g_cs, dv_bs, dv_cs;
    bool vec_ok;  // W % 8 == 0, 16 B aligned rows: 8-pixel strips
};
struct GateBwdParams {
    const void* dyg; const void* y2; const float* gate; void* dy2; float* dgate;
    int B, C, L, mode;
};
struct AdamParams {
    float* param; float* grad; float* m; float* v; float* ema; float* state;
    long n;
    float lr, beta1, beta2, eps, weight_decay;
    int decoupled;
    float grad_scale, max_norm, ema_decay;
    int zero_grad;
    const float* lr_dev;  // nullptr: lr
};
struct PrepJob {
    const float* src; const float* src2; void* dst; void* dst2;
    int type, M, K, N2, ld, ld2;
};
struct PrepParams {
    PrepJob jobs[VMB_PREP_MAX_JOBS];
    int njobs;
};
int prep_weights_launch(const PrepParams& p, int dtype, cudaStream_t stream);
struct WgradParams {
    const void* dy; const void* x; float* out;
    int B, M, K, L;
    int64_t dy_bs, dy_cs, x_bs, x_cs;
    int splits, per_batch;
    float* dbias;  // optional: dbias[m] += sum_{b,p} dy[b][m][p]
};
int wgrad_launch(const WgradParams& p, int dtype, cudaStream_t stream);
struct ChannelBwdParams {
    ChannelParams fwd;
    const float* dc_out; float* d_pooled;
    float *d_cin_w, *d_cin_b, *d_xc_proj, *d_dtc_w, *d_dtc_b, *d_Ac_logs, *d_Dsc, *d_cout_w, *d_cout_b, *d_cn_w, *d_cn_b;
    float* scratch_dB;
};
int channel_bwd_launch(const ChannelBwdParams& q, cudaStream_t stream);
int fused_adam_launch(const AdamParams& p, cudaStream_t stream);
int ln_fwd_launch(const LnFwdParams& p, int dtype, cudaStream_t stream);
int ln_bwd_launch(const LnBwdParams& p, int dtype, cudaStream_t stream);
int merge_bwd_launch(const MergeBwdParams& p, int dtype, cudaStream_t stream);
int dwconv_bwd_launch(const DwBwdParams& p, int dtype, cudaStream_t stream);
int dwconv_wgrad_launch(const DwBwdParams& p, int dtype, cudaStream_t stream);
int gate_bwd_launch(const GateBwdParams& p, int dtype, cudaStream_t stream);
}  // namespace vmb
