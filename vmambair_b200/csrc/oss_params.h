// Internal parameter blocks of the fused OSS-block stages (see include/vmambair_b200.h for the C ABI).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vmb {
struct PixlinParams {
    const void* x; const void* w; const float* bias; const void* residual; void* out;
    const float* ln_w; const float* ln_b; const float* gate;
    int ln_mode, gate_mode, act_from, act_to, B, K, M, P;
    int64_t x_bs, x_cs, r_bs, r_cs, o_bs, o_cs, g_bs, w_ld;
    bool vec_ok, w_vec, w_all;
    int w_tiles;  // weight-tile buffers in smem (2 = double buffer, or every tile of the CTA when w_all)
};
struct DwParams {
    const void* x; const float* w; const float* bias; void* out;
    int B, Cout, H, W, mode;
    int64_t x_bs, x_cs, o_bs, o_cs;
    bool vec_ok;  // W % 8 == 0 and 16 B aligned rows: 8-pixel strips
    void* out_t;  // optional second output: every (H, W) plane transposed to (W, H), dense (B, Cout, W*H) -- the copy of x the
                  // column-major scan directions read (mode 0 only)
};
struct CrossScanParams {
    const void* src[4]; void* out;
    int B, rows, H, W;
    int64_t src_bs, src_rs, out_bs, out_ks;
};
struct CrossScanMulti {
    int nseg;
    int row_end[4];  // cumulative row counts of the segments
    CrossScanParams seg[4];
};
struct MergeParams {
    const void* ys; const void* z; const float* ln_w; const float* ln_b; void* y2; float* pooled;
    int B, C, H, W;
    int64_t z_bs, z_cs;
    int in_place_order;
    void* ws;  // fp32 scratch: B*C*L merged values + 2*B*L per-pixel statistics
    int z_preact;
    int save_ws;  // keep the merged values / statistics in ws for the backward (the two-kernel path always does)
};
struct TransposeParams {
    const void* x; void* out;
    int planes, H, W;
};
struct PixelShuffleParams {
    const void* x; void* out;
    int B, H, W, C;  // C = output channels; the input has 4C
    const float* bias;  // optional fp32 (4C): added to the input channels (the bias of the conv in front)
};
struct ChannelParams {
    const float* pooled; float inv_count;
    const float* cin_w; const float* cin_b; const float* xc_proj; const float* dtc_w; const float* dtc_b;
    const float* Ac_logs; const float* Dsc; const float* cout_w; const float* cout_b; const float* cn_w; const float* cn_b;
    float* c_out;
    int B, C, dc, Rc, N;
};
struct Conv3Params {
    const void* x; const void* w; const float* bias; void* out; const void* add;
    int B, Cin, Cout, H, W;
    int in_nhwc, mode, add_scale;
    int Mpad, Kpad;  // packed weights: [9 taps][Mpad][Kpad], Mpad % 64 == 0, Kpad % 16 == 0, zero padded
    int64_t x_bs, x_cs, o_bs, o_cs, add_bs, add_cs;
};
int conv3x3_launch(const Conv3Params& p, int dtype, cudaStream_t stream);
int pixlin_launch(const PixlinParams& p, int dtype, int out_dtype, cudaStream_t stream);
int dwconv_launch(const DwParams& p, int dtype, cudaStream_t stream);
int cross_scan_launch(const CrossScanParams& p, int dtype, cudaStream_t stream);
int cross_scan_multi_launch(const CrossScanMulti& m, int dtype, cudaStream_t stream);
int merge_launch(const MergeParams& p, int dtype, cudaStream_t stream);
int merge_sum_launch(const MergeParams& p, float* out, int dtype, cudaStream_t stream);
int transpose_launch(const TransposeParams& p, int dtype, cudaStream_t stream);
int pixel_shuffle_launch(const PixelShuffleParams& p, int dtype, cudaStream_t stream);
int channel_launch(const ChannelParams& p, cudaStream_t stream);
}  // namespace vmb

