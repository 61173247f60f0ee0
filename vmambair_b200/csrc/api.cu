#include <stdlib.h>
// C-ABI entry points (include/vmambair_b200.h): argument validation + launch.
#include <stdarg.h>
#include <stdio.h>

#include "common.cuh"
#include "scan_params.h"
#include "oss_params.h"

namespace vmb {
int num_sms() {
    static const int n = [] {
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || v <= 0)
            v = 132;  // H100 SXM
        return v;
    }();
    return n;
}
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
static inline int elt_size(int dtype) { return dtype == VMB_F32 ? 4 : 2; }
static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
}  // namespace vmb

using namespace vmb;

extern "C" const char* vmb_last_error(void) { return g_err; }
extern "C" const char* vmb_version(void) { return "vmambair_b200 0.1 sm_90a"; }
extern "C" int vmb_scan_ckpt_interval(void) { return kScanCkpt; }

extern "C" int vmb_selective_scan_fwd(const vmb_scan_fwd_args* a, void* stream) {
    VMB_CHECK(a != nullptr, "selective_scan_fwd: null args");
    VMB_CHECK(a->dtype == VMB_F32 || a->dtype == VMB_BF16 || a->dtype == VMB_F16,
              "selective_scan_fwd: dtype must be f32/bf16/f16 (got %d)", a->dtype);
    VMB_CHECK(a->u && a->delta && a->A && a->Bm && a->Cm && a->out, "selective_scan_fwd: null tensor pointer");
    VMB_CHECK(a->batch > 0 && a->dim > 0 && a->seqlen > 0 && a->dstate > 0 && a->ngroups > 0,
              "selective_scan_fwd: non-positive size");
    VMB_CHECK(a->dim % a->ngroups == 0, "selective_scan_fwd: dims should be dividable by n_groups");
    VMB_CHECK(a->dstate <= 256, "selective_scan only supports state dimension <= 256");
    VMB_CHECK(a->batch <= 65535, "selective_scan_fwd: batch > 65535");
    VMB_CHECK(a->out_f32 == 0 || a->out_f32 == 1, "selective_scan_fwd: out_f32 must be 0 or 1 (got %d)", a->out_f32);
    VMB_CHECK(!a->out_f32 || a->dtype == VMB_BF16 || a->dtype == VMB_F16, "selective_scan_fwd: out_f32 needs bf16 / fp16 inputs");
    VMB_CHECK((a->z == nullptr) == (a->out_z == nullptr), "selective_scan_fwd: z and out_z must both be given or both be NULL");
    VMB_CHECK(!a->z || !a->out_f32, "selective_scan_fwd: the z gate has no fp32-output form (out_f32)");
    VMB_CHECK(a->ckpt_pairs == 0 || a->ckpt_pairs == 1, "selective_scan_fwd: ckpt_pairs must be 0 or 1 (got %d)", a->ckpt_pairs);
    VMB_CHECK(!a->z || !a->ckpt || a->ckpt_pairs, "selective_scan_fwd: with z, checkpoints are written in the pair layout (ckpt_pairs = 1)");
    VMB_CHECK(!a->ckpt || !a->ckpt_pairs || aligned16(a->ckpt), "selective_scan_fwd: pair-layout checkpoints must be 16-byte aligned");
    ScanFwdParams p{};
    p.u = a->u; p.delta = a->delta; p.Bm = a->Bm; p.Cm = a->Cm; p.A = a->A; p.D = a->D; p.bias = a->delta_bias;
    p.out = a->out; p.ckpt = a->ckpt;
    p.batch = a->batch; p.dim = a->dim; p.L = a->seqlen; p.N = a->dstate; p.G = a->ngroups;
    p.npad = (a->dstate + 15) / 16 * 16;
    p.rows_per_group = a->dim / a->ngroups;
    p.n_ckpt = (a->seqlen + kScanCkpt - 1) / kScanCkpt;
    p.u_bs = a->u_bs; p.u_ds = a->u_ds; p.dl_bs = a->delta_bs; p.dl_ds = a->delta_ds; p.o_bs = a->out_bs; p.o_ds = a->out_ds;
    p.B_bs = a->B_bs; p.B_gs = a->B_gs; p.B_ns = a->B_ns; p.C_bs = a->C_bs; p.C_gs = a->C_gs; p.C_ns = a->C_ns;
    p.softplus = a->delta_softplus;
    const int v = 16 / elt_size(a->dtype), vo = a->out_f32 ? 4 : v;  // 16 B rows of `out` in its own element type
    auto mult = [v](int64_t s) { return s % v == 0; };
    auto mult_o = [vo](int64_t s) { return s % vo == 0; };
    p.vec_ok = aligned16(a->u) && aligned16(a->delta) && aligned16(a->Bm) && aligned16(a->Cm) && aligned16(a->out) &&
               mult(a->u_bs) && mult(a->u_ds) && mult(a->delta_bs) && mult(a->delta_ds) && mult_o(a->out_bs) &&
               mult_o(a->out_ds) && mult(a->B_bs) && mult(a->B_gs) && mult(a->B_ns) && mult(a->C_bs) && mult(a->C_gs) &&
               mult(a->C_ns);
    int ext = 0;
    if (a->z) {
        set_scan_gate(p, ScanGateDesc{a->z, a->out_z, a->z_bs, a->z_ds, a->out_z_bs, a->out_z_ds});
        p.vec_ok = p.vec_ok && aligned16(a->z) && aligned16(a->out_z) && mult(a->z_bs) && mult(a->z_ds) && mult(a->out_z_bs) &&
                   mult(a->out_z_ds);
        ext |= kScanGate;
    }
    if (a->ckpt && a->ckpt_pairs) ext |= kScanPairCkpt;
    return scan_fwd_launch(p, a->dtype, static_cast<cudaStream_t>(stream), a->out_f32 != 0, ext);
}

extern "C" int vmb_scan_gate_bwd(const vmb_scan_gate_args* a, void* stream) {
    VMB_CHECK(a != nullptr, "scan_gate_bwd: null args");
    VMB_CHECK(a->dtype == VMB_F32 || a->dtype == VMB_BF16 || a->dtype == VMB_F16, "scan_gate_bwd: dtype must be f32/bf16/f16 (got %d)",
              a->dtype);
    VMB_CHECK(a->dout && a->out && a->z && a->dout_eff && a->dz, "scan_gate_bwd: null tensor pointer");
    VMB_CHECK(a->batch > 0 && a->dim > 0 && a->seqlen > 0 && (int64_t)a->batch * a->dim < (1LL << 31), "scan_gate_bwd: bad sizes");
    const int v = 16 / elt_size(a->dtype);
    auto mult = [v](int64_t s) { return s % v == 0; };
    const bool vec_ok = aligned16(a->dout) && aligned16(a->out) && aligned16(a->z) && aligned16(a->dz) && aligned16(a->dout_eff) &&
                        (!a->out_z || (aligned16(a->out_z) && mult(a->out_z_bs) && mult(a->out_z_ds))) && mult(a->dout_bs) &&
                        mult(a->dout_ds) && mult(a->out_bs) && mult(a->out_ds) && mult(a->z_bs) && mult(a->z_ds) && mult(a->dz_bs) &&
                        mult(a->dz_ds) && a->seqlen % 4 == 0;  // dout_eff: dense fp32 rows
    return scan_gate_bwd_launch(*a, vec_ok, static_cast<cudaStream_t>(stream));
}

extern "C" int64_t vmb_scan_bwd_workspace_bytes(int batch, int ngroups, int dstate, int seqlen) {
    const int64_t npad = (dstate + 15) / 16 * 16;
    return 16 * (int64_t)batch * ngroups * (npad / 2) * seqlen;
}

// checks + parameter block of vmb_selective_scan_bwd, shared with the workspace query (which needs no workspace: the call requires
// it 16 B aligned, so it never changes the launch configuration)
static int scan_bwd_params(const vmb_scan_bwd_args* a, ScanBwdParams& p) {
    VMB_CHECK(a != nullptr, "selective_scan_bwd: null args");
    VMB_CHECK(a->dtype == VMB_F32 || a->dtype == VMB_BF16 || a->dtype == VMB_F16,
              "selective_scan_bwd: dtype must be f32/bf16/f16 (got %d)", a->dtype);
    VMB_CHECK(a->u && a->delta && a->A && a->Bm && a->Cm && a->dout && a->du && a->ddelta && a->dA && a->dB && a->dC,
              "selective_scan_bwd: null tensor pointer");
    VMB_CHECK(a->batch > 0 && a->dim > 0 && a->seqlen > 0 && a->dstate > 0 && a->ngroups > 0,
              "selective_scan_bwd: non-positive size");
    VMB_CHECK(a->dim % a->ngroups == 0, "selective_scan_bwd: dims should be dividable by n_groups");
    VMB_CHECK(a->dstate <= 256, "selective_scan only supports state dimension <= 256");
    VMB_CHECK(a->batch <= 65535, "selective_scan_bwd: batch > 65535");
    VMB_CHECK(a->ckpt != nullptr || a->seqlen <= kScanCkpt,
              "selective_scan_bwd: forward checkpoints required when seqlen > %d", kScanCkpt);
    VMB_CHECK((a->D == nullptr) == (a->dD == nullptr), "selective_scan_bwd: D and dD must both be given or both be NULL");
    VMB_CHECK((a->delta_bias == nullptr) == (a->ddelta_bias == nullptr),
              "selective_scan_bwd: delta_bias and ddelta_bias must both be given or both be NULL");
    VMB_CHECK(a->dout_f32 == 0 || a->dout_f32 == 1, "selective_scan_bwd: dout_f32 must be 0 or 1 (got %d)", a->dout_f32);
    VMB_CHECK(!a->dout_f32 || a->dtype == VMB_BF16 || a->dtype == VMB_F16, "selective_scan_bwd: dout_f32 needs bf16 / fp16 inputs");
    VMB_CHECK(a->deterministic == 0 || a->deterministic == 1, "selective_scan_bwd: deterministic must be 0 or 1 (got %d)", a->deterministic);
    p = ScanBwdParams{};
    p.u = a->u; p.delta = a->delta; p.Bm = a->Bm; p.Cm = a->Cm; p.dout = a->dout; p.A = a->A; p.D = a->D;
    p.bias = a->delta_bias; p.ckpt = a->ckpt; p.du = a->du; p.ddelta = a->ddelta; p.dA = a->dA; p.dB = a->dB; p.dC = a->dC;
    p.dD = a->dD; p.dbias = a->ddelta_bias;
    p.batch = a->batch; p.dim = a->dim; p.L = a->seqlen; p.N = a->dstate; p.G = a->ngroups;
    p.npad = (a->dstate + 15) / 16 * 16;
    p.rows_per_group = a->dim / a->ngroups;
    p.n_ckpt = (a->seqlen + kScanCkpt - 1) / kScanCkpt;
    p.u_bs = a->u_bs; p.u_ds = a->u_ds; p.dl_bs = a->delta_bs; p.dl_ds = a->delta_ds; p.do_bs = a->dout_bs; p.do_ds = a->dout_ds;
    p.du_bs = a->du_bs; p.du_ds = a->du_ds; p.dd_bs = a->ddelta_bs; p.dd_ds = a->ddelta_ds;
    p.B_bs = a->B_bs; p.B_gs = a->B_gs; p.B_ns = a->B_ns; p.C_bs = a->C_bs; p.C_gs = a->C_gs; p.C_ns = a->C_ns;
    p.softplus = a->delta_softplus;
    const int v = 16 / elt_size(a->dtype), vg = a->dout_f32 ? 4 : v;  // 16 B rows of dout in its own element type
    auto mult = [v](int64_t s) { return s % v == 0; };
    auto mult_g = [vg](int64_t s) { return s % vg == 0; };
    p.vec_ok = aligned16(a->u) && aligned16(a->delta) && aligned16(a->Bm) && aligned16(a->Cm) && aligned16(a->dout) &&
               aligned16(a->du) && aligned16(a->ddelta) && mult(a->u_bs) && mult(a->u_ds) && mult(a->delta_bs) &&
               mult(a->delta_ds) && mult_g(a->dout_bs) && mult_g(a->dout_ds) && mult(a->du_bs) && mult(a->du_ds) &&
               mult(a->ddelta_bs) && mult(a->ddelta_ds) && mult(a->B_bs) && mult(a->B_gs) && mult(a->B_ns) &&
               mult(a->C_bs) && mult(a->C_gs) && mult(a->C_ns);
    return VMB_OK;
}

extern "C" int vmb_selective_scan_bwd(const vmb_scan_bwd_args* a, void* stream) {
    ScanBwdParams p;
    int rc = scan_bwd_params(a, p);
    if (rc != VMB_OK) return rc;
    VMB_CHECK(a->workspace != nullptr, "selective_scan_bwd: null tensor pointer");
    VMB_CHECK(aligned16(a->workspace), "selective_scan_bwd: workspace must be 16-byte aligned");
    p.dBC = static_cast<float*>(a->workspace);
    return scan_bwd_launch(p, a->dtype, static_cast<cudaStream_t>(stream), a->dout_f32 != 0, a->deterministic != 0);
}

extern "C" int64_t vmb_scan_bwd_det_workspace_bytes(const vmb_scan_bwd_args* a) {
    ScanBwdParams p;
    if (scan_bwd_params(a, p) != VMB_OK) return -1;
    return scan_bwd_det_workspace(p);
}

static inline bool dt_ok(int d) { return d == VMB_F32 || d == VMB_BF16 || d == VMB_F16; }

extern "C" int vmb_pixlin(const vmb_pixlin_args* a, void* stream) {
    VMB_CHECK(a && a->x && a->w && a->out, "pixlin: null pointer");
    VMB_CHECK(dt_ok(a->dtype) && (a->out_dtype == a->dtype || a->out_dtype == VMB_F32), "pixlin: bad dtype");
    VMB_CHECK(a->batch > 0 && a->batch <= 65535 && a->K > 0 && a->M > 0 && a->P > 0, "pixlin: bad sizes");
    VMB_CHECK(a->ln_mode == 0 || a->ln_w, "pixlin: ln_w missing");
    VMB_CHECK(a->ln_mode != 1 || a->ln_b, "pixlin: ln_b missing");
    VMB_CHECK(a->gate_mode == 0 || a->gate, "pixlin: gate missing");
    PixlinParams p{a->x, a->w, a->bias, a->residual, a->out, a->ln_w, a->ln_b, a->gate, a->ln_mode, a->gate_mode,
                   a->act_from, a->act_to, a->batch, a->K, a->M, a->P, a->x_bs, a->x_cs, a->r_bs, a->r_cs, a->o_bs, a->o_cs,
                   a->g_bs, a->w_ld > 0 ? a->w_ld : a->K, false, false, false, 2};
    {
        const int vw = 16 / elt_size(a->dtype);
        const int64_t kpad = (a->K + 15) / 16 * 16;
        p.w_vec = aligned16(a->w) && p.w_ld % vw == 0 && p.w_ld >= kpad;
    }
    const int v = 16 / elt_size(a->dtype), vo = 16 / elt_size(a->out_dtype);
    const int vm = v > vo ? v : vo;
    auto mult = [vm](int64_t s) { return s % vm == 0; };
    p.vec_ok = aligned16(a->x) && aligned16(a->out) && (!a->residual || aligned16(a->residual)) && mult(a->x_bs) &&
               mult(a->x_cs) && mult(a->o_bs) && mult(a->o_cs) && (!a->residual || (mult(a->r_bs) && mult(a->r_cs))) &&
               a->P % vm == 0;
    return pixlin_launch(p, a->dtype, a->out_dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_dwconv3x3(const vmb_dwconv_args* a, void* stream) {
    VMB_CHECK(a && a->x && a->w && a->out, "dwconv: null pointer");
    VMB_CHECK(dt_ok(a->dtype), "dwconv: bad dtype");
    VMB_CHECK(a->batch > 0 && a->c_out > 0 && a->H > 0 && a->W > 0 && (long)a->batch * a->c_out <= 65535, "dwconv: bad sizes");
    DwParams p{a->x, a->w, a->bias, a->out, a->batch, a->c_out, a->H, a->W, a->mode, a->x_bs, a->x_cs, a->o_bs, a->o_cs, false, nullptr};
    p.vec_ok = a->W % 8 == 0 && aligned16(a->x) && aligned16(a->out) && a->x_bs % 8 == 0 && a->x_cs % 8 == 0 &&
               a->o_bs % 8 == 0 && a->o_cs % 8 == 0;
    return dwconv_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_dwconv3x3_t(const vmb_dwconv_args* a, void* out_t, void* stream) {
    VMB_CHECK(a && a->x && a->w && a->out && out_t, "dwconv_t: null pointer");
    VMB_CHECK(dt_ok(a->dtype), "dwconv_t: bad dtype");
    VMB_CHECK(a->mode == 0, "dwconv_t: the transposed second output exists for mode 0 (SiLU) only");
    VMB_CHECK(a->batch > 0 && a->c_out > 0 && a->H > 0 && a->W > 0 && (long)a->batch * a->c_out <= 65535, "dwconv_t: bad sizes");
    DwParams p{a->x, a->w, a->bias, a->out, a->batch, a->c_out, a->H, a->W, a->mode, a->x_bs, a->x_cs, a->o_bs, a->o_cs, false, out_t};
    p.vec_ok = a->W % 8 == 0 && aligned16(a->x) && aligned16(a->out) && a->x_bs % 8 == 0 && a->x_cs % 8 == 0 &&
               a->o_bs % 8 == 0 && a->o_cs % 8 == 0;
    // 8 B / 16 B runs of four consecutive h in the (W, H) plane: H % 4 == 0 holds on the row-block path; the base must be aligned
    if (!aligned16(out_t) || a->H % 4 != 0) p.vec_ok = false;
    return dwconv_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_cross_scan(const vmb_cross_scan_args* a, void* stream) {
    VMB_CHECK(a && a->src[0] && a->src[1] && a->src[2] && a->src[3] && a->out, "cross_scan: null pointer");
    VMB_CHECK(dt_ok(a->dtype), "cross_scan: bad dtype");
    CrossScanParams p{{a->src[0], a->src[1], a->src[2], a->src[3]}, a->out, a->batch, a->rows, a->H, a->W, a->src_bs,
                      a->src_rs, a->out_bs, a->out_ks > 0 ? a->out_ks : (int64_t)a->rows * a->H * a->W};
    return cross_scan_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_cross_scan_multi(const vmb_cross_scan_args* segs, int nseg, void* stream) {
    VMB_CHECK(segs && nseg >= 1 && nseg <= 4, "cross_scan_multi: 1..4 segments");
    CrossScanMulti m{};
    m.nseg = nseg;
    int rows = 0;
    for (int i = 0; i < nseg; ++i) {
        const vmb_cross_scan_args* a = segs + i;
        VMB_CHECK(a->src[0] && a->src[1] && a->src[2] && a->src[3] && a->out, "cross_scan_multi: null pointer (segment %d)", i);
        VMB_CHECK(a->dtype == segs[0].dtype && a->batch == segs[0].batch && a->H == segs[0].H && a->W == segs[0].W,
                  "cross_scan_multi: the segments must share dtype, batch, H and W");
        VMB_CHECK(a->rows > 0, "cross_scan_multi: empty segment %d", i);
        m.seg[i] = CrossScanParams{{a->src[0], a->src[1], a->src[2], a->src[3]}, a->out, a->batch, a->rows, a->H, a->W, a->src_bs,
                                   a->src_rs, a->out_bs, a->out_ks > 0 ? a->out_ks : (int64_t)a->rows * a->H * a->W};
        rows += a->rows;
        m.row_end[i] = rows;
    }
    VMB_CHECK(dt_ok(segs[0].dtype), "cross_scan_multi: bad dtype");
    return cross_scan_multi_launch(m, segs[0].dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int64_t vmb_merge_workspace_bytes(int batch, int C, int H, int W) {
    // fp32 merged values + per-pixel (sum, sum of squares) + per-tile channel sums + per-image tile counters of the single-kernel path
    const int64_t tiles = (int64_t)((H + 15) / 16) * ((W + 15) / 16);
    return 4 * ((int64_t)batch * C * H * W + 2 * (int64_t)batch * H * W + (int64_t)batch * tiles * C + batch) + 16;
}

extern "C" int vmb_merge_norm_gate(const vmb_merge_args* a, void* stream) {
    VMB_CHECK(a && a->ys && a->z && a->ln_w && a->ln_b && a->y2 && a->pooled, "merge: null pointer");
    VMB_CHECK(dt_ok(a->dtype), "merge: bad dtype");
    VMB_CHECK(a->batch > 0 && a->batch <= 65535, "merge: bad batch");
    MergeParams p{a->ys, a->z, a->ln_w, a->ln_b, a->y2, a->pooled, a->batch, a->C, a->H, a->W, a->z_bs, a->z_cs, a->in_place_order, a->workspace, a->z_preact, a->save_ws};
    VMB_CHECK(a->workspace && aligned16(a->workspace), "merge: 16 B-aligned workspace of vmb_merge_workspace_bytes() required");
    return merge_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_merge_sum(const vmb_merge_args* a, float* out, void* stream) {
    VMB_CHECK(a && a->ys && out, "merge_sum: null pointer");
    VMB_CHECK(dt_ok(a->dtype), "merge_sum: bad dtype");
    VMB_CHECK(a->batch > 0 && a->batch <= 65535 && a->C > 0 && a->H > 0 && a->W > 0, "merge_sum: bad sizes");
    VMB_CHECK(a->workspace && aligned16(a->workspace), "merge_sum: 16 B-aligned workspace of vmb_merge_workspace_bytes() required");
    MergeParams p{a->ys, nullptr, nullptr, nullptr, nullptr, nullptr, a->batch, a->C, a->H, a->W, 0, 0, a->in_place_order, a->workspace, 0, 0};
    return merge_sum_launch(p, out, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_channel_branch(const vmb_channel_args* a, void* stream) {
    VMB_CHECK(a && a->pooled && a->xc_proj && a->dtc_w && a->dtc_b && a->Ac_logs && a->Dsc && a->cn_w && a->cn_b && a->c_out,
              "channel_branch: null pointer");
    VMB_CHECK((a->cin_w == nullptr) == (a->cin_b == nullptr) && (a->cout_w == nullptr) == (a->cout_b == nullptr),
              "channel_branch: conv_cin / conv_cout weight and bias must come together");
    ChannelParams p{a->pooled, a->inv_count, a->cin_w, a->cin_b, a->xc_proj, a->dtc_w, a->dtc_b, a->Ac_logs, a->Dsc,
                    a->cout_w, a->cout_b, a->cn_w, a->cn_b, a->c_out, a->batch, a->C, a->dc, a->Rc, a->N};
    return channel_launch(p, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_pixel_shuffle2_nhwc(const vmb_pixel_shuffle_args* a, void* stream) {
    VMB_CHECK(a && a->x && a->out, "pixel_shuffle: null pointer");
    VMB_CHECK(dt_ok(a->dtype) && a->batch > 0 && a->H > 0 && a->W > 0 && a->C > 0, "pixel_shuffle: bad arguments");
    VMB_CHECK(aligned16(a->x) && (reinterpret_cast<uintptr_t>(a->out) & 3) == 0, "pixel_shuffle: misaligned pointer");
    VMB_CHECK((a->C * elt_size(a->dtype)) % 4 == 0, "pixel_shuffle: output pixels must be whole 32-bit words");
    PixelShuffleParams p{a->x, a->out, a->batch, a->H, a->W, a->C, nullptr};
    return pixel_shuffle_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_pixel_shuffle2_nhwc_bias(const vmb_pixel_shuffle_args* a, const float* bias, void* stream) {
    VMB_CHECK(a && a->x && a->out && bias, "pixel_shuffle_bias: null pointer");
    VMB_CHECK(dt_ok(a->dtype) && a->batch > 0 && a->H > 0 && a->W > 0 && a->C > 0, "pixel_shuffle_bias: bad arguments");
    VMB_CHECK(aligned16(a->x) && (reinterpret_cast<uintptr_t>(a->out) & 3) == 0, "pixel_shuffle_bias: misaligned pointer");
    VMB_CHECK((a->C * elt_size(a->dtype)) % 4 == 0, "pixel_shuffle_bias: output pixels must be whole 32-bit words");
    PixelShuffleParams p{a->x, a->out, a->batch, a->H, a->W, a->C, bias};
    return pixel_shuffle_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_conv3x3(const vmb_conv3x3_args* a, void* stream) {
    VMB_CHECK(a && a->x && a->w && a->out, "conv3x3: null pointer");
    VMB_CHECK(dt_ok(a->dtype), "conv3x3: bad dtype");
    VMB_CHECK(a->batch > 0 && a->batch <= 65535 && a->Cin > 0 && a->Cout > 0 && a->H > 0 && a->W > 0, "conv3x3: bad sizes");
    VMB_CHECK(a->mode >= VMB_CONV_PLAIN && a->mode <= VMB_CONV_ADD_NEAREST, "conv3x3: unknown store mode %d", a->mode);
    VMB_CHECK(a->mode != VMB_CONV_UNSHUFFLE2 || (a->H % 2 == 0 && a->W % 2 == 0), "conv3x3: PixelUnshuffle(2) needs even H, W");
    VMB_CHECK(a->mode != VMB_CONV_SHUFFLE2 || a->Cout % 4 == 0, "conv3x3: PixelShuffle(2) needs Cout %% 4 == 0");
    VMB_CHECK(a->mode != VMB_CONV_ADD_NEAREST || (a->add && a->add_scale >= 1 && a->H % a->add_scale == 0 && a->W % a->add_scale == 0),
              "conv3x3: add image / scale missing or not dividing H, W");
    VMB_CHECK(!a->in_nhwc || a->Cin % 8 == 0 || a->dtype == VMB_F32, "conv3x3: NHWC input needs Cin %% 8 == 0");
    VMB_CHECK(aligned16(a->w) && (!a->in_nhwc || aligned16(a->x)), "conv3x3: weights (and an NHWC input) must be 16 B aligned");
    VMB_CHECK((cdiv(a->Cout, 16)) <= 65535, "conv3x3: too many output channels");
    Conv3Params p{a->x, a->w, a->bias, a->out, a->add, a->batch, a->Cin, a->Cout, a->H, a->W, a->in_nhwc, a->mode, a->add_scale,
                  (a->Cout + 63) / 64 * 64, (a->Cin + 15) / 16 * 16,
                  a->in_nhwc ? (int64_t)a->H * a->W * a->Cin : a->x_bs, a->x_cs, a->o_bs, a->o_cs, a->add_bs, a->add_cs};
    return conv3x3_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_transpose_hw(const vmb_transpose_args* a, void* stream) {
    VMB_CHECK(a && a->x && a->out, "transpose: null pointer");
    VMB_CHECK(dt_ok(a->dtype) && a->planes > 0 && a->H > 0 && a->W > 0, "transpose: bad arguments");
    TransposeParams p{a->x, a->out, a->planes, a->H, a->W};
    return transpose_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_selective_scan_fwd_grouped(const vmb_scan_grouped_args* a, void* stream) {
    VMB_CHECK(a != nullptr, "scan_fwd_grouped: null args");
    VMB_CHECK(dt_ok(a->dtype), "scan_fwd_grouped: bad dtype");
    VMB_CHECK(a->ngroups >= 1 && a->ngroups <= 4 && a->dim % a->ngroups == 0, "scan_fwd_grouped: 1..4 groups dividing dim");
    VMB_CHECK(a->batch > 0 && a->batch <= 65535 && a->dim > 0 && a->seqlen > 0 && a->dstate > 0 && a->dstate <= 16,
              "scan_fwd_grouped: bad sizes (dstate <= 16)");
    VMB_CHECK(a->A != nullptr, "scan_fwd_grouped: A missing");
    ScanFwdParams p{};
    p.A = a->A; p.D = a->D; p.bias = a->delta_bias; p.ckpt = a->ckpt;
    p.batch = a->batch; p.dim = a->dim; p.L = a->seqlen; p.N = a->dstate; p.G = a->ngroups;
    p.npad = 16;
    p.rows_per_group = a->dim / a->ngroups;
    p.n_ckpt = (a->seqlen + kScanCkpt - 1) / kScanCkpt;
    p.u_bs = a->u_bs; p.u_ds = a->u_ds; p.dl_bs = a->delta_bs; p.dl_ds = a->delta_ds; p.o_bs = a->out_bs; p.o_ds = a->out_ds;
    p.B_bs = a->B_bs; p.B_gs = 0; p.B_ns = a->B_ns; p.C_bs = a->C_bs; p.C_gs = 0; p.C_ns = a->C_ns;
    p.softplus = a->delta_softplus;
    const int v = 16 / elt_size(a->dtype);
    auto mult = [v](int64_t s) { return s % v == 0; };
    bool ok = mult(a->u_bs) && mult(a->u_ds) && mult(a->delta_bs) && mult(a->delta_ds) && mult(a->out_bs) && mult(a->out_ds) &&
              mult(a->B_bs) && mult(a->B_ns) && mult(a->C_bs) && mult(a->C_ns) && a->seqlen % v == 0;
    p.ndesc = a->ngroups;
    for (int g = 0; g < a->ngroups; ++g) {
        VMB_CHECK(a->u[g] && a->delta[g] && a->Bm[g] && a->Cm[g] && a->out[g], "scan_fwd_grouped: null tensor pointer (group %d)", g);
        ok = ok && aligned16(a->u[g]) && aligned16(a->delta[g]) && aligned16(a->Bm[g]) && aligned16(a->Cm[g]) && aligned16(a->out[g]);
        p.grp[g] = ScanGroupDesc{a->u[g], a->delta[g], a->Bm[g], a->Cm[g], a->out[g], a->rev[g]};
    }
    p.vec_ok = ok;
    return scan_fwd_launch(p, a->dtype, static_cast<cudaStream_t>(stream));
}

static int scan_bwd_grouped_params(const vmb_scan_grouped_bwd_args* a, ScanBwdParams& p, ScanBwdGroups& gr) {
    VMB_CHECK(a != nullptr, "selective_scan_bwd_grouped: null args");
    VMB_CHECK(dt_ok(a->dtype), "selective_scan_bwd_grouped: dtype must be f32/bf16/f16 (got %d)", a->dtype);
    VMB_CHECK(a->ngroups >= 1 && a->ngroups <= 4 && a->dim % a->ngroups == 0, "selective_scan_bwd_grouped: 1..4 groups dividing dim");
    VMB_CHECK(a->batch > 0 && a->batch <= 65535 && a->dim > 0 && a->seqlen > 0 && a->dstate > 0 && a->dstate <= 16,
              "selective_scan_bwd_grouped: bad sizes (dstate <= 16)");
    VMB_CHECK(a->A && a->dA, "selective_scan_bwd_grouped: A, dA or workspace missing");
    VMB_CHECK(a->ckpt != nullptr || a->seqlen <= kScanCkpt,
              "selective_scan_bwd_grouped: forward checkpoints required when seqlen > %d", kScanCkpt);
    VMB_CHECK((a->D == nullptr) == (a->dD == nullptr), "selective_scan_bwd_grouped: D and dD must both be given or both be NULL");
    VMB_CHECK((a->delta_bias == nullptr) == (a->ddelta_bias == nullptr),
              "selective_scan_bwd_grouped: delta_bias and ddelta_bias must both be given or both be NULL");
    VMB_CHECK(a->deterministic == 0 || a->deterministic == 1, "selective_scan_bwd_grouped: deterministic must be 0 or 1 (got %d)",
              a->deterministic);
    p = ScanBwdParams{};
    p.A = a->A; p.D = a->D; p.bias = a->delta_bias; p.ckpt = a->ckpt;
    p.dA = a->dA; p.dD = a->dD; p.dbias = a->ddelta_bias;
    p.batch = a->batch; p.dim = a->dim; p.L = a->seqlen; p.N = a->dstate; p.G = a->ngroups;
    p.npad = 16;
    p.rows_per_group = a->dim / a->ngroups;
    p.n_ckpt = (a->seqlen + kScanCkpt - 1) / kScanCkpt;
    p.u_bs = a->u_bs; p.u_ds = a->u_ds; p.dl_bs = a->delta_bs; p.dl_ds = a->delta_ds; p.do_bs = a->dout_bs; p.do_ds = a->dout_ds;
    p.du_bs = a->du_bs; p.du_ds = a->du_ds; p.dd_bs = a->ddelta_bs; p.dd_ds = a->ddelta_ds;
    p.B_bs = a->B_bs; p.B_ns = a->B_ns; p.C_bs = a->C_bs; p.C_ns = a->C_ns;
    p.softplus = a->delta_softplus;
    const int v = 16 / elt_size(a->dtype);
    auto mult = [v](int64_t s) { return s % v == 0; };
    bool ok = mult(a->u_bs) && mult(a->u_ds) && mult(a->delta_bs) && mult(a->delta_ds) && mult(a->dout_bs) && mult(a->dout_ds) &&
              mult(a->du_bs) && mult(a->du_ds) && mult(a->ddelta_bs) && mult(a->ddelta_ds) && mult(a->B_bs) && mult(a->B_ns) &&
              mult(a->C_bs) && mult(a->C_ns) && a->seqlen % v == 0;
    gr = ScanBwdGroups{};
    gr.ndesc = a->ngroups;
    gr.dB_bs = a->dB_bs; gr.dB_ns = a->dB_ns; gr.dC_bs = a->dC_bs; gr.dC_ns = a->dC_ns;
    for (int g = 0; g < a->ngroups; ++g) {
        VMB_CHECK(a->u[g] && a->delta[g] && a->Bm[g] && a->Cm[g] && a->dout[g] && a->du[g] && a->ddelta[g] && a->dB[g] && a->dC[g],
                  "selective_scan_bwd_grouped: null tensor pointer (group %d)", g);
        ok = ok && aligned16(a->u[g]) && aligned16(a->delta[g]) && aligned16(a->Bm[g]) && aligned16(a->Cm[g]) && aligned16(a->dout[g]) &&
             aligned16(a->du[g]) && aligned16(a->ddelta[g]);
        gr.grp[g] = ScanBwdGroupDesc{a->u[g], a->delta[g], a->Bm[g], a->Cm[g], a->dout[g], a->du[g], a->ddelta[g], a->dB[g], a->dC[g], a->rev[g]};
    }
    VMB_CHECK(ok, "selective_scan_bwd_grouped: needs 16 B-aligned rows (base pointers, batch / row strides, seqlen %% %d == 0)", v);
    p.vec_ok = true;
    VMB_CHECK((long)p.batch * p.dim < (1L << 31), "selective_scan_bwd_grouped: batch*dim too large");
    return VMB_OK;
}

extern "C" int vmb_selective_scan_bwd_grouped(const vmb_scan_grouped_bwd_args* a, void* stream) {
    ScanBwdParams p;
    ScanBwdGroups gr;
    int rc = scan_bwd_grouped_params(a, p, gr);
    if (rc != VMB_OK) return rc;
    VMB_CHECK(a->workspace, "selective_scan_bwd_grouped: A, dA or workspace missing");
    VMB_CHECK(aligned16(a->workspace), "selective_scan_bwd_grouped: workspace must be 16-byte aligned");
    p.dBC = static_cast<float*>(a->workspace);
    return scan_bwd_grouped_launch(p, gr, a->dtype, static_cast<cudaStream_t>(stream), a->deterministic != 0);
}

extern "C" int64_t vmb_scan_grouped_bwd_det_workspace_bytes(const vmb_scan_grouped_bwd_args* a) {
    ScanBwdParams p;
    ScanBwdGroups gr;
    if (scan_bwd_grouped_params(a, p, gr) != VMB_OK) return -1;
    const int64_t n = scan_bwd_grouped_det_workspace(p);
    if (n < 0) set_error("selective_scan_bwd_grouped: rows per group (%d) must be even", p.rows_per_group);
    return n;
}
