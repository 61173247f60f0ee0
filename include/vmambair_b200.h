/* vmambair_b200 -- C ABI of the H100-native Omni-Selective-Scan operator stack.
 *
 * Plain C: raw device pointers, explicit sizes/strides (in ELEMENTS), a dtype
 * enum and a cudaStream_t (passed as void*).  The caller owns every buffer;
 * the library allocates nothing persistent, never synchronises the host, and
 * is safe to call under CUDA-graph capture.  Every function returns 0 on
 * success; on failure a thread-local message is available from
 * vmb_last_error().
 *
 * Each entry point names the reference interface it replaces (paths relative
 * to the reference repo root).
 */
#ifndef VMAMBAIR_B200_H
#define VMAMBAIR_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VMB_OK 0
#define VMB_ERR_INVALID 1 /* bad shape / dtype / stride / pointer */
#define VMB_ERR_CUDA 2    /* a CUDA runtime call or kernel launch failed */

typedef enum { VMB_F32 = 0, VMB_BF16 = 1, VMB_F16 = 2 } vmb_dtype;

const char* vmb_last_error(void);
/* library / build identification: "vmambair_b200 <ver> sm_90a" */
const char* vmb_version(void);

/* Checkpoint interval (in sequence positions) of the opaque `ckpt` buffer shared by
 * vmb_selective_scan_fwd and _bwd:  ckpt is fp32 (batch, dim, n_ckpt, dstate) with
 * n_ckpt = ceil(seqlen / interval).  Replaces the reference's `x`
 * (B, D, ceil(L/2048), 2N) -- Mamba/kernels/selective_scan/csrc/selective_scan/cus/selective_scan.cpp:217-220. */
int vmb_scan_ckpt_interval(void);

/* ---- B0 operator boundary ------------------------------------------------
 * selective_scan_cuda_core.fwd  (cus/selective_scan.cpp:157-239, kernel
 * cus/selective_scan_fwd_kernel.cuh:61-172).
 *   u, delta, out : (batch, dim, seqlen)   dtype `dt`, last-dim stride 1
 *   A             : (dim, dstate) fp32 contiguous
 *   Bm, Cm        : (batch, ngroups, dstate, seqlen) dtype `dt`, last-dim stride 1
 *   D, delta_bias : (dim) fp32 or NULL
 *   ckpt          : fp32 (batch, dim, n_ckpt, dstate) or NULL (inference: no checkpoints)
 * out = D*u + sum_n C_n * h_n,   h_n,l = exp(dt_l*A_n) h_n,l-1 + dt_l*u_l*B_n,l,
 * dt = softplus?(delta + delta_bias).  State and accumulation in fp32.
 *   out_f32       : 0 -> `out` has dtype `dt`;  1 (bf16 / fp16 `dt` only) -> `out` is fp32, the fp32 accumulator stored without
 *                   rounding: selective_scan_cuda_oflex.fwd(..., out_float=True) (cusoflex/selective_scan_oflex.cpp:157-243,
 *                   out allocated at :219, the <input_t, weight_t, float> kernel at :238).  A zero-initialised tail (out_f32 and
 *                   the members below) keeps the plain operator.
 * The z gate and the last state of mamba_ssm's selective_scan_cuda.fwd(u, delta, A, B, C, D, z, delta_bias, delta_softplus)
 * (its wrapper: Mamba/kernels/selective_scan/test_selective_scan.py:18-165; RealSR/VmambaIR/archs/MambaRealSR11_arch.py:294):
 *   z, out_z      : (batch, dim, seqlen) dtype `dt`, last-dim stride 1, both given or both NULL.  out_z = out * z * sigmoid(z),
 *                   from the fp32 accumulator, rounded once; `out` is still written, ungated.  Not with out_f32 (VMB_ERR_INVALID).
 *   ckpt_pairs    : 1 -> ckpt is fp32 (batch, dim, n_ckpt, 2 dstate), 16 B aligned: ckpt[b,d,k,2n+1] = h_n after position
 *                   min(interval (k+1), seqlen) - 1 and ckpt[b,d,k,2n] = 0, so ckpt[:, :, -1, 1::2] is the last state for every
 *                   seqlen (the reference wrapper's `x[:, :, -1, 1::2]`, :79).  vmb_selective_scan_bwd reads the dense
 *                   ckpt[..., 1::2] copy.  0 -> the layout above.  z with a ckpt buffer requires ckpt_pairs = 1. */
typedef struct {
    const void* u; const void* delta; const float* A; const void* Bm; const void* Cm;
    const float* D; const float* delta_bias; void* out; float* ckpt;
    int batch, dim, seqlen, dstate, ngroups;
    int64_t u_bs, u_ds;         /* batch / dim strides of u      */
    int64_t delta_bs, delta_ds; /* ... of delta                   */
    int64_t out_bs, out_ds;     /* ... of out                     */
    int64_t B_bs, B_gs, B_ns;   /* batch / group / state strides  */
    int64_t C_bs, C_gs, C_ns;
    int delta_softplus;
    int dtype; /* vmb_dtype of u, delta, Bm, Cm, out (out: fp32 when out_f32) */
    int out_f32;
    const void* z; void* out_z;
    int64_t z_bs, z_ds;         /* batch / dim strides of z       */
    int64_t out_z_bs, out_z_ds; /* ... of out_z                   */
    int ckpt_pairs;
} vmb_scan_fwd_args;
int vmb_selective_scan_fwd(const vmb_scan_fwd_args* a, void* stream);

/* Backward of the z gate of vmb_selective_scan_fwd (mamba_ssm's selective_scan_cuda.bwd, which then runs the scan backward on
 * dout_eff: here vmb_selective_scan_bwd with dout_f32 = 1, or plain for fp32).  Element-wise, fp32 math, s = sigmoid(z):
 *   dout_eff = dout * z * s                      fp32 (batch, dim, seqlen) dense
 *   dz       = dout * out * s * (1 + z (1 - s))  dtype `dt`, caller's buffer (strides dz_bs, dz_ds)
 *   out_z    = out * z * s                       dtype `dt`, optional (NULL: not written; the reference's recompute_out_z)
 * dout, out (the forward's ungated `out`), z: (batch, dim, seqlen) dtype `dt`.  Every tensor has last-dim stride 1. */
typedef struct {
    const void* dout; const void* out; const void* z;
    float* dout_eff; void* dz; void* out_z;
    int batch, dim, seqlen;
    int64_t dout_bs, dout_ds, out_bs, out_ds, z_bs, z_ds, dz_bs, dz_ds, out_z_bs, out_z_ds;
    int dtype;
} vmb_scan_gate_args;
int vmb_scan_gate_bwd(const vmb_scan_gate_args* a, void* stream);

/* Direction-aware variant for the fused OSS path: group g (<= 4 groups, dim = ngroups * rows_per_group) reads its
 * rows from its own tensors and, when rev[g] != 0, walks them backwards (sequence position l <-> memory index
 * L-1-l for u, delta, B, C and out), so the four scan orders of cross_scan_2d
 * (SRGAN/VmambaIR/archs/MambaSISR6_arch.py:401-404) need no flipped / gathered copies: directions 0,2 read the
 * natural (H,W) tensors, directions 1,3 the (W,H)-transposed ones.  Strides are shared by the groups; u/delta/out
 * rows are indexed inside the group.  Requires 16 B-aligned rows (seqlen % 8 == 0 for 16-bit I/O), dstate <= 16.
 *   ckpt : NULL (inference), or fp32 (batch, dim, n_ckpt, dstate) as written by vmb_selective_scan_fwd, indexed by SEQUENCE
 *          position: a reversed group's checkpoints equal the flat forward's on the flipped copy (`out` is the same as without
 *          checkpoints, except that shapes left to the generic kernel run it at <= 2 rows per warp, which may change rounding).  Training forward of
 *          cross_selective_scan (RealSR/VmambaIR/archs/MambaRealSR11_arch.py:371-434; CrossScan :325-343 + SelectiveScan fwd). */
typedef struct {
    const void* u[4]; const void* delta[4]; const void* Bm[4]; const void* Cm[4]; void* out[4]; int rev[4];
    const float* A; const float* D; const float* delta_bias;   /* (dim, dstate), (dim), (dim): indexed by g*rows+r */
    int batch, dim, seqlen, dstate, ngroups;
    int64_t u_bs, u_ds, delta_bs, delta_ds, out_bs, out_ds, B_bs, B_ns, C_bs, C_ns;
    int delta_softplus;
    int dtype;
    float* ckpt;
} vmb_scan_grouped_args;
int vmb_selective_scan_fwd_grouped(const vmb_scan_grouped_args* a, void* stream);

/* selective_scan_cuda_core.bwd  (cus/selective_scan.cpp:241-349, kernel
 * cus/selective_scan_bwd_kernel.cuh:66-273).
 *   dout, du, ddelta : (batch, dim, seqlen) dtype `dt`
 *   dA (dim,dstate), dD (dim), ddelta_bias (dim): fp32, ACCUMULATED into (caller zero-fills,
 *       like the reference's torch::zeros_like, cpp:321-327)
 *   dB, dC : (batch, ngroups, dstate, seqlen) contiguous, dtype `dt`, fully written (the reference
 *       accumulates in fp32 and casts in torch, cpp:322-323,347; here the fp32 accumulation lives in
 *       `workspace` and the cast is done by the library)
 *   workspace : device scratch of vmb_scan_bwd_workspace_bytes(...) bytes, 16 B aligned; the library
 *       zero-fills it on `stream`
 *   ckpt  : as written by the forward (required when seqlen > interval).
 *   dout_f32 : 0 -> dout has dtype `dt`;  1 (bf16 / fp16 `dt` only) -> dout is fp32, read without rounding:
 *       selective_scan_cuda_oflex.bwd (cusoflex/selective_scan_oflex.cpp:245-358; output_type == Float at :260, :353).
 *       du, ddelta, dB, dC keep dtype `dt`; dA, dD, ddelta_bias stay fp32 (cpp:324-356).  Zero keeps the plain operator.
 *   deterministic : 0 -> the fp32 sums over rows and batch are float atomics (run-to-run differences in the last bits), `workspace`
 *       as above;  1 -> bitwise reproducible: every contributing CTA stores its partial sums into its own slot of `workspace`
 *       (vmb_scan_bwd_det_workspace_bytes(a) bytes, 16 B aligned, not zero-filled: every slot read is written) and a second
 *       kernel sums them in a fixed order, writes dB / dC and ADDS one sum to each element of dA, dD, ddelta_bias.  Other
 *       values return VMB_ERR_INVALID.  Last member. */
typedef struct {
    const void* u; const void* delta; const float* A; const void* Bm; const void* Cm;
    const float* D; const float* delta_bias; const void* dout; const float* ckpt;
    void* du; void* ddelta; float* dA; void* dB; void* dC; float* dD; float* ddelta_bias; void* workspace;
    int batch, dim, seqlen, dstate, ngroups;
    int64_t u_bs, u_ds, delta_bs, delta_ds, dout_bs, dout_ds;
    int64_t du_bs, du_ds, ddelta_bs, ddelta_ds;
    int64_t B_bs, B_gs, B_ns, C_bs, C_gs, C_ns;
    int delta_softplus;
    int dtype;
    int dout_f32;
    int deterministic;
} vmb_scan_bwd_args;
int vmb_selective_scan_bwd(const vmb_scan_bwd_args* a, void* stream);
int64_t vmb_scan_bwd_workspace_bytes(int batch, int ngroups, int dstate, int seqlen);
/* workspace of the deterministic mode for exactly these arguments (the launch configuration depends on the sizes, dtype, strides
 * and alignment; `workspace` and `deterministic` are ignored): 16 nc batch ngroups ceil16(dstate)/2 seqlen + 4 batch dim (dstate + 2)
 * bytes, nc = the CTAs that share one (batch, group).  -1 for invalid arguments (vmb_last_error()). */
int64_t vmb_scan_bwd_det_workspace_bytes(const vmb_scan_bwd_args* a);

/* Direction-aware backward, the adjoint of vmb_selective_scan_fwd_grouped: group g (<= 4) reads u, delta, Bm, Cm, dout from its own
 * tensors and writes du, ddelta (batch, rows, seqlen) and dB, dC (batch, dstate, seqlen) to its own destinations, every one in the
 * memory order of that group's sources (rev[g] != 0: sequence position l <-> memory index L-1-l).  Same values as
 * vmb_selective_scan_bwd on the gathered / flipped copies followed by scattering the results back -- what CrossScan.backward +
 * SelectiveScan.backward compute (RealSR/VmambaIR/archs/MambaRealSR11_arch.py:295-343) without the four gathered copies.
 *   dA (dim,dstate), dD (dim), ddelta_bias (dim): fp32, indexed by g*rows+r, ACCUMULATED into (caller zero-fills)
 *   workspace : vmb_scan_bwd_workspace_bytes(batch, ngroups, dstate, seqlen) bytes, 16 B aligned, zero-filled by the library
 *       (deterministic = 1: vmb_scan_grouped_bwd_det_workspace_bytes(a) bytes, not zero-filled)
 *   ckpt : as written by vmb_selective_scan_fwd_grouped (required when seqlen > interval)
 *   deterministic : 0 or 1, as for vmb_selective_scan_bwd; last member
 * Strides are shared by the groups.  Requires 16 B-aligned rows of u, delta, Bm, Cm, dout, du, ddelta (seqlen % 8 == 0 for
 * 16-bit I/O, % 4 for fp32) and dstate <= 16; dB / dC need no alignment.  Anything else returns VMB_ERR_INVALID. */
typedef struct {
    const void* u[4]; const void* delta[4]; const void* Bm[4]; const void* Cm[4]; const void* dout[4];
    void* du[4]; void* ddelta[4]; void* dB[4]; void* dC[4]; int rev[4];
    const float* A; const float* D; const float* delta_bias; const float* ckpt;
    float* dA; float* dD; float* ddelta_bias; void* workspace;
    int batch, dim, seqlen, dstate, ngroups;
    int64_t u_bs, u_ds, delta_bs, delta_ds, dout_bs, dout_ds, du_bs, du_ds, ddelta_bs, ddelta_ds;
    int64_t B_bs, B_ns, C_bs, C_ns, dB_bs, dB_ns, dC_bs, dC_ns;
    int delta_softplus;
    int dtype;
    int deterministic;
} vmb_scan_grouped_bwd_args;
int vmb_selective_scan_bwd_grouped(const vmb_scan_grouped_bwd_args* a, void* stream);
int64_t vmb_scan_grouped_bwd_det_workspace_bytes(const vmb_scan_grouped_bwd_args* a);  /* as vmb_scan_bwd_det_workspace_bytes */


/* ---- B1 module boundary: fused stages of one OSS block (inference) -------------------------------
 * These replace the un-fused PyTorch ops of SS2D_1 / MamberBlock / FeedForward
 * (SRGAN/VmambaIR/archs/MambaSISR6_arch.py:166-218, 395-515).  Activations are NCHW, pixel-contiguous. */

/* out[b,m,p] = epi( sum_k W[m,k] * pro(x)[b,k,p] ): 1x1 conv with fused LayerNorm / channel-gate prologue and
 * bias / SiLU-range / residual epilogue.  Replaces norm1+in_conv (:487-489), x_proj (:409-410), gate+out_conv+
 * residual (:494-498,:512), norm2+project_in (:213), project_out+residual (:217,:513). */
typedef struct {
    const void* x; const void* w; const float* bias; const void* residual; void* out;
    const float* ln_w; const float* ln_b;   /* LayerNorm over K per pixel (ln_mode 1: WithBias, 2: BiasFree) */
    const float* gate;                      /* (B,K) fp32: gate_mode 1: x*(1+g), 2: x+g */
    int ln_mode, gate_mode;
    int act_from, act_to;                   /* SiLU on output channels [act_from, act_to) */
    int batch, K, M, P;
    int64_t x_bs, x_cs, r_bs, r_cs, o_bs, o_cs, g_bs;
    int64_t w_ld;                           /* row stride of w (0: = K); rows padded to a multiple of 16 elements load vectorised */
    int dtype, out_dtype;                   /* x / w / residual dtype; out dtype (same, or VMB_F32) */
} vmb_pixlin_args;
int vmb_pixlin(const vmb_pixlin_args* a, void* stream);

/* depthwise 3x3 (pad 1) + bias, then mode 0: SiLU (SS2D_1.conv2d+act :490-491), mode 1: gelu(conv[c]) *
 * conv[c+C_out] (FeedForward.dwconv + gate :215-216), or mode 2: nothing (the transposed conv of the backward pass, called
 * with the spatially flipped taps).  w: (channels, 9) fp32. */
typedef struct {
    const void* x; const float* w; const float* bias; void* out;
    int batch, c_out, H, W, mode;
    int64_t x_bs, x_cs, o_bs, o_cs;
    int dtype;
} vmb_dwconv_args;
int vmb_dwconv3x3(const vmb_dwconv_args* a, void* stream);
/* mode 0 with a second output out_t (B, c_out, W*H) dense: every plane of `out` transposed -- the (W,H)-ordered copy of x that the
 * column-major scan directions (cross_scan_2d :402) and their x_proj GEMM read; replaces a vmb_transpose_hw pass behind the conv
 * (`out` must be dense). */
int vmb_dwconv3x3_t(const vmb_dwconv_args* a, void* out_t, void* stream);

/* four scan orders by index arithmetic (cross_scan_2d :401-404; CrossScan RealSR arch :325-343):
 * out[b][k][row][l] = src[k][b][row][pi_k(l)];  pi_0(l)=l, pi_1(w*H+h)=h*W+w, pi_2 = pi_0(L-1-l), pi_3 = pi_1(L-1-l). */
typedef struct {
    const void* src[4]; void* out;
    int batch, rows, H, W;
    int64_t src_bs, src_rs, out_bs;
    int dtype;
    int64_t out_ks; /* element stride between the four directions of `out` (0: rows * H * W, dense) */
} vmb_cross_scan_args;
int vmb_cross_scan(const vmb_cross_scan_args* a, void* stream);
/* 1..4 cross-scans of one geometry (same dtype, batch, H, W; own sources, row counts and destinations) in ONE launch: what the
 * training path needs per block -- x, delta and B|C gathered into the four scan orders (forward), du, ddelta, dB, dC scattered back
 * (backward; the inverse orders = H and W swapped).  Same values as nseg calls of vmb_cross_scan. */
int vmb_cross_scan_multi(const vmb_cross_scan_args* segs, int nseg, void* stream);

/* (B*C) planes of H x W -> W x H (the transposed copy of x that directions 1 and 3 scan). */
typedef struct { const void* x; void* out; int planes, H, W; int dtype; } vmb_transpose_args;
int vmb_transpose_hw(const vmb_transpose_args* a, void* stream);

/* PixelShuffle(2) of the SR tail (Upsampler, SRGAN/VmambaIR/archs/common.py:45-60; nn.PixelShuffle semantics:
 * out[b, c, 2h+i, 2w+j] = in[b, 4c + 2i + j, h, w]) on channels-last storage: x (B,H,W,4C) -> out (B,2H,2W,C), so the
 * 3x3 convs either side run on their native NHWC layout without layout-transform kernels.  A pure permutation:
 * results are bit-identical to torch.nn.functional.pixel_shuffle. */
typedef struct { const void* x; void* out; int batch, H, W, C; int dtype; } vmb_pixel_shuffle_args;
int vmb_pixel_shuffle2_nhwc(const vmb_pixel_shuffle_args* a, void* stream);
/* the same with bias (fp32, 4C values) added to the input channels first: the Upsampler convs (archs/common.py:52) run without
 * their bias and the permutation pass that follows them adds it -- one elementwise pass over the widest tensors of the net less. */
int vmb_pixel_shuffle2_nhwc_bias(const vmb_pixel_shuffle_args* a, const float* bias, void* stream);

/* Dense 3x3 convolution, stride 1, zero padding 1 -- the non-OSS convolutions of the U-Net (SURVEY 8f rank 1):
 * OverlapPatchEmbed.proj (SRGAN/VmambaIR/archs/MambaSISR6_arch.py:520-528), Downsample.body = Conv2d + PixelUnshuffle(2)
 * (:533-541), Upsample.body = Conv2d + PixelShuffle(2) (:544-553), the SR tail's last conv + the nearest-neighbour up-sampled
 * input (:607,640; Upsampler in archs/common.py:45-60), Mamber32.output + inp_img (Deraining mamber32_arch.py forward).
 * What the reference runs as separate passes behind the conv is index arithmetic of the store:
 *   mode VMB_CONV_PLAIN        out[b, m, y, x]                                   (out may be a channel slice of a wider tensor:
 *                                                                                 the decoder's torch.cat([up, skip], 1) never runs)
 *        VMB_CONV_UNSHUFFLE2   out[b, 4m + 2(y%2) + x%2, y/2, x/2]               nn.PixelUnshuffle(2); H, W even
 *        VMB_CONV_SHUFFLE2     out[b, m/4, 2y + (m/2)%2, 2x + m%2]               nn.PixelShuffle(2); Cout % 4 == 0
 *        VMB_CONV_ADD_NEAREST  out[b, m, y, x] = conv + add[b, m, y/s, x/s]      F.interpolate(add, scale_factor=s, 'nearest'), s >= 1
 * x: NCHW view (x_bs, x_cs element strides; planes dense) or, in_nhwc = 1, dense NHWC (B,H,W,Cin) with Cin % 8 == 0.
 * out: NCHW planes dense with (o_bs, o_cs) strides; its spatial size is (H/2, W/2), (2H, 2W) or (H, W) by mode.
 * w: the Conv2d weight (Cout, Cin, 3, 3) re-packed by the caller as [tap = 3*ky + kx][Mpad][Kpad] in the I/O dtype, zero padded,
 *    Mpad = Cout rounded up to 64, Kpad = Cin rounded up to 16 (static parameters: the kernel may read them before the preceding
 *    kernel of the stream has finished).  bias: fp32 (Cout) or NULL.  16-bit I/O: tensor-core implicit GEMM, fp32 accumulation;
 *    fp32 I/O: FFMA. */
#define VMB_CONV_PLAIN 0
#define VMB_CONV_UNSHUFFLE2 1
#define VMB_CONV_SHUFFLE2 2
#define VMB_CONV_ADD_NEAREST 3
typedef struct {
    const void* x; const void* w; const float* bias; void* out; const void* add;
    int batch, Cin, Cout, H, W;
    int in_nhwc, mode, add_scale;
    int64_t x_bs, x_cs, o_bs, o_cs, add_bs, add_cs;
    int dtype;
} vmb_conv3x3_args;
int vmb_conv3x3(const vmb_conv3x3_args* a, void* stream);

/* inverse orders + 4-way fp32 sum (:427-430 / CrossMerge) + out_norm (:433) + gate y*SiLU(z) (:493) +
 * per-(b,c) sums of the result for AdaptiveAvgPool2d (:441; `pooled` fp32 (B,C), fully written).
 * workspace: vmb_merge_workspace_bytes() bytes of device scratch (fp32 merged values + per-pixel statistics + tile sums).
 * 16-bit I/O with H, W multiples of 16 and C <= 96 runs ONE kernel (all channels of a 16x16 pixel tile per CTA, no atomics on the
 * statistics); other shapes a channel-split sum kernel + a normalisation kernel. */
typedef struct {
    const void* ys; const void* z; const float* ln_w; const float* ln_b; void* y2; float* pooled;
    int batch, C, H, W;
    int64_t z_bs, z_cs;
    int dtype;
    void* workspace;
    int in_place_order; /* 0: ys[k] in scan order (k=2,3 reversed); 1: ys[0],ys[2] in natural (H,W) pixel order and
                           ys[1],ys[3] in transposed (W,H) pixel order (outputs of vmb_selective_scan_fwd_grouped) */
    int z_preact;       /* 0: z already holds SiLU(z) (inference: the in_conv epilogue applied it); 1: z is the pre-activation
                           and SiLU is applied here (training: the backward needs the pre-activation) */
    int save_ws;        /* 1: the workspace keeps the fp32 merged values (B,C,L) followed by the per-pixel (sum, sum of squares)
                           over C (B,L,2) for vmb_merge_norm_gate_bwd; 0: its content is unspecified afterwards */
} vmb_merge_args;
int vmb_merge_norm_gate(const vmb_merge_args* a, void* stream);
int64_t vmb_merge_workspace_bytes(int batch, int C, int H, int W);
/* the inverse orders + 4-way fp32 sum alone (CrossMerge.forward, RealSR/VmambaIR/archs/MambaRealSR11_arch.py:346-355): out fp32 (batch,
 * C, H*W) dense, same values as the merged sum of vmb_merge_norm_gate.  Uses a->ys, batch, C, H, W, in_place_order, dtype and the
 * workspace (per-pixel statistics); z, ln_w, ln_b, y2, pooled are ignored. */
int vmb_merge_sum(const vmb_merge_args* a, float* out, void* stream);

/* the channel-direction OSS for one image per CTA (cforward_corev1 :438-483; Mamber32/33 and RealSR variants):
 * pooled means -> conv_cin -> xc_proj / dtc_proj -> bidirectional selective scan over L=C -> conv_cout ->
 * channel_norm.  All parameters fp32; c_out fp32 (B,C). cin_w / cout_w may be NULL (RealSR: dc=1). */
typedef struct {
    const float* pooled; float inv_count;
    const float* cin_w; const float* cin_b; const float* xc_proj; const float* dtc_w; const float* dtc_b;
    const float* Ac_logs; const float* Dsc; const float* cout_w; const float* cout_b; const float* cn_w; const float* cn_b;
    float* c_out;
    int batch, C, dc, Rc, N;
} vmb_channel_args;
int vmb_channel_branch(const vmb_channel_args* a, void* stream);

/* ---- training path: backward of the fused stages (autograd of the modules above; SURVEY.md 8 a15) ----------------
 * The 1x1-conv data gradients are vmb_pixlin with the transposed weight, the scan gradient is vmb_selective_scan_bwd,
 * the direction gathers are vmb_cross_scan (pi_k^-1 = pi_k with H and W swapped).  Parameter gradients (dw, db, ...) are
 * fp32 and ACCUMULATED into (the caller zero-fills), like the reference's autograd accumulates .grad. */

/* y = LayerNorm_C(x) per pixel, materialised (the weight-gradient GEMMs of in_conv / project_in need it);
 * mode 1: WithBias, 2: BiasFree (MambaSISR6_arch.py:166-195).  y and/or stats (B, L, 2) = (mean, rstd) may be NULL. */
typedef struct {
    const void* x; const float* w; const float* b; void* y; float* stats;
    int batch, C, L, mode;
    int64_t x_bs, x_cs, y_bs, y_cs;
    int dtype;
} vmb_ln_fwd_args;
int vmb_layernorm_fwd(const vmb_ln_fwd_args* a, void* stream);

/* dx = LayerNorm backward of g (gradient w.r.t. the LayerNorm output) [+ add]; dw += sum g*xhat, db += sum g (dw/db may be NULL).
 * stats: fp32 scratch (B, L, 2), written by the data-gradient kernel.  Two-phase use (weight gradients on another stream):
 * dw = NULL -> dx (+ stats) only; dx = NULL -> dw / db only, from x, g and the stats of the earlier call. */
typedef struct {
    const void* x; const void* g; const void* add; const float* w; void* dx; float* dw; float* db; float* stats;
    int batch, C, L, mode;
    int64_t x_bs, x_cs, g_bs, g_cs, a_bs, a_cs, dx_bs, dx_cs;
    int dtype;
} vmb_ln_bwd_args;
int vmb_layernorm_bwd(const vmb_ln_bwd_args* a, void* stream);

/* backward of vmb_merge_norm_gate (z_preact = 1): merged / stats = the forward's workspace (fp32 merged scan output (B,C,L) and the
 * per-pixel (sum, sum of squares) over C); dy2 (B,C,L) dense, dpooled (B,C) fp32 or NULL.
 * -> dm (B,C,L) dense: gradient w.r.t. the merged scan output (gathered into the four scan orders by vmb_cross_scan),
 *    dz: gradient w.r.t. the pre-activation z, dw/db += out_norm parameter gradients.
 * Two-phase use: dw = db = NULL -> data gradients only; dm = dz = NULL -> parameter gradients only. */
typedef struct {
    const float* merged; const float* stats; const void* z; const void* dy2; const float* dpooled;
    const float* w; const float* b; void* dm; void* dz; float* dw; float* db;
    int batch, C, L;
    int64_t z_bs, z_cs, dz_bs, dz_cs;
    int dtype;
} vmb_merge_bwd_args;
int vmb_merge_norm_gate_bwd(const vmb_merge_bwd_args* a, void* stream);

/* backward of vmb_dwconv3x3 up to the conv output: dv = gradient w.r.t. the conv result before the activation
 * (mode 0: g * silu'(v); mode 1: dv[c] = g * v2 * gelu'(v1), dv[c+c_out] = g * gelu(v1)); the conv itself is recomputed from x.
 * dw (channels, 9) / dbias (channels) fp32 accumulated when dw != NULL.  The input gradient is vmb_dwconv3x3(dv, flipped taps, mode 2).
 * Two-phase use: dw = NULL -> dv only; g = NULL -> dv is an INPUT (an earlier call's) and only dw / dbias are accumulated. */
typedef struct {
    const void* x; const float* w; const float* bias; const void* g; void* dv; float* dw; float* dbias;
    int batch, c_out, H, W, mode;
    int64_t x_bs, x_cs, g_bs, g_cs, dv_bs, dv_cs;
    int dtype;
} vmb_dwconv_bwd_args;
int vmb_dwconv3x3_bwd(const vmb_dwconv_bwd_args* a, void* stream);

/* backward of the channel gate in front of out_conv (vmb_pixlin gate_mode 1: y*(1+c), 2: y+c): dyg, y2 (B,C,L) dense ->
 * dy2 (B,C,L), dgate (B,C) fp32 (fully written). */
typedef struct {
    const void* dyg; const void* y2; const float* gate; void* dy2; float* dgate;
    int batch, C, L, mode;
    int dtype;
} vmb_gate_bwd_args;
int vmb_channel_gate_bwd(const vmb_gate_bwd_args* a, void* stream);

/* backward of vmb_channel_branch (one CTA per image recomputes the forward in shared memory and walks it backwards).
 * fwd: the forward's arguments (c_out unused).  dc_out (B,C) fp32: gradient w.r.t. the forward's output.
 * -> d_pooled (B,C) fp32, fully written (gradient w.r.t. the pooled SUMS); every parameter gradient fp32, ACCUMULATED (zero-filled
 * by the caller), shaped like its parameter; d_cin_* / d_cout_* NULL exactly when the forward's are.
 * scratch: vmb_channel_branch_bwd_scratch_bytes(batch, dc, C) bytes.  Shared memory: vmb_channel_branch_bwd_smem_bytes(C, dc, Rc, N)
 * must be <= 227 KB (C <= 192 for dc = 4; wider levels keep the composed torch path). */
typedef struct {
    vmb_channel_args fwd;
    const float* dc_out; float* d_pooled;
    float* d_cin_w; float* d_cin_b; float* d_xc_proj; float* d_dtc_w; float* d_dtc_b; float* d_Ac_logs; float* d_Dsc;
    float* d_cout_w; float* d_cout_b; float* d_cn_w; float* d_cn_b;
    float* scratch;
} vmb_channel_bwd_args;
int vmb_channel_branch_bwd(const vmb_channel_bwd_args* a, void* stream);
int64_t vmb_channel_branch_bwd_smem_bytes(int C, int dc, int Rc, int N);
int64_t vmb_channel_branch_bwd_scratch_bytes(int batch, int dc, int C);

/* Two-direction channel selective scan, cross_selective_scanC (RealSR/VmambaIR/archs/MambaRealSR11_arch.py:438-534: CrossScanC,
 * the x_proj / dt_proj einsums, SelectiveScan, CrossMergeC), one CTA per image, everything in fp32 shared memory:
 *   xs_0 = x[b] (D, L), xs_1 = flip_L(x[b]);  x_dbl_k = W_k xs_k (+ bias_k);  dt_k = softplus?(Wdt_k x_dbl_k[:R] + dt_bias_k)
 *   y_k = selective scan of (u = xs_k, dt_k, A_k = -exp(A_logs[k]), B = x_dbl_k[R:R+N], C = x_dbl_k[R+N:], D = Ds[k])
 *   y[b][l][d] = y_0[d][l] + y_1[d][L-1-l]
 *   x : (batch, D, L) in `dtype`, element strides x_bs / x_ds, last stride 1
 *   x_proj_weight (2, R+2N, D), x_proj_bias (2, R+2N) or NULL, dt_projs_weight (2, D, R), dt_projs_bias (2D), A_logs (2D, N),
 *   Ds (2D): fp32 contiguous
 *   y : forward output, fp32 (batch, L, D) dense (the reference's (B, L, 1, D))
 * Bounds: d_state N <= 16, D <= 16 and vmb_cross_selective_scan_c_smem_bytes(D, L, R, N) <= 227 KB (every RealSR channel call:
 * D = 1, N = 16, L = C <= 384, R = ceil(C/16)); anything else returns VMB_ERR_INVALID. */
typedef struct {
    const void* x;
    const float* x_proj_weight; const float* x_proj_bias; const float* dt_projs_weight; const float* dt_projs_bias;
    const float* A_logs; const float* Ds;
    float* y;
    int batch, D, L, R, N;
    int64_t x_bs, x_ds;
    int delta_softplus;
    int dtype;
} vmb_cross_scan_c_args;
int vmb_cross_selective_scan_c_fwd(const vmb_cross_scan_c_args* a, void* stream);
/* backward: recomputes the forward per image and walks the recurrence backwards.  fwd: the forward's arguments (y unused).
 *   dy : fp32 (batch, L, D) dense, gradient w.r.t. y;  dx : (batch, D, L) dense, x's dtype, fully written
 *   d_params : fp32, fully written (not accumulated), packed as x_proj_weight (2(R+2N)D), x_proj_bias (2(R+2N); written even when
 *              the bias is NULL), dt_projs_weight (2DR), dt_projs_bias (2D), A_logs (2DN), Ds (2D)
 *   workspace : vmb_cross_selective_scan_c_workspace_bytes(batch, D, R, N) bytes: the per-image gradients, which a second kernel
 *               sums over the batch in a fixed order (no atomics: bitwise reproducible) */
typedef struct {
    vmb_cross_scan_c_args fwd;
    const float* dy; void* dx; float* d_params; float* workspace;
} vmb_cross_scan_c_bwd_args;
int vmb_cross_selective_scan_c_bwd(const vmb_cross_scan_c_bwd_args* a, void* stream);
/* shared-memory bytes the backward (the larger of the two kernels) needs at (D, L, R, N); -1 when N > 16 or D > 16 */
int64_t vmb_cross_selective_scan_c_smem_bytes(int D, int L, int R, int N);
int64_t vmb_cross_selective_scan_c_workspace_bytes(int batch, int D, int R, int N);

/* weight gradient of a 1x1 conv: out[m][k] += sum_{b,p} dy[b][m][p] * x[b][k][p]  (out fp32 (M,K), accumulated: the caller zero-fills;
 * per_batch != 0: out is (B,M,K) and batches are not summed -- the channel gate in front of out_conv scales them per image).
 * dy (B,M,L), x (B,K,L): bf16 / fp16 views with 16 B aligned, pixel-contiguous rows.  mma.sync tensor-core kernel, split over
 * pixels.  (fp32 activations: use the library GEMM.)
 * deterministic = 0: the pixel splits meet in fp32 atomics (workspace unused, may be NULL);  1: bitwise reproducible -- every CTA stores
 * its partial into its own slot of `workspace` (vmb_pixlin_wgrad_workspace_bytes(a) bytes, 16 B aligned, not zero-filled) and a
 * second kernel adds the slots' sum, taken in a fixed order, once to each element of out and dbias.  Other values: VMB_ERR_INVALID. */
typedef struct {
    const void* dy; const void* x; float* out;
    int batch, M, K, L;
    int64_t dy_bs, dy_cs, x_bs, x_cs;
    int per_batch;
    int dtype;
    float* dbias; /* optional (M) fp32, accumulated: dbias[m] += sum_{b,p} dy[b][m][p] (the conv's bias gradient) */
    void* workspace;
    int deterministic;
} vmb_wgrad_args;
int vmb_pixlin_wgrad(const vmb_wgrad_args* a, void* stream);
/* 4 batch splits (M K + M if dbias) bytes: the deterministic mode's partial slots for exactly these arguments; -1 for bad sizes */
int64_t vmb_pixlin_wgrad_workspace_bytes(const vmb_wgrad_args* a);

/* Per-step weight preparation of one OSS block in ONE launch: every job converts an fp32 parameter into the layout a kernel of
 * this library consumes.  type 0: (M,K) -> dst (M, ld) in `dtype`, columns >= K zero;  1: (M,K) -> dst (K, ld) = transpose, columns
 * >= M zero;  2: fold x_proj (src: (4, K+N2, M)) and dt_proj (src2: (4, M, K)) into big (dst: (4(M+N2), ld)) and its transpose
 * (dst2: (M, ld2)) -- big[k] = [W_dt,k W_x,k[:K] ; W_x,k[K:]], M = C, K = dt_rank, N2 = 2*d_state;  3: dst = -exp(src), fp32 (M,K);
 * 4: dst = the 9 taps of (M, 9) spatially flipped, fp32. */
#define VMB_PREP_MAX_JOBS 16
typedef struct {
    const float* src; const float* src2; void* dst; void* dst2;
    int type, M, K, N2, ld, ld2;
} vmb_prep_job;
typedef struct {
    vmb_prep_job jobs[VMB_PREP_MAX_JOBS];
    int njobs;
    int dtype;
} vmb_prep_args;
int vmb_prep_block_weights(const vmb_prep_args* a, void* stream);

/* out = add + x4[:,0] + x4[:,1] + x4[:,2] + x4[:,3]: x4 (batch, 4, per_dir) contiguous, add / out (batch, per_dir) contiguous
 * (the four un-permuted direction gradients of the scan input joined with the x_proj data gradient). */
int vmb_sum4_add(const void* x4, const void* add, void* out, int batch, long per_dir, int dtype, void* stream);

/* Fused Adam / AdamW step + gradient clipping + EMA over FLAT fp32 buffers of n elements (optimizer_g.step(), clip_grad_norm_,
 * model_ema(): SRGAN/VmambaIR/models/MambaSISR_model.py:141-147, Deraining/basicsr/models/image_restoration_model.py:165-173,
 * Deraining/basicsr/models/base_model.py:54-62).  grad is first multiplied by grad_scale (1/world after the all-reduce) and, when
 * max_grad_norm > 0, by min(1, max_grad_norm / (||grad|| + 1e-6)).  state: 4 floats on the device, zero-initialised by the
 * caller; state[0] is the step count, advanced by this call (so CUDA-graph replays keep the bias correction right).
 * ema (NULL: none): ema = ema_decay * ema + (1 - ema_decay) * param.  zero_grad != 0 clears the gradient buffer. */
typedef struct {
    float* param; float* grad; float* exp_avg; float* exp_avg_sq; float* ema; float* state;
    long n;
    float lr, beta1, beta2, eps, weight_decay;
    int decoupled_weight_decay;   /* 0: Adam (L2 added to the gradient), 1: AdamW */
    float grad_scale, max_grad_norm, ema_decay;
    int zero_grad;
} vmb_adam_args;
int vmb_fused_adam(const vmb_adam_args* a, void* stream);

/* ---- image-level I/O: the host-side conversions of RealESRGANer.enhance (RealSR/VmambaIR/utils.py:174-243) ----------------------
 * Images are 8- or 16-bit (u16 = 0 / 1), H x W pixels of `channels` (1 gray, 3 BGR, 4 BGRA) values; element strides between rows,
 * pixels and channels are given separately, so crops, flips and channel views need no copy.  Planes are NCHW in the compute dtype. */

/* largest value of an image (every channel) -> *max_out (uint32, device); the library zero-fills it first on `stream`.  enhance() reads
 * it back once to choose 8- or 16-bit processing (np.max(img) > 256, utils.py:178). */
typedef struct {
    const void* img;
    int H, W, channels, u16;
    int64_t row_stride, pixel_stride, channel_stride;
    unsigned int* max_out;
} vmb_image_max_args;
int vmb_image_max(const vmb_image_max_args* a, void* stream);

/* image -> planes (pre_process + the colour conversions of enhance, utils.py:71-91,177-196), one pass:
 *   v = img / max_range (an IEEE float division, as numpy's), BGR -> RGB, a gray channel repeated three times;
 *   out (1 + alpha_plane, 3, Hp, Wp) dense in `dtype`; alpha_plane = 1 (channels 4 only): image 1 of the batch is the alpha channel
 *   repeated three times (the 'realesrgan' alpha upsampler runs it through the network);
 *   pad_h[i] / pad_w[i]: three successive bottom / right reflect pads (F.pad 'reflect'): pre_pad, the mod pad, the pad to the
 *   network's multiple; each smaller than the size it pads.  Hp = H + sum pad_h, Wp = W + sum pad_w. */
typedef struct {
    const void* img; void* out;
    int H, W, channels, u16;
    int64_t row_stride, pixel_stride, channel_stride;
    float max_range;
    int pad_h[3], pad_w[3];
    int alpha_plane;
    int dtype;
} vmb_image_to_planes_args;
int vmb_image_to_planes(const vmb_image_to_planes_args* a, void* stream);

/* planes -> image (post_process + the output half of enhance, utils.py:162-171,205-234), one pass:
 *   planes (batch, 3, *, *) in `dtype` with element strides p_bs, p_cs, p_rs (pixels contiguous); the top-left H x W pixels are read
 *   (post_process's crops); v = clamp(plane, 0, 1); RGB -> BGR;
 *   channels 1: the gray value fma(r, 0.299f, fma(b, 0.114f, g * 0.587f)) (cv2 COLOR_BGR2GRAY on float32);
 *   channels 4: alpha_mode 0 -> the gray value of planes image 1;  alpha_mode 1 -> cv2.resize(alpha_src / max_range, (W, H),
 *     INTER_LINEAR) of the source image's alpha channel (alpha_src: alpha_H x alpha_W, uint8 or uint16 (alpha_u16), strides
 *     alpha_rs / alpha_ps): half-pixel centres, replicated border, s0 a0 + s1 a1 per row then per column in float32;
 *   out = saturate(rint(v * max_range)) (numpy's round half to even), uint8 or uint16 (u16) HWC, element strides out_rs (rows),
 *   out_ps (pixels); channels stride 1. */
typedef struct {
    const void* planes; void* out; const void* alpha_src;
    int H, W, channels, u16;
    int64_t p_bs, p_cs, p_rs;
    int64_t out_rs, out_ps;
    int alpha_mode, alpha_H, alpha_W, alpha_u16;
    int64_t alpha_rs, alpha_ps;
    float max_range;
    int dtype;
} vmb_planes_to_image_args;
int vmb_planes_to_image(const vmb_planes_to_image_args* a, void* stream);

/* cv2.resize(src, (dW, dH), interpolation=cv2.INTER_LANCZOS4) on uint8 / uint16 HWC images (enhance's outscale, utils.py:236-241):
 * sample x = (dx + 0.5) sW / dW - 0.5 (OpenCV's float rounding of it), 8 x 8 taps at floor(x) - 3 .. floor(x) + 4 clamped to the
 * image, Lanczos weights normalised in float; 8-bit: 11-bit fixed-point weights, int32 sums, the 22-bit result rounded; 16-bit:
 * float sums, row pass then column pass, rounded half to even and saturated.  Strides in elements; channels stride 1. */
typedef struct {
    const void* src; void* dst;
    int sH, sW, dH, dW, channels, u16;
    int64_t src_rs, src_ps, dst_rs, dst_ps;
} vmb_resize_lanczos4_args;
int vmb_resize_lanczos4(const vmb_resize_lanczos4_args* a, void* stream);

/* ---- image metrics: PSNR and SSIM of Deraining/basicsr/metrics/psnr_ssim.py and Deraining/Deraining/utils.py ----------------------
 * A source is `batch` images of H x W pixels of `channels` values (1 gray, or 3 in BGR order), already cropped: element (b, y, x, c) is
 * at img + b batch_stride + y row_stride + x pixel_stride + c channel_stride (element strides; any sign, so an RGB planar network
 * output is read as BGR through a negative channel stride).  `dtype` says how an element becomes the reference's float64 value:
 *   VMB_MSRC_U8 / U16 / F32 / F64 : the value itself (img.astype(np.float64));
 *   VMB_MSRC_Q_F32 / Q_BF16 / Q_F16: tensor2img (SRGAN/VmambaIR/utils/img_util.py:36-): rint(clamp(float(v), 0, 1) * 255.f) in float32,
 *                                    half to even, as uint8.
 * y_channel = 1: every metric sees to_y_channel(img) (metrics/metric_util.py, utils/matlab_functions.py:207-238,305-361) instead:
 *   3 channels: x_c = fl32(fl32(v_c) / 255);  Y = fl32(fl32((x_B 24.966 + x_G 128.553 + x_R 65.481 + 16) / 255) * 255), the sum
 *               in float64 left to right, never contracted;  1 channel: Y = fl32(fl32(fl32(v) / 255) * 255). */
#define VMB_MSRC_U8 0
#define VMB_MSRC_U16 1
#define VMB_MSRC_F32 2
#define VMB_MSRC_F64 3
#define VMB_MSRC_Q_F32 4
#define VMB_MSRC_Q_BF16 5
#define VMB_MSRC_Q_F16 6
typedef struct {
    const void* img;
    int dtype;
    int64_t batch_stride, row_stride, pixel_stride, channel_stride;
} vmb_metric_src;

/* to_y_channel (metrics/metric_util.py) of every pixel of `src` -> out (batch, H, W) dense float32.  channels 1 or 3. */
typedef struct {
    vmb_metric_src src;
    int batch, H, W, channels;
    float* out;
} vmb_to_y_args;
int vmb_to_y_channel(const vmb_to_y_args* a, void* stream);

/* PSNR of each image pair (calculate_psnr, psnr_ssim.py:9-63; utils.py:10-25), deterministic: per-CTA float64 partial sums of the
 * squared differences in a fixed order, then one CTA per image adds them in index order.  The squared difference is float64, or with
 * y_channel float32 (a - b) squared in float32, as the reference forms it.  Per image b:
 *   mse[b] = sum / (H W channels') (channels' = 1 with y_channel), max_value[b] = the largest value of img1 (after y_channel),
 *   psnr[b] = mse == 0 ? inf : 20 log10(m / sqrt(mse)), m = 1 if max_value[b] <= 1 else 255 (device log10).
 * workspace: vmb_psnr_workspace_bytes(a) bytes of device memory. */
typedef struct {
    vmb_metric_src img1, img2;
    int batch, H, W, channels, y_channel;
    double *mse, *max_value, *psnr;
    void* workspace;
} vmb_psnr_args;
int vmb_psnr(const vmb_psnr_args* a, void* stream);
int64_t vmb_psnr_workspace_bytes(const vmb_psnr_args* a);

/* SSIM of each image pair in float64, from 11 x 11 Gaussian moments (x, y, x^2, y^2, xy) filtered separably from a shared-memory tile
 * with its 5-pixel halo; taps: cv2.getGaussianKernel(11, 1.5).  ssim[b] is the mean of the SSIM map:
 *   VMB_SSIM_VALID       the map where the window fits, (H - 10) x (W - 10) per channel, averaged per channel, then over the channels
 *                        (_ssim, psnr_ssim.py:66-99; ssim / calculate_ssim, utils.py:31-78); nan when H or W < 11;
 *   VMB_SSIM_REPLICATE   full-size map, borders replicated (_ssim_cly, psnr_ssim.py:184-222); one channel (y_channel or gray);
 *   VMB_SSIM_REPLICATE3D as REPLICATE, and the channels filtered too, by the 11-tap filter with replicated ends across them
 *                        (_ssim_3d, psnr_ssim.py:131-182): moment[c] = sum_c' mix[c][c'] moment2d[c'] (mix: channels x channels,
 *                        row-major, the taps folded onto the clamped channel indices).
 * C1 = (0.01 m)^2, C2 = (0.03 m)^2 with m = 255, except in REPLICATE3D, where m = 1 if max_value[b] <= 1 else 255 (max_value: device,
 * per image, e.g. vmb_psnr's).  Partial sums per CTA and channel, added in index order by one CTA per image: deterministic.
 * workspace: vmb_ssim_workspace_bytes(a) bytes of device memory. */
#define VMB_SSIM_VALID 0
#define VMB_SSIM_REPLICATE 1
#define VMB_SSIM_REPLICATE3D 2
typedef struct {
    vmb_metric_src img1, img2;
    int batch, H, W, channels, y_channel;
    int mode;
    double taps[11];
    double mix[9];
    const double* max_value;
    double* ssim;
    void* workspace;
} vmb_ssim_args;
int vmb_ssim(const vmb_ssim_args* a, void* stream);
int64_t vmb_ssim_workspace_bytes(const vmb_ssim_args* a);

/* ---- NIQE: calculate_niqe of Deraining/basicsr/metrics/niqe.py (niqe, compute_feature, estimate_aggd_param) --------------------
 * Three launches per call: vmb_niqe_prep, vmb_niqe_features, vmb_niqe_score; vmb_niqe_table once per device.  Blocks are 96 x 96 at
 * scale 1 and 48 x 48 on the half plane; an image's H and W are cut to whole blocks before anything is filtered.  No atomics: every
 * sum has a fixed order, so results are bitwise reproducible and do not depend on the batch. */
#define VMB_NIQE_BLOCK 96
#define VMB_NIQE_TABLE 9801   /* gam = np.arange(0.2, 10.001, 0.001) */
#define VMB_NIQE_FEATURES 36  /* 18 per scale */
#define VMB_NIQE_Y 0          /* to_y_channel (1 or 3 channels), bit for bit as vmb_to_y_channel */
#define VMB_NIQE_GRAY 1       /* cv2.cvtColor(img / 255., COLOR_BGR2GRAY) * 255. in float32: (B .114f + G .587f) + R .299f, unfused */
#define VMB_NIQE_PLANE 2      /* the value as float32 (input_order='HW'); 1 channel */

/* table[i] = gamma(2 / g)^2 / (gamma(1 / g) gamma(3 / g)), g = 0.2 + i ((0.2 + 0.001) - 0.2), in fp64 (device tgamma). */
int vmb_niqe_table(double* table, void* stream);

/* The float32 plane of `src` (batch images, H x W, already cropped to whole blocks: H, W multiples of 96) after the float32 cast and
 * `convert` -> plane (batch, H, W), and half (batch, H / 2, W / 2) = fl32(((q00 + q01) + (q10 + q11)) * .25f) * 255.f with
 * q = fl32(v / 255.f) over each 2 x 2 quad, standing in for cv2.resize(img / 255., (w // 2, h // 2), INTER_LINEAR) * 255. */
typedef struct {
    vmb_metric_src src;
    int batch, H, W, channels, convert;
    float *plane, *half;
} vmb_niqe_prep_args;
int vmb_niqe_prep(const vmb_niqe_prep_args* a, void* stream);

/* One CTA per block and scale.  MSCN: mu = window * img, sigma = sqrt(|window * fl32(img^2) - mu^2|), n = (img - mu) / (sigma + 1),
 * each convolution (edges 'nearest' on the cut plane) summed in fp64 and rounded once to float32, the rest float32.  Per block, five
 * distributions (n, and n times n rolled circularly within the block by [0,1], [1,0], [1,1], [1,-1], float32 products) fitted as
 * estimate_aggd_param does, from fp64 sums; alpha by search of `table` (vmb_niqe_table, on the device).  features (batch, blocks, 36)
 * fp64: row w nbh + h for block (h, w), scale 1's 18 features then scale 2's.  mscn, mscn_half (NULL: not written): the normalised
 * planes, (batch, H, W) and (batch, H / 2, W / 2).  window: the 7 x 7 Gaussian of the pristine parameters, row-major. */
typedef struct {
    const float *plane, *half;
    const double* table;
    double* features;
    float *mscn, *mscn_half;
    double window[49];
    int batch, H, W;
} vmb_niqe_features_args;
int vmb_niqe_features(const vmb_niqe_features_args* a, void* stream);

/* One CTA per image: score[b] = sqrt(d ((cov_pris + cov_d) / 2)^-1 d^T), d = mu_pris - nanmean(features[b], axis 0), cov_d the
 * ddof-1 covariance of the rows without a NaN, all fp64, sums in row order; NaN with fewer than two such rows (blocks 0 included).
 * mu_pris (36) and cov_pris (36 x 36, row-major): fp64 on the device. */
typedef struct {
    const double* features;
    const double *mu_pris, *cov_pris;
    double* score;
    int batch, blocks;
} vmb_niqe_score_args;
int vmb_niqe_score(const vmb_niqe_score_args* a, void* stream);

/* ---- degradations: the Real-ESRGAN synthesis operators of basicsr that RealSR/VmambaIR/models/MambaRealSR_model.py:145-260 uses --
 * Every image is float32 NCHW, contiguous: `batch` images of `channels` planes of H x W.  Nothing reads the host. */

/* filter2D (basicsr.utils.img_process_util): out = the k x k cross-correlation of each plane with `kernel` (k x k float32, one shared
 * kernel, per_image = 0, or one per image, per_image = 1, (batch, k, k)), pads of k / 2 with torch's 'reflect' semantics.  k odd,
 * 1..51; H and W > k / 2 (where torch's reflect pad works).  quantize_out: out = clamp(rint(v 255), 0, 255) / 255. */
typedef struct {
    const float* img;
    float* out;
    const float* kernel;
    int batch, channels, H, W, k, per_image, quantize_out;
} vmb_filter2d_args;
int vmb_filter2d(const vmb_filter2d_args* a, void* stream);

/* USMSharp(radius).forward(img, weight, threshold) (basicsr.utils.img_process_util) with the separable kernel taps x taps^T (taps:
 * cv2.getGaussianKernel(k, sigma) in float32, k odd <= 51): blur = G * img, residual = img - blur,
 * mask = |residual| 255 > threshold, soft = G * mask, out = soft clip(img + weight residual, 0, 1) + (1 - soft) img.  Two launches;
 * workspace: batch channels H W floats (the mask).  img, out and workspace must not alias. */
typedef struct {
    const float* img;
    float* out;
    float* workspace;
    int batch, channels, H, W, k;
    float taps[51];
    float weight, threshold;
} vmb_usm_sharp_args;
int vmb_usm_sharp(const vmb_usm_sharp_args* a, void* stream);

/* DiffJPEG(differentiable=False)(img, quality) (basicsr.utils.diffjpeg) of 3-channel RGB images in [0, 1]: zero pads to multiples of
 * 16, x 255, YCbCr (JFIF matrix, shift 128), 4:2:0 by 2 x 2 averages, orthonormal 8 x 8 DCT-II, rint(D / (T factor)) (T factor) with
 * basicsr's transposed tables, inverse DCT, chroma repeated 2 x 2, back to RGB, clamped to [0, 255], / 255, cropped.  One CTA per four
 * 16 x 16 MCUs.  quality: (batch,) device float32, factor = (q < 50 ? 5000 / q : 200 - 2 q) / 100 per image in float32 (not
 * modified); NULL: the host-computed `factor` for every image.  A zero step (quality 100) keeps the coefficient: the lossless limit.
 * clamp_in: clamp(img, 0, 1) on load.  quantize_out: as in vmb_filter2d_args. */
typedef struct {
    const float* img;
    float* out;
    const float* quality;
    float factor;
    int batch, H, W, clamp_in, quantize_out;
} vmb_jpeg_args;
int vmb_jpeg(const vmb_jpeg_args* a, void* stream);

/* The levels of generate_poisson_noise_pt (basicsr.data.degradations) of 3-channel images, without a host read: q = clamp(rint(x 255),
 * 0, 255) / 255 per element and qg the same of torchvision's gray 0.2989 r + 0.587 g + 0.114 b (separate float32 roundings);
 * vals[b] = 2^ceil(log2(distinct q of image b)), vals_gray[b] likewise of qg (256-bit presence masks, atomicOr: deterministic);
 * rates = q vals (batch, 3, H, W), rates_gray = qg vals_gray (batch, 1, H, W).  workspace: 64 batch bytes. */
typedef struct {
    const float* img;
    float *rates, *rates_gray, *vals, *vals_gray;
    void* workspace;
    int batch, H, W;
} vmb_noise_levels_args;
int vmb_noise_levels(const vmb_noise_levels_args* a, void* stream);

/* out = img + noise of random_add_gaussian_noise_pt / random_add_poisson_noise_pt, from torch's draws:
 *   param[b] = u_param[b] param_span + param_lo (sigma or scale), g[b] = (u_gray[b] < gray_prob);
 *   GAUSSIAN: noise = randn(b, c, H, W) sigma / 255, noise_gray = randn(H, W) sigma / 255, mixed noise (1 - g) + noise_gray g;
 *   POISSON (3 channels): noise = P / vals - q, noise_gray = Pg / vals_gray - qg (P, Pg: torch.poisson of vmb_noise_levels' rates,
 *            rates_gray), mixed as above, times scale.
 * Then clip and rounds as the reference: clamp(rint(v 255), 0, 255) / 255, clamp(v, 0, 1), or rint(v 255) / 255.  Every operation is
 * one float32 rounding, in the reference's order.  out must not alias img. */
#define VMB_NOISE_GAUSSIAN 0
#define VMB_NOISE_POISSON 1
typedef struct {
    const float* img;
    float* out;
    const float *noise, *noise_gray, *u_param, *u_gray;
    float param_lo, param_span, gray_prob;
    const float *vals, *vals_gray;
    int kind, batch, channels, H, W, clip, rounds;
} vmb_noise_apply_args;
int vmb_noise_apply(const vmb_noise_apply_args* a, void* stream);

/* ---- GAN stage: UNetDiscriminatorSN (RealSR/VmambaIR/archs/discriminator_arch.py:19-67) between its convolutions, and basicsr's
 * vanilla GANLoss (MambaRealSRGAN_model.py:289-359 calls both).  Activations are NCHW contiguous, fp32 or bf16 (dtype VMB_F32 /
 * VMB_BF16); all math is fp32.  No atomics: every reduction has one fixed order, so results are bitwise reproducible. */

/* torch.nn.utils.spectral_norm (dim 0, one power iteration) of up to VMB_SN_MAX_LAYERS layers in one call (discriminator_arch.py:
 * 28-38 wraps conv1..conv8).  Layer i: w[i] = weight_orig viewed as (rows[i], cols[i]) fp32; u[i] (rows), v[i] (cols) fp32.
 *   train = 1: v = normalize(W^T u), u = normalize(W v) (normalize(x) = x / max(|x|, eps)), written back to u[i], v[i];
 *   train = 0: u, v as stored.
 * Then sigma[i] = u . (W v), wn[i] = W / sigma[i] in `dtype`, and the u, v used are copied to u_save[i], v_save[i] (the backward's
 * constants).  Four launches in train mode, two in eval mode, whatever the layer count.
 * workspace: vmb_sn_workspace_bytes(layers, rows, cols) bytes; columns <= 56 K (v is staged in shared memory). */
#define VMB_SN_MAX_LAYERS 8
typedef struct {
    const float* w[VMB_SN_MAX_LAYERS];
    void* wn[VMB_SN_MAX_LAYERS];
    float* u[VMB_SN_MAX_LAYERS];
    float* v[VMB_SN_MAX_LAYERS];
    float* u_save[VMB_SN_MAX_LAYERS];
    float* v_save[VMB_SN_MAX_LAYERS];
    int rows[VMB_SN_MAX_LAYERS], cols[VMB_SN_MAX_LAYERS];
    float* sigma;
    void* workspace;
    int layers, train, dtype;
    float eps;
} vmb_sn_fwd_args;
int vmb_sn_fwd(const vmb_sn_fwd_args* a, void* stream);
int64_t vmb_sn_workspace_bytes(int layers, const int* rows, const int* cols);

/* Backward of vmb_sn_fwd with u, v constant (as spectral_norm's clones): g[i] = dL/dwn (dtype), then
 * dW_orig = g / sigma - (<g, W_orig> / sigma^2) u v^T, written to grad[i] (fp32), or added to it where accumulate[i] != 0 (the
 * .grad accumulation of the parameter).  Two launches: per-chunk partials of <g, W_orig>, then the update, which adds each
 * layer's partials in index order.  workspace: vmb_sn_bwd_workspace_bytes(layers, rows, cols) bytes. */
typedef struct {
    const void* g[VMB_SN_MAX_LAYERS];
    const float* w[VMB_SN_MAX_LAYERS];
    const float* u[VMB_SN_MAX_LAYERS];
    const float* v[VMB_SN_MAX_LAYERS];
    float* grad[VMB_SN_MAX_LAYERS];
    int rows[VMB_SN_MAX_LAYERS], cols[VMB_SN_MAX_LAYERS], accumulate[VMB_SN_MAX_LAYERS];
    const float* sigma;
    void* workspace;
    int layers, dtype;
} vmb_sn_bwd_args;
int vmb_sn_bwd(const vmb_sn_bwd_args* a, void* stream);
int64_t vmb_sn_bwd_workspace_bytes(int layers, const int* rows, const int* cols);

/* Decoder junction (discriminator_arch.py:49-56): out = F.interpolate(leaky_relu(pre, 0.2) [+ skip], scale_factor=2,
 * mode='bilinear', align_corners=False) of `planes` planes of H x W into 2H x 2W; weights 0.75 / 0.25 with clamped borders, in
 * torch's order of operations.  skip: NULL for none. */
typedef struct {
    const void *pre, *skip;
    void* out;
    int planes, H, W, dtype;
} vmb_gan_up_args;
int vmb_gan_up(const vmb_gan_up_args* a, void* stream);

/* Its backward: adj = up2^T(dout) as a gather (each input element sums its 4 x 4 output neighbourhood in a fixed order; torch's
 * upsample_bilinear2d_backward scatters with atomics), dskip = adj (NULL: not written), dpre = adj leaky'(pre). */
typedef struct {
    const void *dout, *pre;
    void *dpre, *dskip;
    int planes, H, W, dtype;
} vmb_gan_up_bwd_args;
int vmb_gan_up_bwd(const vmb_gan_up_bwd_args* a, void* stream);

/* Encoder activation (discriminator_arch.py:42-45, 59-63): out = leaky_relu(x, 0.2) [+ skip] over n elements; out may be x. */
typedef struct {
    const void *x, *skip;
    void* out;
    int64_t n;
    int dtype;
} vmb_gan_act_args;
int vmb_gan_act(const vmb_gan_act_args* a, void* stream);

/* Its backward: dx = (g [+ g2]) leaky'(ref), ref the pre-activation or the in-place result (same sign); g2 NULL for none, dx may
 * be g.  At x0, x1, x2 g2 is the skip connection's gradient, so the sum is never stored. */
typedef struct {
    const void *g, *g2, *ref;
    void* dx;
    int64_t n;
    int dtype;
} vmb_gan_act_bwd_args;
int vmb_gan_act_bwd(const vmb_gan_act_bwd_args* a, void* stream);

/* basicsr GANLoss(gan_type='vanilla'): *loss = weight mean(BCEWithLogits(x, target)) over n logits, per element
 * max(x, 0) - x target + log1p(exp(-|x|)).  Per-CTA partials, then one CTA adds them in order.
 * workspace: vmb_bce_logits_workspace_bytes(n) bytes. */
typedef struct {
    const void* x;
    float* loss;
    void* workspace;
    int64_t n;
    float target, weight;
    int dtype;
} vmb_bce_logits_args;
int vmb_bce_logits(const vmb_bce_logits_args* a, void* stream);
int64_t vmb_bce_logits_workspace_bytes(int64_t n);

/* Its backward: grad_x = grad_loss weight (sigmoid(x) - target) / n, grad_loss read from the device (fp32 scalar). */
typedef struct {
    const void* x;
    const float* grad_loss;
    void* grad_x;
    int64_t n;
    float target, weight;
    int dtype;
} vmb_bce_logits_bwd_args;
int vmb_bce_logits_bwd(const vmb_bce_logits_bwd_args* a, void* stream);

/* ---- Perceptual loss: basicsr's PerceptualLoss (losses/basic_loss.py) on VGGFeatureExtractor (archs/vgg_arch.py), the generator
 * step's perceptual_opt of both GAN recipes, between its convolutions.  It replaces the extractor's ReLU and MaxPool2d modules, the
 * feature clone()s, the subtractions and the L1Loss / MSELoss / torch.norm of every feature, and their autograd backward.  The
 * output x and the ground truth gt run as one 2B batch: images 0..B-1 are x's, B..2B-1 gt's.  Activations are NCHW contiguous,
 * fp32 or bf16 (dtype VMB_F32 / VMB_BF16); all math is fp32.  No atomics: every reduction has one fixed order. */
#define VMB_PERCEP_L1 0  /* criterion 'l1': mean |d| */
#define VMB_PERCEP_L2 1  /* 'l2': mean d^2 */
#define VMB_PERCEP_FRO 2 /* 'fro': sqrt(sum d^2) */
#define VMB_PERCEP_MAX_FEATS 37 /* every layer name of vgg19 */

/* The extractor's input (vgg_arch.py forward, range_norm then use_input_norm): out[b] = norm(x[b]), out[B + b] = norm(gt[b]) with
 * norm(v) = ((v + 1) / 2 - mean[c]) / std[c], the first step only when range_norm, the second only when mean / std are given (the
 * module's fp32 buffers, read on the device; NULL for neither).  x, gt: fp32 (B, 3, H, W) through element strides; out (2B, 3, H, W). */
typedef struct {
    const float *x, *gt;
    int64_t x_stride[4], gt_stride[4];
    const float *mean, *std;
    void* out;
    int B, H, W, range_norm, dtype;
} vmb_percep_norm_args;
int vmb_percep_norm(const vmb_percep_norm_args* a, void* stream);

/* Its backward for x: dx = g / std[c] (when std), then / 2 (when range_norm); g (B, 3, H, W) dtype, dx fp32 contiguous. */
typedef struct {
    const void* g;
    float* dx;
    const float* std;
    int B, H, W, range_norm, dtype;
} vmb_percep_norm_bwd_args;
int vmb_percep_norm_bwd(const vmb_percep_norm_bwd_args* a, void* stream);

/* One stage after a convolution: y (2B, C, H, W) is the conv output (with bias).  Three feature sites: 0 conv (y before the ReLU;
 * basicsr clones it because the ReLU is in place), 1 relu (after it), 2 pool (after MaxPool2d(2, 2), floor sizes, the first maximum
 * of the row-major window wins).  feat[k] != 0: site k is a feature, and partial[k][cta] receives the CTA's sum of |d| (l1) or d^2
 * (l2, fro) of d = x half - gt half there, vmb_percep_stage_ctas(B, C, H, W) CTAs.
 * relu: y = max(y, 0) in place (not written back when pool: only the pooled tensor is read again); pool: pooled (2B, C, H/2, W/2).
 * Saved for the backward, x half only, per 2 x 2 cell of ceil(H/2) x ceil(W/2): code[cell] bits 0-3 = [y > 0] of the cell's
 * elements in row-major order, bits 4-5 the pool argmax (code NULL: nothing saved).  save[k] (NULL: nothing saved) for l1 a byte per
 * cell with 2 bits per element (bit 0 d > 0, bit 1 d < 0), at the pool site a byte per pooled element; for l2 / fro d itself in fp32
 * (the site's x-half shape). */
typedef struct {
    void* y;
    void* pooled;
    uint8_t* code;
    void* save[3];
    float* partial[3];
    int feat[3];
    int B, C, H, W, relu, pool, crit, dtype;
} vmb_percep_stage_args;
int vmb_percep_stage(const vmb_percep_stage_args* a, void* stream);
int vmb_percep_stage_ctas(int B, int C, int H, int W);

/* The loss in one CTA: feature k's partials are partial[offset[k] .. offset[k + 1]), added in index order; value[k] = sum / numel[k]
 * (l1, l2) or sqrt(sum) (fro), and *loss = perceptual_weight * sum_k value[k] weight[k], k ascending (basicsr's order). */
typedef struct {
    const float* partial;
    float* loss;
    float* value;
    int offset[VMB_PERCEP_MAX_FEATS + 1];
    int64_t numel[VMB_PERCEP_MAX_FEATS];
    float weight[VMB_PERCEP_MAX_FEATS];
    int feats, crit;
    float perceptual_weight;
} vmb_percep_loss_args;
int vmb_percep_loss(const vmb_percep_loss_args* a, void* stream);

/* Backward of one stage for the x half: g_out (B, C, H, W) = [y > 0] (dpost) + c0 crit'(d at the conv site), where dpost = the
 * pool adjoint of g_in (+ c2 crit'), a gather through the saved argmax, or g_in itself without a pool, + c1 crit' at the relu site.
 * g_in: the gradient at the stage's output ((B, C, H/2, W/2) with pool, else (B, C, H, W)); NULL at the deepest stage.
 * c_k = *grad_loss scale[k] (scale = pw w_k / N_k for l1, 2 pw w_k / N_k for l2, pw w_k for fro), for fro divided by
 * value[feat_index[k]] (0 where that norm is 0).  grad_loss: the upstream fp32 scalar, read on the device.  Without relu (a stage
 * cut before its ReLU) the mask is all ones and code may be NULL. */
typedef struct {
    const void* g_in;
    void* g_out;
    const uint8_t* code;
    const void* save[3];
    const float* grad_loss;
    const float* value;
    int feat[3], feat_index[3];
    float scale[3];
    int B, C, H, W, relu, pool, crit, dtype;
} vmb_percep_stage_bwd_args;
int vmb_percep_stage_bwd(const vmb_percep_stage_bwd_args* a, void* stream);

/* ---- Perceptual metrics: LPIPS (lpips.LPIPS(net='vgg'), version 0.1; RealSR/Metric/LPIPS.py) and DISTS (RealSR/Metric/dists.py)
 * between the VGG16 convolutions.  The two images of each pair run as one 2B batch: images 0..B-1 are the first of each pair,
 * B..2B-1 the second.  Activations are fp32 NCHW contiguous; the ReLU (and LPIPS's max-pool) between the convolutions is
 * vmb_percep_stage.  No atomics: every partial has one writer and the final kernels add them in index order. */
#define VMB_PMETRIC_LPIPS 0
#define VMB_PMETRIC_DISTS 1
#define VMB_PMETRIC_MAX_LAYERS 6 /* DISTS: the input and relu1_2 .. relu5_3 */

/* An input image batch: element (b, c, h, w) at data + b stride[0] + c stride[1] + h stride[2] + w stride[3] (elements, c in RGB
 * order; a BGR image is addressed from its channel 2 with a negative channel stride).  u8 = 0: fp32 values; 1: uint8 levels. */
typedef struct {
    const void* data;
    int64_t stride[4];
    int u8;
} vmb_pmetric_src;

/* The input preparation of both metrics in one launch (replaces LPIPS's `2 * in0 - 1` and ScalingLayer, LPIPS.py:25-31's
 * `/ 255.` and normalize(mean=.5, std=.5); DISTS's forward_once `(x - self.mean) / self.std` (dists.py:71), prepare_image's
 * ToTensor (:117-121) and the layer-0 statistics of forward's loop (:99-109)).  out[b] from src[0], out[B + b] from src[1], (2B, 3, H, W) fp32:
 *   LPIPS: v = u / 255 then (v - .5) / .5 (uint8), or 2 v - 1 (fp32 with normalize), or v; out = (v - shift[c]) / scale[c].
 *   DISTS: v = u / 255 (uint8) or v; out = (v - shift[c]) / scale[c] (the ImageNet mean / std), and when stats != NULL the
 *   statistics of the raw v as vmb_dists_layer writes them, C = 3, tiles = vmb_pmetric_tiles(3 B, H W) over pixels.
 * Each step is one IEEE fp32 operation, as the scripts' numpy / torch conversions.  shift, scale: 3 fp32 on the device. */
typedef struct {
    vmb_pmetric_src src[2];
    const float *shift, *scale;
    float* out;
    double* stats;
    int B, H, W, metric, normalize;
} vmb_pmetric_prep_args;
int vmb_pmetric_prep(const vmb_pmetric_prep_args* a, void* stream);
/* CTAs per plane of the statistics kernels: `items` (pixels or 2 x 2 cells) of each of `planes` planes, split so that a
 * layer fills the GPU even at B = 1 (a fixed rule, not the device's SM count, so the partials do not depend on the device). */
int vmb_pmetric_tiles(int planes, int64_t items);

/* One LPIPS feature layer (replaces lpips.normalize_tensor, (f0 - f1) ** 2, lin{k} and spatial_average's sum): y (2B, C, H, W) is
 * the conv output before the ReLU, applied on load.  Per pixel n_i = sqrt(sum_c f_i^2) + 1e-10, then
 * sum_c w[c] (f0 / n0 - f1 / n1)^2 (two passes over the channels, held in registers; the square is never expanded).
 * partial[b * ctas + cta] = the CTA's sum of that over its pixels of image b, ctas = vmb_lpips_layer_ctas(B, H, W).
 * C / 16 must be 4, 8, 16 or 32 (VGG16: 64 .. 512). */
typedef struct {
    const float* y;
    const float* w;
    float* partial;
    int B, C, H, W;
} vmb_lpips_layer_args;
int vmb_lpips_layer(const vmb_lpips_layer_args* a, void* stream);
int vmb_lpips_layer_ctas(int B, int H, int W);

/* LPIPS's result in one CTA (replaces spatial_average's division and `val += res[l]`): layer k's partials of image b are
 * partial[offset[k] + b * ctas[k] + i], i ascending; layer[k * B + b] = their sum / hw[k]; out[b] = sum over k ascending. */
typedef struct {
    const float* partial;
    float *layer, *out;
    int offset[VMB_PMETRIC_MAX_LAYERS], ctas[VMB_PMETRIC_MAX_LAYERS];
    int64_t hw[VMB_PMETRIC_MAX_LAYERS];
    int B, layers;
} vmb_lpips_final_args;
int vmb_lpips_final(const vmb_lpips_final_args* a, void* stream);

/* One DISTS feature layer (replaces the stage's ReLU, the next stage's L2pooling (dists.py:24-27) and the means / variances /
 * covariance of forward's loop (:100-108)): y (2B, C, H, W) is the conv output before the ReLU, applied on load.  stats[((b C + c) tiles + t) 5 + s], s = sum f0,
 * sum f1, sum f0^2, sum f1^2, sum f0 f1 over tile t of the 2 x 2 cells of plane c of pair b (tiles = vmb_pmetric_tiles(B C,
 * ceil(H/2) ceil(W/2))), accumulated in fp64.  pooled (NULL: none): L2pooling, sqrt(sum 3 x 3 [.25 .5 .25]^T [.25 .5 .25] f^2 +
 * 1e-12) with stride 2 and zero padding 1, (2B, C, ceil(H/2), ceil(W/2)). */
typedef struct {
    const float* y;
    float* pooled;
    double* stats;
    int B, C, H, W;
} vmb_dists_layer_args;
int vmb_dists_layer(const vmb_dists_layer_args* a, void* stream);

/* DISTS's score in one CTA (replaces forward's S1, S2, the alpha / beta sums and batch_average, dists.py:92-115): layer k's statistics start at entry offset[k]
 * (entries of 5 doubles), C[k] channels, tiles[k] tiles per channel, n[k] pixels per plane.  Per channel, in fp64: the tiles added
 * in order, mu = sum / n, var = sum f^2 / n - mu^2, cov = sum f0 f1 / n - mu0 mu1, S1 = (2 mu0 mu1 + 1e-6) / (mu0^2 + mu1^2 + 1e-6),
 * S2 = (2 cov + 1e-6) / (var0 + var1 + 1e-6); score[b] = 1 - sum_j (alpha_j S1_j + beta_j S2_j) / (sum alpha + sum beta) over all
 * channels j in layer order.  alpha, beta: sum C[k] fp32 on the device.  mean (NULL: not written): the mean of score over b. */
typedef struct {
    const double* stats;
    const float *alpha, *beta;
    float *score, *mean;
    int64_t offset[VMB_PMETRIC_MAX_LAYERS], n[VMB_PMETRIC_MAX_LAYERS];
    int C[VMB_PMETRIC_MAX_LAYERS], tiles[VMB_PMETRIC_MAX_LAYERS];
    int B, layers;
} vmb_dists_final_args;
int vmb_dists_final(const vmb_dists_final_args* a, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VMAMBAIR_B200_H */
