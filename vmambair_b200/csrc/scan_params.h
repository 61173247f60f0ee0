// Internal parameter blocks of the selective-scan kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vmb {

constexpr int kScanT = 16;      // sequence positions per lane per chunk
constexpr int kScanCkpt = 64;   // checkpoint interval (positions); see vmb_scan_ckpt_interval()

// Per-group sources (direction-aware fused path): group g of the scan reads its rows from its own tensors and may
// walk them backwards (rev: sequence position l <-> memory index L-1-l for u, delta, B, C and out).
struct ScanGroupDesc {
    const void *u, *delta, *Bm, *Cm;
    void* out;
    int rev;
};

struct ScanFwdParams {
    const void *u, *delta, *Bm, *Cm;
    const float *A, *D, *bias;
    void* out;
    float* ckpt;
    int batch, dim, L, N, G, npad, rows_per_group, n_ckpt;
    int64_t u_bs, u_ds, dl_bs, dl_ds, o_bs, o_ds;
    int64_t B_bs, B_gs, B_ns, C_bs, C_gs, C_ns;
    int softplus;
    bool vec_ok;
    int ndesc;              // 0: flat tensors (B0 operator); else = G <= 4 group descriptors (strides shared, per-group bases)
    ScanGroupDesc grp[4];
    int num_sms;
};

// Per-group operands of the direction-aware backward: the forward's sources, the incoming gradient and the four gradient
// outputs of group g, all in the memory order of that group's sources (rev: sequence position l <-> memory index L-1-l).
struct ScanBwdGroupDesc {
    const void *u, *delta, *Bm, *Cm, *dout;
    void *du, *ddelta, *dB, *dC;
    int rev;
};

struct ScanBwdParams {
    const void *u, *delta, *Bm, *Cm, *dout;
    const float *A, *D, *bias, *ckpt;
    void *du, *ddelta, *dB, *dC;  // I/O dtype
    float *dA, *dD, *dbias;      // fp32, accumulated into
    float* dBC;                  // fp32 scratch [b][g][npad/2][L][4], zeroed by the launcher
    int batch, dim, L, N, G, npad, rows_per_group, n_ckpt;
    int64_t u_bs, u_ds, dl_bs, dl_ds, do_bs, do_ds, du_bs, du_ds, dd_bs, dd_ds;
    int64_t B_bs, B_gs, B_ns, C_bs, C_gs, C_ns;
    int softplus;
    bool vec_ok;
    int debug_nored;  // profiling only (VMB_BWD_NORED=1): skip the dB/dC global reductions
};

// Grouped backward (vmb_selective_scan_bwd_grouped): G = ndesc <= 4 group descriptors; strides are the ScanBwdParams ones, shared by
// the groups, rows indexed inside the group.  Kept out of ScanBwdParams so that the flat kernels' parameter layout is unchanged.
struct ScanBwdGroups {
    int ndesc;
    ScanBwdGroupDesc grp[4];
    int64_t dB_bs, dB_ns, dC_bs, dC_ns;  // strides of every group's dB / dC (B,N,L) destination
};

// out_f32 / dout_f32 (16-bit dtype only): `out` / `dout` are fp32 (selective_scan_cuda_oflex).  They are launcher arguments, not
// parameter-block members, so that the kernels instantiated without them keep their parameter layout.
int scan_fwd_launch(const ScanFwdParams& p, int dtype, cudaStream_t stream, bool out_f32 = false);
bool scan_fwd_tma_pick(const ScanFwdParams& p, int& rb, int& ss);
int scan_fwd_tma_launch(const ScanFwdParams& p, int dtype, int rb, int ss, cudaStream_t stream, bool out_f32 = false);
int scan_bwd_launch(const ScanBwdParams& p, int dtype, cudaStream_t stream, bool dout_f32 = false);
bool scan_bwd_tma_pick(const ScanBwdParams& p, int dtype, int& rb, int& ss);
int scan_bwd_tma_launch(const ScanBwdParams& p, int dtype, int rb, int ss, cudaStream_t stream, bool dout_f32 = false);
int scan_bwd_grouped_launch(const ScanBwdParams& p, const ScanBwdGroups& gr, int dtype, cudaStream_t stream);

}  // namespace vmb
