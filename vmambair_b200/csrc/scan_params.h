// Internal parameter blocks of the selective-scan kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/vmambair_b200.h"

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

// z-gated flat forward (selective_scan_cuda): out_z = out * SiLU(z), both (batch, dim, L) in the input dtype, last stride 1.
struct ScanGateDesc {
    const void* z;
    void* out_z;
    int64_t z_bs, z_ds, oz_bs, oz_ds;
};

// Forward MODE flags on top of the base modes 0..3 (flat modes 0 / 1 only): kScanGate also stores out_z; kScanPairCkpt writes the
// checkpoints as (batch, dim, n_ckpt, 2 N) with h_n in slot 2n+1 and 0 in slot 2n, and row n_ckpt-1 always holds the last state.
constexpr int kScanGate = 4, kScanPairCkpt = 8;

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
    ScanGroupDesc grp[4];   // flat gated modes: the bytes of a ScanGateDesc (scan_gate_desc / set_scan_gate)
    int num_sms;
};

// The flat modes never read the group descriptors, so the gated ones carry their ScanGateDesc in that storage: the type of the
// parameter block, and with it the code of every kernel that does not gate, stays as it was.
static_assert(sizeof(ScanGateDesc) <= sizeof(ScanGroupDesc[4]), "the gate must fit in the group descriptors");
inline void set_scan_gate(ScanFwdParams& p, const ScanGateDesc& g) { memcpy(p.grp, &g, sizeof(g)); }
#ifdef __CUDACC__
__device__ __forceinline__ ScanGateDesc scan_gate_desc(const ScanFwdParams& p) {
    ScanGateDesc g;
    memcpy(&g, p.grp, sizeof(g));
    return g;
}
#endif

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
};

// Grouped backward (vmb_selective_scan_bwd_grouped): G = ndesc <= 4 group descriptors; strides are the ScanBwdParams ones, shared by
// the groups, rows indexed inside the group.  Kept out of ScanBwdParams so that the flat kernels' parameter layout is unchanged.
struct ScanBwdGroups {
    int ndesc;
    ScanBwdGroupDesc grp[4];
    int64_t dB_bs, dB_ns, dC_bs, dC_ns;  // strides of every group's dB / dC (B,N,L) destination
};

// Deterministic backward (det = true below): the workspace holds per-contributor partials instead of one atomically accumulated
// scratch, and scan_bwd_det_finalize sums them in a fixed order.  Layout, in fp32:
//   [nc][batch][G][npad/2][L][4]  dB/dC row sums of each contributor (nc = the CTAs / warps that share a (batch, group))
//   [batch][dim][N]  dA,  [batch][dim]  dD,  [batch][dim]  ddelta_bias  (one slot per (batch, row): written by one CTA)
// Every slot the finalize reads is written by the backward kernel, so nothing is zero-filled.
struct ScanBwdDetFin {
    const float4* bc;                 // dB/dC partials
    const float *pA, *pD, *pbias;     // parameter partials
    float *dA, *dD, *dbias;           // destinations: the sums over the batch are ADDED (accumulate-into contract)
    void *dB, *dC;                    // flat operator: (batch, G, N, L) contiguous
    int batch, dim, N, npad, G, L, nc;
};
inline int64_t scan_bwd_det_bytes(const ScanBwdParams& p, int nc) {
    return 16 * (int64_t)nc * p.batch * p.G * (p.npad / 2) * p.L + 4 * (int64_t)p.batch * p.dim * (p.N + 2);
}
// points p's accumulators at the partial slots of the workspace p.dBC; returns the finalize's view (the real destinations)
inline ScanBwdDetFin scan_bwd_det_carve(ScanBwdParams& p, int nc) {
    ScanBwdDetFin f{};
    float* ws = p.dBC;
    float* prm = ws + 4 * (int64_t)nc * p.batch * p.G * (p.npad / 2) * p.L;
    const int64_t rows = (int64_t)p.batch * p.dim;
    f.bc = reinterpret_cast<const float4*>(ws);
    f.pA = prm;
    f.pD = p.dD ? prm + rows * p.N : nullptr;
    f.pbias = p.dbias ? prm + rows * (p.N + 1) : nullptr;
    f.dA = p.dA; f.dD = p.dD; f.dbias = p.dbias; f.dB = p.dB; f.dC = p.dC;
    f.batch = p.batch; f.dim = p.dim; f.N = p.N; f.npad = p.npad; f.G = p.G; f.L = p.L; f.nc = nc;
    p.dA = prm;
    p.dD = const_cast<float*>(f.pD);
    p.dbias = const_cast<float*>(f.pbias);
    return f;
}
// gr: NULL for the flat operator, else the grouped destinations (each group's dB / dC in its memory order)
int scan_bwd_det_finalize(const ScanBwdDetFin& f, const ScanBwdGroups* gr, int dtype, cudaStream_t stream);
int64_t scan_bwd_det_workspace(const ScanBwdParams& p);
int64_t scan_bwd_grouped_det_workspace(const ScanBwdParams& p);

// out_f32 / dout_f32 (16-bit dtype only): `out` / `dout` are fp32 (selective_scan_cuda_oflex).  They are launcher arguments, not
// parameter-block members, so that the kernels instantiated without them keep their parameter layout.
// ext: kScanGate | kScanPairCkpt (launcher argument as well; kScanPairCkpt only with checkpoints, neither with out_f32 or groups).
int scan_fwd_launch(const ScanFwdParams& p, int dtype, cudaStream_t stream, bool out_f32 = false, int ext = 0);
bool scan_fwd_tma_pick(const ScanFwdParams& p, int& rb, int& ss);
int scan_fwd_tma_launch(const ScanFwdParams& p, int dtype, int rb, int ss, cudaStream_t stream, bool out_f32 = false, int ext = 0);
// elementwise backward of the z gate (vmb_scan_gate_bwd)
int scan_gate_bwd_launch(const vmb_scan_gate_args& a, bool vec_ok, cudaStream_t stream);
int scan_bwd_launch(const ScanBwdParams& p, int dtype, cudaStream_t stream, bool dout_f32 = false, bool det = false);
bool scan_bwd_tma_pick(const ScanBwdParams& p, int& rb, int& ss);
int scan_bwd_tma_launch(const ScanBwdParams& p, int dtype, int rb, int ss, cudaStream_t stream, bool dout_f32 = false, bool det = false);
int scan_bwd_grouped_launch(const ScanBwdParams& p, const ScanBwdGroups& gr, int dtype, cudaStream_t stream, bool det = false);

}  // namespace vmb
