// Two-direction channel selective scan as a standalone operator: cross_selective_scanC
// (RealSR/VmambaIR/archs/MambaRealSR11_arch.py:438-534; CrossScanC + x_proj / dt_proj einsums + SelectiveScan + CrossMergeC).
// One CTA per image does everything in shared memory, in fp32:
//   xs_0 = x (D, L), xs_1 = flip_L(x);  x_dbl_k = W_k xs_k (+ b_k);  dt_k = softplus?(Wdt_k x_dbl_k[:R] + dt_bias_k)
//   y_k = selective scan of (xs_k, dt_k, A_k = -exp(A_logs_k), B = x_dbl_k[R:R+N], C = x_dbl_k[R+N:], D_k)
//   y = y_0 + flip_L(y_1), stored (L, D) per image.
// The R dt-rank rows of x_dbl are folded into dt as soon as they are formed (and recomputed from x in the backward), so only the B
// and C rows stay resident: [2][2N][L] plus, in the backward, the (2D, N, L) state history and the (2, N, L) dC rows.
// The backward writes every parameter gradient per image into a workspace (no atomics); a second kernel sums the images in a fixed
// order, so gradients are bitwise reproducible.
#include "common.cuh"

namespace vmb {

constexpr int CSC_THREADS = 512;  // the scan runs one thread per (row, state): 2 D 16 <= CSC_THREADS
constexpr int CSC_MAX_SMEM = 227 * 1024;

struct CscParams {
    const void* x;
    const float* xw;   // (2, R+2N, D)
    const float* xb;   // (2, R+2N) or null
    const float* dtw;  // (2, D, R)
    const float* dtb;  // (2D)
    const float* A_logs;  // (2D, N)
    const float* Ds;   // (2D)
    float* y;          // fwd: (B, L, D)
    const float* dy;   // bwd: (B, L, D)
    void* dx;          // bwd: (B, D, L) dense, x's dtype
    float* part;       // bwd: (B, P) per-image parameter gradients
    float* dparams;    // bwd: (P) their sum over the batch
    int B, D, L, R, N;
    int64_t x_bs, x_ds;
    int softplus;
};

// packed parameter-gradient layout (fp32): x_proj_weight, x_proj_bias, dt_projs_weight, dt_projs_bias, A_logs, Ds
struct CscOffsets {
    int xw, xb, dtw, dtb, A, Ds, total;
    __host__ __device__ CscOffsets(int D, int R, int N) {
        const int RN = R + 2 * N;
        xw = 0;
        xb = xw + 2 * RN * D;
        dtw = xb + 2 * RN;
        dtb = dtw + 2 * D * R;
        A = dtb + 2 * D;
        Ds = A + 2 * D * N;
        total = Ds + 2 * D;
    }
};

static int64_t csc_fwd_floats(int D, int L, int R, int N) {
    const int64_t RN = R + 2 * N, LP = L | 1;
    return 2 * RN * D + 2 * RN + 2 * (int64_t)D * R + 4 * (int64_t)D   // parameters
           + (int64_t)D * L                                             // x
           + 4 * N * LP                                                 // B / C rows of both directions
           + 2 * (int64_t)D * L;                                        // dt (forward: later y)
}
static int64_t csc_bwd_floats(int D, int L, int R, int N) {
    const int64_t LP = L | 1;
    return csc_fwd_floats(D, L, R, N) + 2 * (int64_t)D * N * LP  // state history, later the per-row dB terms
           + 2 * N * LP                                           // dC
           + 4 * (int64_t)D * L;                                  // dy (later d pre-softplus dt), du
}

struct CscSmem {
    float *W, *Xb, *Wdt, *Dtb, *Dsv, *X, *BC, *Dt;
    int RN, LP;
};

__device__ __forceinline__ float csc_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// the forward up to the scan: parameters and x into shared memory, B / C rows, dt.  Ends with __syncthreads().
template <typename T>
__device__ __forceinline__ CscSmem csc_prologue(const CscParams& p, float* sm) {
    const int D = p.D, L = p.L, R = p.R, N = p.N, RN = R + 2 * N, LP = L | 1, tid = threadIdx.x, b = blockIdx.x;
    CscSmem s;
    s.RN = RN;
    s.LP = LP;
    s.W = sm;                     // [2][RN][D]
    s.Xb = s.W + 2 * RN * D;      // [2][RN]
    s.Wdt = s.Xb + 2 * RN;        // [2][D][R]
    s.Dtb = s.Wdt + 2 * D * R;    // [2D]
    s.Dsv = s.Dtb + 2 * D;        // [2D]
    s.X = s.Dsv + 2 * D;          // [D][L] x, natural order
    s.BC = s.X + D * L;           // [2][2N][LP] B rows then C rows of each direction, sequence order
    s.Dt = s.BC + 4 * N * LP;     // [2D][L] dt, sequence order
    for (int i = tid; i < 2 * RN * D; i += CSC_THREADS) s.W[i] = p.xw[i];
    for (int i = tid; i < 2 * RN; i += CSC_THREADS) s.Xb[i] = p.xb ? p.xb[i] : 0.f;
    for (int i = tid; i < 2 * D * R; i += CSC_THREADS) s.Wdt[i] = p.dtw[i];
    for (int i = tid; i < 2 * D; i += CSC_THREADS) {
        s.Dtb[i] = p.dtb[i];
        s.Dsv[i] = p.Ds[i];
    }
    const T* __restrict__ xg = static_cast<const T*>(p.x) + (int64_t)b * p.x_bs;
    for (int i = tid; i < D * L; i += CSC_THREADS) {
        const int d = i / L, l = i - d * L;
        s.X[i] = to_f32<T>(xg[(int64_t)d * p.x_ds + l]);
    }
    __syncthreads();
    // B / C rows: x_dbl[k][R + c][l] = b[k][R + c] + sum_d W[k][R + c][d] xs_k[d][l]
    for (int i = tid; i < 4 * N * L; i += CSC_THREADS) {
        const int kc = i / L, l = i - kc * L, k = kc / (2 * N), c = kc - k * 2 * N;
        const int lm = k ? L - 1 - l : l;
        const float* w = s.W + (k * RN + R + c) * D;
        float v = s.Xb[k * RN + R + c];
        for (int d = 0; d < D; ++d) v = fmaf(w[d], s.X[d * L + lm], v);
        s.BC[kc * LP + l] = v;
    }
    // dt[k][d][l] = softplus?(dt_bias[k][d] + sum_r Wdt[k][d][r] x_dbl[k][r][l])
    for (int i = tid; i < 2 * D * L; i += CSC_THREADS) {
        const int row = i / L, l = i - row * L, k = row / D;
        const int lm = k ? L - 1 - l : l;
        float pre = s.Dtb[row];
        for (int r = 0; r < R; ++r) {
            const float* w = s.W + (k * RN + r) * D;
            float v = s.Xb[k * RN + r];
            for (int d = 0; d < D; ++d) v = fmaf(w[d], s.X[d * L + lm], v);
            pre = fmaf(s.Wdt[row * R + r], v, pre);
        }
        s.Dt[i] = p.softplus ? softplus_f(pre) : pre;
    }
    __syncthreads();
    return s;
}

template <typename T>
__global__ void __launch_bounds__(CSC_THREADS) cross_scan_c_fwd_kernel(const CscParams p) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float sm[];
    const CscSmem s = csc_prologue<T>(p, sm);
    const int D = p.D, L = p.L, N = p.N, LP = s.LP, tid = threadIdx.x, b = blockIdx.x;
    const int row = tid >> 4, n = tid & 15, rows = 2 * D;
    // sequential scan, thread = (row, state); rows * 16 is a multiple of 32, so every warp is either wholly in or wholly out
    if (row < rows) {
        const int k = row / D, d = row - k * D;
        const bool act = n < N;
        const float A2 = act ? -__expf(p.A_logs[row * N + n]) * kLog2e : 0.f;
        const float Dv = s.Dsv[row];
        const float* __restrict__ Br = s.BC + (k * 2 * N + (act ? n : 0)) * LP;
        const float* __restrict__ Cr = s.BC + (k * 2 * N + N + (act ? n : 0)) * LP;
        const float* __restrict__ ur = s.X + d * L;
        float* dtr = s.Dt + row * L;  // dt[l] is replaced by y[l] once step l has read it
        float h = 0.f;
        for (int l = 0; l < L; ++l) {
            const float dt = dtr[l], u = ur[k ? L - 1 - l : l];
            h = fmaf(ex2(dt * A2), h, act ? dt * u * Br[l] : 0.f);
            float t = act ? h * Cr[l] : 0.f;
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o, 16);
            __syncwarp();
            if (n == 0) dtr[l] = fmaf(Dv, u, t);
        }
    }
    __syncthreads();
    // merge: y[l][d] = y_0[d][l] + y_1[d][L-1-l]
    float* __restrict__ yg = p.y + (int64_t)b * L * D;
    for (int i = tid; i < L * D; i += CSC_THREADS) {
        const int l = i / D, d = i - l * D;
        yg[i] = s.Dt[d * L + l] + s.Dt[(D + d) * L + (L - 1 - l)];
    }
}

template <typename T>
__global__ void __launch_bounds__(CSC_THREADS) cross_scan_c_bwd_kernel(const CscParams p) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ float sm[];
    const CscSmem s = csc_prologue<T>(p, sm);
    const int D = p.D, L = p.L, R = p.R, N = p.N, RN = s.RN, LP = s.LP, tid = threadIdx.x, b = blockIdx.x;
    const int warp = tid >> 5, lane = tid & 31, rows = 2 * D;
    constexpr int NW = CSC_THREADS / 32;
    float* sH = s.Dt + 2 * D * L;    // [2D][N][LP] h_l; during the reverse scan replaced by the per-row dB terms dh dt u
    float* sDC = sH + 2 * D * N * LP;  // [2][N][LP] dC = sum_d dy h
    float* sDy = sDC + 2 * N * LP;     // [2D][L] dy (sequence order); later d(pre-softplus dt)
    float* sDu = sDy + 2 * D * L;      // [2D][L] du (sequence order)
    const CscOffsets off(D, R, N);
    float* __restrict__ part = p.part + (int64_t)b * off.total;
    const int srow = tid >> 4, n = tid & 15;
    const bool sact = srow < rows && n < N;
    const float Araw = sact ? -__expf(p.A_logs[srow * N + n]) : 0.f;
    const float A2 = Araw * kLog2e;
    // ---- forward scan, keeping every h_l
    if (srow < rows) {
        const int k = srow / D, d = srow - k * D;
        const float* __restrict__ dtr = s.Dt + srow * L;
        const float* __restrict__ ur = s.X + d * L;
        const float* __restrict__ Br = s.BC + (k * 2 * N + (sact ? n : 0)) * LP;
        float* __restrict__ hh = sH + (srow * N + (sact ? n : 0)) * LP;
        float h = 0.f;
        for (int l = 0; l < L; ++l) {
            const float dt = dtr[l], u = ur[k ? L - 1 - l : l];
            h = fmaf(ex2(dt * A2), h, sact ? dt * u * Br[l] : 0.f);
            if (sact) hh[l] = h;
        }
    }
    // dy in sequence order: dy_0[d][l] = g[l][d], dy_1[d][l] = g[L-1-l][d]
    const float* __restrict__ dyg = p.dy + (int64_t)b * L * D;
    for (int i = tid; i < 2 * D * L; i += CSC_THREADS) {
        const int row = i / L, l = i - row * L, k = row / D, d = row - k * D;
        sDy[i] = dyg[(k ? L - 1 - l : l) * D + d];
    }
    __syncthreads();
    // dC[k][n][l] = sum_d dy_k[d][l] h_k,d[n][l];  dD[row] = sum_l dy u
    for (int i = tid; i < 2 * N * L; i += CSC_THREADS) {
        const int kn = i / L, l = i - kn * L, k = kn / N, nn = kn - k * N;
        float v = 0.f;
        for (int d = 0; d < D; ++d) v = fmaf(sDy[(k * D + d) * L + l], sH[((k * D + d) * N + nn) * LP + l], v);
        sDC[kn * LP + l] = v;
    }
    for (int row = warp; row < rows; row += NW) {
        const int k = row / D, d = row - k * D;
        float acc = 0.f;
        for (int l = lane; l < L; l += 32) acc = fmaf(sDy[row * L + l], s.X[d * L + (k ? L - 1 - l : l)], acc);
        acc = csc_warp_sum(acc);
        if (lane == 0) part[off.Ds + row] = acc;
    }
    __syncthreads();
    // ---- reverse scan, thread = (row, state):  dh_l = C_l dy_l + a_{l+1} dh_{l+1},  a_l = exp(dt_l A)
    if (srow < rows) {
        const int k = srow / D, d = srow - k * D;
        const float* __restrict__ dtr = s.Dt + srow * L;
        const float* __restrict__ ur = s.X + d * L;
        const float* __restrict__ Br = s.BC + (k * 2 * N + (sact ? n : 0)) * LP;
        const float* __restrict__ Cr = s.BC + (k * 2 * N + N + (sact ? n : 0)) * LP;
        float* __restrict__ hh = sH + (srow * N + (sact ? n : 0)) * LP;
        float* dyr = sDy + srow * L;  // dy[l] is replaced by d(pre-softplus dt)[l] once step l has read it
        float* dur = sDu + srow * L;
        const float Dv = s.Dsv[srow];
        float dh = 0.f, a_next = 0.f, dA = 0.f;
        for (int l = L - 1; l >= 0; --l) {
            const float dt = dtr[l], u = ur[k ? L - 1 - l : l], dy = dyr[l];
            const float a = ex2(dt * A2);
            const float hprev = sact && l > 0 ? hh[l - 1] : 0.f;
            dh = sact ? fmaf(a_next, dh, Cr[l] * dy) : 0.f;
            a_next = a;
            const float g = a * hprev;
            float t1 = sact ? dh * Br[l] : 0.f;     // -> sum_n dh B
            float t2 = sact ? Araw * dh * g : 0.f;  // -> sum_n dh A a h_{l-1}
            dA = fmaf(dh * dt, g, dA);
            if (sact) hh[l] = dh * dt * u;  // dB term of this row (h_l is not read again)
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) {
                t1 += __shfl_xor_sync(0xffffffffu, t1, o, 16);
                t2 += __shfl_xor_sync(0xffffffffu, t2, o, 16);
            }
            __syncwarp();
            if (n == 0) {
                const float ddt = fmaf(u, t1, t2);
                dyr[l] = p.softplus ? ddt * (1.f - ex2(-dt * kLog2e)) : ddt;  // softplus' = sigmoid(pre) = 1 - exp(-softplus(pre))
                dur[l] = fmaf(dt, t1, Dv * dy);
            }
        }
        if (sact) part[off.A + srow * N + n] = dA * Araw;  // d/dA_log = A d/dA
    }
    __syncthreads();
    // d x_dbl of the B / C rows (in place of the B / C values): dB = sum_d dB terms, dC
    for (int i = tid; i < 2 * N * L; i += CSC_THREADS) {
        const int kn = i / L, l = i - kn * L, k = kn / N, nn = kn - k * N;
        float v = 0.f;
        for (int d = 0; d < D; ++d) v += sH[((k * D + d) * N + nn) * LP + l];
        s.BC[(k * 2 * N + nn) * LP + l] = v;
        s.BC[(k * 2 * N + N + nn) * LP + l] = sDC[kn * LP + l];
    }
    // dt_projs: d bias[row] = sum_l dpre;  d Wdt[k][d][r] = sum_l dpre[k][d][l] x_dbl[k][r][l] (x_dbl recomputed from x)
    for (int row = warp; row < rows; row += NW) {
        float acc = 0.f;
        for (int l = lane; l < L; l += 32) acc += sDy[row * L + l];
        acc = csc_warp_sum(acc);
        if (lane == 0) part[off.dtb + row] = acc;
    }
    for (int t = warp; t < rows * R; t += NW) {
        const int row = t / R, r = t - row * R, k = row / D;
        const float* w = s.W + (k * RN + r) * D;
        const float xb = s.Xb[k * RN + r];
        float acc = 0.f;
        for (int l = lane; l < L; l += 32) {
            const int lm = k ? L - 1 - l : l;
            float v = xb;
            for (int d = 0; d < D; ++d) v = fmaf(w[d], s.X[d * L + lm], v);
            acc = fmaf(sDy[row * L + l], v, acc);
        }
        acc = csc_warp_sum(acc);
        if (lane == 0) part[off.dtw + t] = acc;
    }
    __syncthreads();
    // d x_dbl[k][c][l]: c < R: sum_d Wdt[k][d][c] dpre[k][d][l];  else the B / C rows above
    auto ddbl = [&](int k, int c, int l) -> float {
        if (c >= R) return s.BC[(k * 2 * N + c - R) * LP + l];
        float v = 0.f;
        for (int d = 0; d < D; ++d) v = fmaf(s.Wdt[(k * D + d) * R + c], sDy[(k * D + d) * L + l], v);
        return v;
    };
    // x_proj: dW[k][c][d] = sum_l ddbl xs_k[d][l];  d bias[k][c] = sum_l ddbl
    for (int t = warp; t < 2 * RN * (D + 1); t += NW) {
        const int kc = t / (D + 1), d = t - kc * (D + 1), k = kc / RN, c = kc - k * RN;  // d == D: the bias
        float acc = 0.f;
        for (int l = lane; l < L; l += 32) {
            const float g = ddbl(k, c, l);
            acc = d < D ? fmaf(g, s.X[d * L + (k ? L - 1 - l : l)], acc) : acc + g;
        }
        acc = csc_warp_sum(acc);
        if (lane == 0) {
            if (d < D) part[off.xw + kc * D + d] = acc;
            else part[off.xb + kc] = acc;
        }
    }
    // dx[d][l] = sum_k (du_k + W_k^T ddbl_k)[d][position of l in direction k]
    T* __restrict__ dxg = static_cast<T*>(p.dx) + (int64_t)b * D * L;
    for (int i = tid; i < D * L; i += CSC_THREADS) {
        const int d = i / L, l = i - d * L;
        float v = 0.f;
        for (int k = 0; k < 2; ++k) {
            const int ls = k ? L - 1 - l : l;
            float a = sDu[(k * D + d) * L + ls];
            for (int c = 0; c < RN; ++c) a = fmaf(s.W[(k * RN + c) * D + d], ddbl(k, c, ls), a);
            v += a;
        }
        dxg[i] = from_f32<T>(v);
    }
}

// dparams[i] = sum_b part[b][i], images in order: bitwise reproducible
__global__ void __launch_bounds__(256) cross_scan_c_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, int B, int P) {
    pdl_trigger();
    pdl_wait();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += part[(int64_t)b * P + i];
    out[i] = s;
}

static int csc_check(const vmb_cross_scan_c_args* a, const char* who) {
    VMB_CHECK(a && a->x && a->x_proj_weight && a->dt_projs_weight && a->dt_projs_bias && a->A_logs && a->Ds,
              "%s: null pointer", who);
    VMB_CHECK(a->batch > 0 && a->D > 0 && a->L > 0 && a->R > 0 && a->N > 0, "%s: bad sizes", who);
    VMB_CHECK(a->N <= 16 && 2 * a->D * 16 <= CSC_THREADS, "%s: needs d_state <= 16 and D <= %d (got D=%d, N=%d)", who,
              CSC_THREADS / 32, a->D, a->N);
    VMB_CHECK(a->dtype == VMB_F32 || a->dtype == VMB_BF16 || a->dtype == VMB_F16, "%s: bad dtype %d", who, a->dtype);
    VMB_CHECK(4 * csc_bwd_floats(a->D, a->L, a->R, a->N) <= CSC_MAX_SMEM, "%s: D=%d L=%d R=%d N=%d needs %lld B of shared memory (> %d)",
              who, a->D, a->L, a->R, a->N, (long long)(4 * csc_bwd_floats(a->D, a->L, a->R, a->N)), CSC_MAX_SMEM);
    return VMB_OK;
}

static CscParams csc_params(const vmb_cross_scan_c_args* a) {
    CscParams p{};
    p.x = a->x; p.xw = a->x_proj_weight; p.xb = a->x_proj_bias; p.dtw = a->dt_projs_weight; p.dtb = a->dt_projs_bias;
    p.A_logs = a->A_logs; p.Ds = a->Ds; p.y = a->y;
    p.B = a->batch; p.D = a->D; p.L = a->L; p.R = a->R; p.N = a->N;
    p.x_bs = a->x_bs; p.x_ds = a->x_ds; p.softplus = a->delta_softplus;
    return p;
}

template <typename K>
static int csc_launch(K kern, const CscParams& p, size_t smem, cudaStream_t st) {
    if (smem > 48 * 1024) VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    VMB_CUDA(launch_pdl(kern, dim3(p.B), dim3(CSC_THREADS), smem, st, p));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

}  // namespace vmb

using namespace vmb;

extern "C" int64_t vmb_cross_selective_scan_c_smem_bytes(int D, int L, int R, int N) {
    if (D <= 0 || L <= 0 || R <= 0 || N <= 0 || N > 16 || 2 * D * 16 > CSC_THREADS) return -1;
    return 4 * csc_bwd_floats(D, L, R, N);
}

extern "C" int64_t vmb_cross_selective_scan_c_workspace_bytes(int batch, int D, int R, int N) {
    return 4 * (int64_t)batch * CscOffsets(D, R, N).total;
}

extern "C" int vmb_cross_selective_scan_c_fwd(const vmb_cross_scan_c_args* a, void* stream) {
    if (int e = csc_check(a, "cross_selective_scan_c_fwd")) return e;
    VMB_CHECK(a->y, "cross_selective_scan_c_fwd: null y");
    const CscParams p = csc_params(a);
    const size_t smem = 4 * csc_fwd_floats(a->D, a->L, a->R, a->N);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    switch (a->dtype) {
        case VMB_F32: return csc_launch(cross_scan_c_fwd_kernel<float>, p, smem, st);
        case VMB_BF16: return csc_launch(cross_scan_c_fwd_kernel<__nv_bfloat16>, p, smem, st);
        default: return csc_launch(cross_scan_c_fwd_kernel<__half>, p, smem, st);
    }
}

extern "C" int vmb_cross_selective_scan_c_bwd(const vmb_cross_scan_c_bwd_args* a, void* stream) {
    VMB_CHECK(a, "cross_selective_scan_c_bwd: null args");
    if (int e = csc_check(&a->fwd, "cross_selective_scan_c_bwd")) return e;
    VMB_CHECK(a->dy && a->dx && a->d_params && a->workspace, "cross_selective_scan_c_bwd: null pointer");
    CscParams p = csc_params(&a->fwd);
    p.y = nullptr;
    p.dy = a->dy; p.dx = a->dx; p.part = a->workspace; p.dparams = a->d_params;
    const size_t smem = 4 * csc_bwd_floats(p.D, p.L, p.R, p.N);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int e;
    switch (a->fwd.dtype) {
        case VMB_F32: e = csc_launch(cross_scan_c_bwd_kernel<float>, p, smem, st); break;
        case VMB_BF16: e = csc_launch(cross_scan_c_bwd_kernel<__nv_bfloat16>, p, smem, st); break;
        default: e = csc_launch(cross_scan_c_bwd_kernel<__half>, p, smem, st); break;
    }
    if (e) return e;
    const int P = CscOffsets(p.D, p.R, p.N).total;
    VMB_CUDA(launch_pdl(cross_scan_c_reduce_kernel, dim3(cdiv(P, 256)), dim3(256), 0, st, (const float*)p.part, p.dparams, p.B, P));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}
