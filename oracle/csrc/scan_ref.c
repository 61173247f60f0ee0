/* CPU oracle for the selective-scan operator -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C restatement (sequential recurrence, one (b,d) row at a time) of the
 * reference's selective_scan_ref
 * (Mamba/kernels/selective_scan/test_selective_scan.py:168-234) and of the
 * analytic backward evaluated by the reference bwd kernel
 * (csrc/selective_scan/cus/selective_scan_bwd_kernel.cuh:139-241).
 * Used by tests/ (checker), __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference leg.  Never linked into the product library.
 *
 * Layouts (all contiguous, fp32):  u,delta,out,dout: (B,D,L)   A: (D,N)
 *   Bm,Cm: (B,G,N,L)   Dv,bias: (D) or NULL.   Rows are independent -> OpenMP.
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif
/* torchrun exports OMP_NUM_THREADS=1; the CPU baseline must use every host core it can */
void scan_ref_set_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

static inline float softplus_f(float x) { return x <= 20.f ? log1pf(expf(x)) : x; }
static inline double softplus_d(double x) { return x <= 20.0 ? log1p(exp(x)) : x; }

/* fp32 sequential forward (the reference oracle is fp32 throughout). */
void scan_ref_fwd_f32(const float *u, const float *delta, const float *A,
                      const float *Bm, const float *Cm, const float *Dv,
                      const float *bias, int softplus, float *out,
                      float *last_state /* (B,D,N) or NULL */,
                      int Bsz, int D, int L, int N, int G) {
    const int rep = D / G;
#pragma omp parallel for collapse(2) schedule(static)
    for (int b = 0; b < Bsz; ++b)
        for (int d = 0; d < D; ++d) {
            const float *ur = u + ((size_t)b * D + d) * L;
            const float *dr = delta + ((size_t)b * D + d) * L;
            float *orow = out + ((size_t)b * D + d) * L;
            const int g = d / rep;
            const float *Bg = Bm + ((size_t)b * G + g) * N * L;
            const float *Cg = Cm + ((size_t)b * G + g) * N * L;
            const float *Ar = A + (size_t)d * N;
            float h[256];
            for (int n = 0; n < N; ++n) h[n] = 0.f;
            const float bi = bias ? bias[d] : 0.f;
            const float Dd = Dv ? Dv[d] : 0.f;
            for (int l = 0; l < L; ++l) {
                float dt = dr[l] + bi;
                if (softplus) dt = softplus_f(dt);
                const float dtu = dt * ur[l];
                float y = 0.f;
                for (int n = 0; n < N; ++n) {
                    h[n] = expf(dt * Ar[n]) * h[n] + dtu * Bg[(size_t)n * L + l];
                    y += h[n] * Cg[(size_t)n * L + l];
                }
                orow[l] = Dv ? y + ur[l] * Dd : y;
            }
            if (last_state)
                for (int n = 0; n < N; ++n) last_state[((size_t)b * D + d) * N + n] = h[n];
        }
}

/* Relative-error multiplier of dt in units of the rounding: 1 + |x| with the softplus (exp(-|x|) and the log carry errors that
 * grow with |x|, and the bias addition that cancels as much), 1 without it. */
static inline double dt_mult(int softplus, double x) { return softplus ? 1.0 + fabs(x) : 1.0; }

/* fp64 forward; with Sout != NULL also the magnitude S of every output (scan_bound.py):
 *   Mh[l] = a_l Mh[l-1] + |b_l|                                            (b_l = dt u B, a_l = exp(x_l), x_l = dt A)
 *   Sh[l] = a_l Sh[l-1] + (1 + r_l |x_l|) a_l Mh[l-1] + r_l |b_l|          (r_l = dt_mult)
 *   S_out = sum_n |C| (Sh + Mh) + |D u|
 * Mh is the sum of the absolute terms of h, Sh how far an fp32 evaluation of h may drift, in units of the rounding. */
static void fwd_core(const float *u, const float *delta, const float *A, const float *Bm, const float *Cm, const float *Dv,
                     const float *bias, int softplus, double *out, double *Sout, int Bsz, int D, int L, int N, int G) {
    const int rep = D / G;
#pragma omp parallel for collapse(2) schedule(static)
    for (int b = 0; b < Bsz; ++b)
        for (int d = 0; d < D; ++d) {
            const float *ur = u + ((size_t)b * D + d) * L;
            const float *dr = delta + ((size_t)b * D + d) * L;
            double *orow = out + ((size_t)b * D + d) * L;
            double *srow = Sout ? Sout + ((size_t)b * D + d) * L : NULL;
            const int g = d / rep;
            const float *Bg = Bm + ((size_t)b * G + g) * N * L;
            const float *Cg = Cm + ((size_t)b * G + g) * N * L;
            const float *Ar = A + (size_t)d * N;
            double h[256], Mh[256], Sh[256];
            for (int n = 0; n < N; ++n) h[n] = Mh[n] = Sh[n] = 0.0;
            const double bi = bias ? bias[d] : 0.0;
            const double Dd = Dv ? Dv[d] : 0.0;
            for (int l = 0; l < L; ++l) {
                double dt = (double)dr[l] + bi;
                const double r = dt_mult(softplus, dt);
                if (softplus) dt = softplus_d(dt);
                const double dtu = dt * ur[l];
                double y = 0.0, s = 0.0;
                for (int n = 0; n < N; ++n) {
                    const double a = exp(dt * Ar[n]);
                    h[n] = a * h[n] + dtu * Bg[(size_t)n * L + l];
                    y += h[n] * Cg[(size_t)n * L + l];
                    if (srow) {
                        const double bl = fabs(dtu * Bg[(size_t)n * L + l]);
                        Sh[n] = a * Sh[n] + (1.0 + r * fabs(dt * Ar[n])) * a * Mh[n] + r * bl;
                        Mh[n] = a * Mh[n] + bl;
                        s += fabs((double)Cg[(size_t)n * L + l]) * (Sh[n] + Mh[n]);
                    }
                }
                orow[l] = y + ur[l] * Dd;
                if (srow) srow[l] = s + fabs(ur[l] * Dd);
            }
        }
}

/* fp64-internal forward ("ground truth" to show both fp32 results are equidistant). */
void scan_ref_fwd_f64(const float *u, const float *delta, const float *A,
                      const float *Bm, const float *Cm, const float *Dv,
                      const float *bias, int softplus, double *out,
                      int Bsz, int D, int L, int N, int G) {
    fwd_core(u, delta, A, Bm, Cm, Dv, bias, softplus, out, NULL, Bsz, D, L, N, G);
}

/* scan_ref_fwd_f64 + the magnitude S (B,D,L) of each output */
void scan_ref_fwd_mag(const float *u, const float *delta, const float *A, const float *Bm, const float *Cm, const float *Dv,
                      const float *bias, int softplus, double *out, double *Sout, int Bsz, int D, int L, int N, int G) {
    fwd_core(u, delta, A, Bm, Cm, Dv, bias, softplus, out, Sout, Bsz, D, L, N, G);
}

/* Magnitudes of the backward (all NULL: values only).  Same layouts as the gradients; every one must be zero-initialised. */
typedef struct { double *du, *ddelta, *dA, *dB, *dC, *dD, *dbias; } BwdMag;

/* Analytic backward, fp64 internal, fp64 outputs; with m != NULL also the magnitude S of every gradient (scan_bound.py).  The
 * adjoint dh[l] = a_{l+1} dh[l+1] + C_l dout_l takes the forward's Mh / Sh recurrences (fwd_core) in reverse:
 *   Mdh[l] = a_{l+1} Mdh[l+1] + |C dout|
 *   Sdh[l] = a_{l+1} Sdh[l+1] + (1 + r_{l+1} |x_{l+1}|) a_{l+1} Mdh[l+1] + |C dout|
 * and each term e * f of a gradient adds Se |f| + |e| Sf, with |h| + |b| for the h - b factor (a kernel may form it with
 * cancellation, or as a h_{l-1}):
 *   du     |D dout| + sum_n (Sdh + r Mdh) |B| dt
 *   ddelta sum_n Sdh Mv + Mdh (Mv + |A| (Sh + (1 + r)(Mh + |b|))),  Mv = |u B| + |A| (Mh + |b|);  with the softplus, times
 *          sigmoid(x), plus (2 + r dt) times the same sum over Mdh Mv: 1 - exp(-dt), the sigmoid's usual fp32 form, errs by a
 *          few roundings absolute, not relative
 *   dA     sum Sdh dt (Mh + |b|) + Mdh dt (Sh + (1 + r)(Mh + |b|))
 *   dB     sum (Sdh + r Mdh) dt |u|          dC  sum |dout| (Sh + Mh)          dD  sum |dout u|          dbias  sum S_ddelta
 * du,ddelta: (B,D,L); dA: (D,N); dB,dC: (B,G,N,L); dD,dbias: (D) (may be NULL).
 * All outputs must be zero-initialised by the caller. */
static void bwd_core(const float *u, const float *delta, const float *A, const float *Bm, const float *Cm, const float *Dv,
                     const float *bias, int softplus, const float *dout, double *du, double *ddelta, double *dA, double *dB,
                     double *dC, double *dD, double *dbias, const BwdMag *m, int Bsz, int D, int L, int N, int G) {
    const int rep = D / G;
    /* parallel over (b, g): rows of one group write the same dB/dC slab. */
#pragma omp parallel
    {
        double *hs = (double *)malloc(sizeof(double) * (size_t)N * L);
        double *dts = (double *)malloc(sizeof(double) * (size_t)L);
        double *dA_loc = (double *)calloc((size_t)D * N, sizeof(double));
        double *dD_loc = (double *)calloc((size_t)D, sizeof(double));
        double *db_loc = (double *)calloc((size_t)D, sizeof(double));
        double *Mhs = m ? (double *)malloc(sizeof(double) * (size_t)N * L) : NULL;
        double *Shs = m ? (double *)malloc(sizeof(double) * (size_t)N * L) : NULL;
        double *rs = m ? (double *)malloc(sizeof(double) * (size_t)L) : NULL;
        double *SdA_loc = m ? (double *)calloc((size_t)D * N, sizeof(double)) : NULL;
        double *SdD_loc = m ? (double *)calloc((size_t)D, sizeof(double)) : NULL;
        double *Sdb_loc = m ? (double *)calloc((size_t)D, sizeof(double)) : NULL;
#pragma omp for collapse(2) schedule(static)
        for (int b = 0; b < Bsz; ++b)
            for (int g = 0; g < G; ++g) {
                const float *Bg = Bm + ((size_t)b * G + g) * N * L;
                const float *Cg = Cm + ((size_t)b * G + g) * N * L;
                double *dBg = dB + ((size_t)b * G + g) * N * L;
                double *dCg = dC + ((size_t)b * G + g) * N * L;
                double *SdBg = m ? m->dB + ((size_t)b * G + g) * N * L : NULL;
                double *SdCg = m ? m->dC + ((size_t)b * G + g) * N * L : NULL;
                for (int d = g * rep; d < (g + 1) * rep; ++d) {
                    const float *ur = u + ((size_t)b * D + d) * L;
                    const float *dr = delta + ((size_t)b * D + d) * L;
                    const float *gor = dout + ((size_t)b * D + d) * L;
                    double *dur = du + ((size_t)b * D + d) * L;
                    double *ddr = ddelta + ((size_t)b * D + d) * L;
                    const float *Ar = A + (size_t)d * N;
                    const double bi = bias ? bias[d] : 0.0;
                    const double Dd = Dv ? Dv[d] : 0.0;
                    double h[256], dh[256], Mh[256], Sh[256], Mdh[256], Sdh[256];
                    for (int n = 0; n < N; ++n) { h[n] = 0.0; dh[n] = 0.0; Mh[n] = Sh[n] = Mdh[n] = Sdh[n] = 0.0; }
                    for (int l = 0; l < L; ++l) {
                        double dt = (double)dr[l] + bi;
                        if (m) rs[l] = dt_mult(softplus, dt);
                        if (softplus) dt = softplus_d(dt);
                        dts[l] = dt;
                        for (int n = 0; n < N; ++n) {
                            h[n] = exp(dt * Ar[n]) * h[n] + dt * ur[l] * Bg[(size_t)n * L + l];
                            hs[(size_t)n * L + l] = h[n];
                            if (m) {
                                const double a = exp(dt * Ar[n]), bl = fabs(dt * ur[l] * Bg[(size_t)n * L + l]);
                                Sh[n] = a * Sh[n] + (1.0 + rs[l] * fabs(dt * Ar[n])) * a * Mh[n] + rs[l] * bl;
                                Mh[n] = a * Mh[n] + bl;
                                Shs[(size_t)n * L + l] = Sh[n];
                                Mhs[(size_t)n * L + l] = Mh[n];
                            }
                        }
                    }
                    for (int l = L - 1; l >= 0; --l) {
                        const double dt = dts[l], ul = ur[l], go = gor[l];
                        double du_acc = Dd * go, ddt_acc = 0.0;
                        double Sdu = fabs(Dd * go), Sdt = 0.0, Mdt = 0.0;
                        for (int n = 0; n < N; ++n) {
                            if (m) {
                                const double cg = fabs((double)Cg[(size_t)n * L + l] * go);
                                if (l + 1 < L) {
                                    const double a = exp(dts[l + 1] * Ar[n]);
                                    Sdh[n] = a * Sdh[n] + (1.0 + rs[l + 1] * fabs(dts[l + 1] * Ar[n])) * a * Mdh[n];
                                    Mdh[n] = a * Mdh[n];
                                }
                                Sdh[n] += cg;
                                Mdh[n] += cg;
                            }
                            if (l + 1 < L) dh[n] *= exp(dts[l + 1] * Ar[n]);
                            dh[n] += (double)Cg[(size_t)n * L + l] * go;
                            const double Bv = Bg[(size_t)n * L + l];
                            const double hl = hs[(size_t)n * L + l];
                            const double bl = dt * ul * Bv;
                            du_acc += dh[n] * Bv * dt;
                            ddt_acc += dh[n] * (ul * Bv + Ar[n] * (hl - bl));
                            dA_loc[(size_t)d * N + n] += dh[n] * dt * (hl - bl);
                            dBg[(size_t)n * L + l] += dh[n] * dt * ul;
                            dCg[(size_t)n * L + l] += go * hl;
                            if (m) {
                                const double r = rs[l], Mhl = Mhs[(size_t)n * L + l], Shl = Shs[(size_t)n * L + l];
                                const double hb = Mhl + fabs(bl), Shb = Shl + (1.0 + r) * hb, aA = fabs((double)Ar[n]);
                                const double Mv = fabs(ul * Bv) + aA * hb;
                                Sdu += (Sdh[n] + r * Mdh[n]) * fabs(Bv) * dt;
                                Sdt += Sdh[n] * Mv + Mdh[n] * (Mv + aA * Shb);
                                Mdt += Mdh[n] * Mv;
                                SdA_loc[(size_t)d * N + n] += Sdh[n] * dt * hb + Mdh[n] * dt * Shb;
                                SdBg[(size_t)n * L + l] += (Sdh[n] + r * Mdh[n]) * dt * fabs(ul);
                                SdCg[(size_t)n * L + l] += fabs(go) * (Shl + Mhl);
                            }
                        }
                        dur[l] = du_acc;
                        if (softplus) {
                            const double x = (double)dr[l] + bi;
                            if (x <= 20.0) {
                                const double sg = 1.0 / (1.0 + exp(-x));
                                ddt_acc *= sg;
                                if (m) Sdt = sg * Sdt + (2.0 + rs[l] * dt) * Mdt;
                            }
                        }
                        ddr[l] = ddt_acc;
                        dD_loc[d] += go * ul;
                        db_loc[d] += ddt_acc;
                        if (m) {
                            m->du[((size_t)b * D + d) * L + l] = Sdu;
                            m->ddelta[((size_t)b * D + d) * L + l] = Sdt;
                            SdD_loc[d] += fabs(go * ul);
                            Sdb_loc[d] += Sdt;
                        }
                    }
                }
            }
#pragma omp critical
        {
            for (size_t i = 0; i < (size_t)D * N; ++i) dA[i] += dA_loc[i];
            if (dD) for (int d = 0; d < D; ++d) dD[d] += dD_loc[d];
            if (dbias) for (int d = 0; d < D; ++d) dbias[d] += db_loc[d];
            if (m) {
                for (size_t i = 0; i < (size_t)D * N; ++i) m->dA[i] += SdA_loc[i];
                if (m->dD) for (int d = 0; d < D; ++d) m->dD[d] += SdD_loc[d];
                if (m->dbias) for (int d = 0; d < D; ++d) m->dbias[d] += Sdb_loc[d];
            }
        }
        free(hs); free(dts); free(dA_loc); free(dD_loc); free(db_loc);
        free(Mhs); free(Shs); free(rs); free(SdA_loc); free(SdD_loc); free(Sdb_loc);
    }
}

void scan_ref_bwd_f64(const float *u, const float *delta, const float *A,
                      const float *Bm, const float *Cm, const float *Dv,
                      const float *bias, int softplus, const float *dout,
                      double *du, double *ddelta, double *dA, double *dB,
                      double *dC, double *dD, double *dbias,
                      int Bsz, int D, int L, int N, int G) {
    bwd_core(u, delta, A, Bm, Cm, Dv, bias, softplus, dout, du, ddelta, dA, dB, dC, dD, dbias, NULL, Bsz, D, L, N, G);
}

/* scan_ref_bwd_f64 + the magnitudes S_* (same shapes, zero-initialised; S_dD / S_dbias NULL with dD / dbias) */
void scan_ref_bwd_mag(const float *u, const float *delta, const float *A, const float *Bm, const float *Cm, const float *Dv,
                      const float *bias, int softplus, const float *dout, double *du, double *ddelta, double *dA, double *dB,
                      double *dC, double *dD, double *dbias, double *S_du, double *S_ddelta, double *S_dA, double *S_dB,
                      double *S_dC, double *S_dD, double *S_dbias, int Bsz, int D, int L, int N, int G) {
    const BwdMag m = {S_du, S_ddelta, S_dA, S_dB, S_dC, S_dD, S_dbias};
    bwd_core(u, delta, A, Bm, Cm, Dv, bias, softplus, dout, du, ddelta, dA, dB, dC, dD, dbias, &m, Bsz, D, L, N, G);
}

/* The same analytic backward evaluated sequentially in fp32 (fp32 outputs, zero-initialised by the caller): what an fp32 kernel
 * without approximate exp computes, to calibrate the backward's bound on the CPU as scan_ref_fwd_f32 does the forward's. */
void scan_ref_bwd_f32(const float *u, const float *delta, const float *A, const float *Bm, const float *Cm, const float *Dv,
                      const float *bias, int softplus, const float *dout, float *du, float *ddelta, float *dA, float *dB,
                      float *dC, float *dD, float *dbias, int Bsz, int D, int L, int N, int G) {
    const int rep = D / G;
#pragma omp parallel
    {
        float *hs = (float *)malloc(sizeof(float) * (size_t)N * L);
        float *dts = (float *)malloc(sizeof(float) * (size_t)L);
        float *dA_loc = (float *)calloc((size_t)D * N, sizeof(float));
        float *dD_loc = (float *)calloc((size_t)D, sizeof(float));
        float *db_loc = (float *)calloc((size_t)D, sizeof(float));
#pragma omp for collapse(2) schedule(static)
        for (int b = 0; b < Bsz; ++b)
            for (int g = 0; g < G; ++g) {
                const float *Bg = Bm + ((size_t)b * G + g) * N * L;
                const float *Cg = Cm + ((size_t)b * G + g) * N * L;
                float *dBg = dB + ((size_t)b * G + g) * N * L;
                float *dCg = dC + ((size_t)b * G + g) * N * L;
                for (int d = g * rep; d < (g + 1) * rep; ++d) {
                    const float *ur = u + ((size_t)b * D + d) * L;
                    const float *dr = delta + ((size_t)b * D + d) * L;
                    const float *gor = dout + ((size_t)b * D + d) * L;
                    const float *Ar = A + (size_t)d * N;
                    const float bi = bias ? bias[d] : 0.f;
                    const float Dd = Dv ? Dv[d] : 0.f;
                    float h[256], dh[256];
                    for (int n = 0; n < N; ++n) { h[n] = 0.f; dh[n] = 0.f; }
                    for (int l = 0; l < L; ++l) {
                        float dt = dr[l] + bi;
                        if (softplus) dt = softplus_f(dt);
                        dts[l] = dt;
                        for (int n = 0; n < N; ++n) {
                            h[n] = expf(dt * Ar[n]) * h[n] + dt * ur[l] * Bg[(size_t)n * L + l];
                            hs[(size_t)n * L + l] = h[n];
                        }
                    }
                    for (int l = L - 1; l >= 0; --l) {
                        const float dt = dts[l], ul = ur[l], go = gor[l];
                        float du_acc = Dd * go, ddt_acc = 0.f;
                        for (int n = 0; n < N; ++n) {
                            if (l + 1 < L) dh[n] *= expf(dts[l + 1] * Ar[n]);
                            dh[n] += Cg[(size_t)n * L + l] * go;
                            const float Bv = Bg[(size_t)n * L + l], hl = hs[(size_t)n * L + l], bl = dt * ul * Bv;
                            du_acc += dh[n] * Bv * dt;
                            ddt_acc += dh[n] * (ul * Bv + Ar[n] * (hl - bl));
                            dA_loc[(size_t)d * N + n] += dh[n] * dt * (hl - bl);
                            dBg[(size_t)n * L + l] += dh[n] * dt * ul;
                            dCg[(size_t)n * L + l] += go * hl;
                        }
                        du[((size_t)b * D + d) * L + l] = du_acc;
                        if (softplus) {
                            const float x = dr[l] + bi;
                            if (x <= 20.f) ddt_acc *= 1.f / (1.f + expf(-x));
                        }
                        ddelta[((size_t)b * D + d) * L + l] = ddt_acc;
                        dD_loc[d] += go * ul;
                        db_loc[d] += ddt_acc;
                    }
                }
            }
#pragma omp critical
        {
            for (size_t i = 0; i < (size_t)D * N; ++i) dA[i] += dA_loc[i];
            if (dD) for (int d = 0; d < D; ++d) dD[d] += dD_loc[d];
            if (dbias) for (int d = 0; d < D; ++d) dbias[d] += db_loc[d];
        }
        free(hs); free(dts); free(dA_loc); free(dD_loc); free(db_loc);
    }
}
