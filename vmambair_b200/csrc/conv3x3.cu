// Dense 3x3 convolution (stride 1, pad 1) of the U-Net's non-OSS stages (SURVEY.md 8f rank 1): OverlapPatchEmbed.proj
// (SRGAN/VmambaIR/archs/MambaSISR6_arch.py:520-528), Downsample = conv + PixelUnshuffle(2) (:533-541), Upsample = conv +
// PixelShuffle(2) (:544-553), the SR tail's conv_last (+ the nearest-upsampled input image, :607,640) and Mamber32's output
// conv.  One implicit GEMM per launch -- M = output channels, N = a tile of 8 x 16 output pixels, K = 9 taps x input
// channels -- on mma.sync.m16n8k16 (the problems are 0.02-3 GFLOP: launch / latency bound, the tensor pipe is not the
// limit), with everything the reference does around the conv as separate passes folded into the load or the store:
//   * the input halo tile comes straight from NCHW (or NHWC) global memory as TMA boxes (cp.async.bulk.tensor, borders = the
//     TMA's zero fill) -- no layout-transform kernel in front of the conv;
//   * the store applies PixelUnshuffle(2) / PixelShuffle(2) index arithmetic, writes into a channel slice of a wider tensor
//     (the skip concatenation of the decoder: torch.cat never runs) or adds the nearest-neighbour up-sampled input image
//     and emits NCHW -- no permutation / cat / interpolate / add kernels behind it.
// fp32 I/O (parity mode) runs a SIMT FFMA kernel with the same tiling and the same store.
#include "common.cuh"
#include "oss_params.h"
#include "tma.cuh"

namespace vmb {
namespace {

constexpr int kTH = 8, kTW = 16;                      // output pixels of a CTA tile
constexpr int kHaloW = kTW + 2, kHalo = (kTH + 2) * kHaloW;  // 10 x 18 input pixels

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
    const uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
    const int sz = valid ? 16 : 0;  // src-size 0: the 16 destination bytes are zero-filled
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldsm4(uint32_t (&r)[4], const void* smem) {
    const uint32_t s = static_cast<uint32_t>(__cvta_generic_to_shared(smem));
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(s));
}
template <typename T> __device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);
template <> __device__ __forceinline__ void mma16816<__nv_bfloat16>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <> __device__ __forceinline__ void mma16816<__half>(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// One output element (b, m, y, x) of the convolution -> its place in `out` (see vmb_conv3x3_args.mode).
template <typename T>
__device__ __forceinline__ void conv_store_raw(const Conv3Params& p, int b, int m, int y, int x, float v) {
    T* out = static_cast<T*>(p.out) + (int64_t)b * p.o_bs;
    if (p.mode == VMB_CONV_PLAIN) {
        out[(int64_t)m * p.o_cs + (int64_t)y * p.W + x] = from_f32<T>(v);
    } else if (p.mode == VMB_CONV_UNSHUFFLE2) {  // nn.PixelUnshuffle(2): out[b, 4m + 2(y%2) + x%2, y/2, x/2]
        const int oc = 4 * m + 2 * (y & 1) + (x & 1);
        out[(int64_t)oc * p.o_cs + (int64_t)(y >> 1) * (p.W >> 1) + (x >> 1)] = from_f32<T>(v);
    } else if (p.mode == VMB_CONV_SHUFFLE2) {    // nn.PixelShuffle(2): out[b, m/4, 2y + (m/2)%2, 2x + m%2]
        out[(int64_t)(m >> 2) * p.o_cs + (int64_t)(2 * y + ((m >> 1) & 1)) * (2 * p.W) + 2 * x + (m & 1)] = from_f32<T>(v);
    } else {                                      // VMB_CONV_ADD_NEAREST: + add[b, m, y/s, x/s]
        const T* add = static_cast<const T*>(p.add) + (int64_t)b * p.add_bs + (int64_t)m * p.add_cs;
        v += to_f32<T>(add[(int64_t)(y / p.add_scale) * (p.W / p.add_scale) + x / p.add_scale]);
        out[(int64_t)m * p.o_cs + (int64_t)y * p.W + x] = from_f32<T>(v);
    }
}

// Fragment store of the tensor-core kernels: this lane holds channel m at (y, x) and (y, x + 1), x even.  Called by all 32 lanes
// (the shuffle modes trade one element with a neighbour lane so that every lane writes one 32-bit word):
//   PLAIN / ADD_NEAREST  (x, x+1) of channel m are adjacent in the output;
//   SHUFFLE2             channels (m even, m+1) at x are adjacent (columns 2x, 2x+1): partner = lane ^ 4 (row g ^ 1);
//   UNSHUFFLE2           x and x+2 of one parity are adjacent (columns x/2, x/2+1 of channel 4m+2(y%2)+x%2): partner = lane ^ 1.
// pair_ok: the 32-bit stores are aligned (even strides / base, W % 4 == 0); otherwise element-wise stores.
template <typename T>
__device__ __forceinline__ void conv_store_frag(const Conv3Params& p, int b, int m, int y, int x, float v0, float v1, bool pair_ok,
                                                int lane) {
    const bool valid = m < p.Cout && y < p.H && x < p.W;
    const float bs = (p.bias && m < p.Cout) ? p.bias[m] : 0.f;
    v0 += bs;
    v1 += bs;
    T* out = static_cast<T*>(p.out) + (int64_t)b * p.o_bs;
    if (!pair_ok) {
        if (valid) {
            conv_store_raw<T>(p, b, m, y, x, v0);
            if (x + 1 < p.W) conv_store_raw<T>(p, b, m, y, x + 1, v1);
        }
        return;
    }
    if (p.mode == VMB_CONV_SHUFFLE2) {
        const float s0 = __shfl_xor_sync(0xffffffffu, v0, 4), s1 = __shfl_xor_sync(0xffffffffu, v1, 4);
        if (valid) {
            const bool odd = (lane >> 2) & 1;  // m odd
            T* o = out + (int64_t)(m >> 2) * p.o_cs + (int64_t)(2 * y + ((m >> 1) & 1)) * (2 * p.W) + 2 * x + (odd ? 2 : 0);
            *reinterpret_cast<uint32_t*>(o) = odd ? pack2<T>(s1, v1) : pack2<T>(v0, s0);
        }
    } else if (p.mode == VMB_CONV_UNSHUFFLE2) {
        const float s0 = __shfl_xor_sync(0xffffffffu, v0, 1), s1 = __shfl_xor_sync(0xffffffffu, v1, 1);
        if (valid) {
            const bool odd = lane & 1;  // x / 2 odd
            T* o = out + (int64_t)(4 * m + 2 * (y & 1) + (odd ? 1 : 0)) * p.o_cs + (int64_t)(y >> 1) * (p.W >> 1) + (x >> 1) - (odd ? 1 : 0);
            *reinterpret_cast<uint32_t*>(o) = odd ? pack2<T>(s1, v1) : pack2<T>(v0, s0);
        }
    } else if (valid) {
        if (p.mode == VMB_CONV_ADD_NEAREST) {
            const T* add = static_cast<const T*>(p.add) + (int64_t)b * p.add_bs + (int64_t)m * p.add_cs +
                           (int64_t)(y / p.add_scale) * (p.W / p.add_scale);
            v0 += to_f32<T>(add[x / p.add_scale]);
            v1 += to_f32<T>(add[(x + 1) / p.add_scale]);
        }
        *reinterpret_cast<uint32_t*>(out + (int64_t)m * p.o_cs + (int64_t)y * p.W + x) = pack2<T>(v0, v1);
    }
}

template <typename T>
__device__ __forceinline__ void conv_store(const Conv3Params& p, int b, int m, int y, int x, float v) {
    conv_store_raw<T>(p, b, m, y, x, p.bias ? v + p.bias[m] : v);
}

// ---- 16-bit I/O, any NCHW geometry (ragged W, unaligned views): implicit GEMM on mma.sync ------------------------------------
// Shared memory per stage: A = weights of the K chunk [9 taps][MT rows][KC] and B = input halo tile [180 pixels][KC], rows
// padded by 16 B (row pitch 48 B at KC = 16: the eight 16 B rows of an ldmatrix phase fall into distinct bank groups).  Two
// stages: the weights of chunk k+1 arrive by cp.async and its input pixels through registers (the [channel][pixel] ->
// [pixel][channel] transposition happens in the register -> shared store) while chunk k is multiplied.  The fallback of
// conv3x3_pipe_kernel below, which needs 16 B-aligned rows.
template <typename T, int MT, int KC, bool NHWC>
__global__ void __launch_bounds__(128) conv3x3_generic_kernel(const Conv3Params p) {
    pdl_trigger();
    constexpr int PITCH = KC * 2 + 16;            // bytes per smem row
    constexpr int A_BYTES = 9 * MT * PITCH, B_BYTES = kHalo * PITCH, STAGE = A_BYTES + B_BYTES;
    constexpr int MI = MT / 16;
    constexpr int KH = KC / 8;                    // 16 B pieces per row
    constexpr int NPAIR = KC / 2;                 // channel pairs per chunk
    constexpr int BREG = (NPAIR * kHalo + 127) / 128;
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tiles_x = (p.W + kTW - 1) / kTW;
    const int x0 = (blockIdx.x % tiles_x) * kTW, y0 = (blockIdx.x / tiles_x) * kTH;
    const int m0 = blockIdx.y * MT, b = blockIdx.z;
    const T* __restrict__ xin = static_cast<const T*>(p.x) + (int64_t)b * p.x_bs;
    const T* __restrict__ wgt = static_cast<const T*>(p.w);
    const int nchunk = (p.Cin + KC - 1) / KC;

    float acc[MI][4][4];
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

    auto stage_A = [&](int kc, int s) {  // weights are static parameters: may be fetched before pdl_wait()
        unsigned char* A = smem + s * STAGE;
        for (int i = tid; i < 9 * MT * KH; i += 128) {
            const int piece = i % KH, row = (i / KH) % MT, tap = i / (KH * MT);
            const T* src = wgt + ((int64_t)(tap * p.Mpad + m0 + row)) * p.Kpad + kc * KC + piece * 8;
            cp_async16(A + (tap * MT + row) * PITCH + piece * 16, src, kc * KC + piece * 8 < p.Kpad);
        }
    };
    uint32_t breg[BREG];
    auto load_B = [&](int kc, int s) {
        if constexpr (NHWC) {
            unsigned char* Bs = smem + s * STAGE + A_BYTES;
            for (int i = tid; i < kHalo * KH; i += 128) {
                const int piece = i % KH, hp = i / KH;
                const int gy = y0 - 1 + hp / kHaloW, gx = x0 - 1 + hp % kHaloW, c = kc * KC + piece * 8;
                const bool ok = gy >= 0 && gy < p.H && gx >= 0 && gx < p.W && c < p.Cin;
                const T* src = ok ? xin + ((int64_t)gy * p.W + gx) * p.Cin + c : xin;
                cp_async16(Bs + hp * PITCH + piece * 16, src, ok);
            }
        } else {
#pragma unroll
            for (int j = 0; j < BREG; ++j) {
                const int i = tid + 128 * j;
                const int hp = i % kHalo, cp = i / kHalo;
                const int gy = y0 - 1 + hp / kHaloW, gx = x0 - 1 + hp % kHaloW, c = kc * KC + 2 * cp;
                uint32_t v = 0;
                if (cp < NPAIR && gy >= 0 && gy < p.H && gx >= 0 && gx < p.W && c < p.Cin) {
                    const T* src = xin + (int64_t)c * p.x_cs + (int64_t)gy * p.W + gx;
                    const uint32_t lo = *reinterpret_cast<const unsigned short*>(src);
                    const uint32_t hi = c + 1 < p.Cin ? *reinterpret_cast<const unsigned short*>(src + p.x_cs) : 0u;
                    v = lo | (hi << 16);
                }
                breg[j] = v;
            }
        }
    };
    auto store_B = [&](int s) {
        if constexpr (!NHWC) {
            unsigned char* Bs = smem + s * STAGE + A_BYTES;
#pragma unroll
            for (int j = 0; j < BREG; ++j) {
                const int i = tid + 128 * j;
                const int hp = i % kHalo, cp = i / kHalo;
                if (cp < NPAIR) *reinterpret_cast<uint32_t*>(Bs + hp * PITCH + cp * 4) = breg[j];
            }
        }
    };

    stage_A(0, 0);
    pdl_wait();  // the activations are the preceding kernel's output
    load_B(0, 0);
    cp_async_commit();
    store_B(0);

    // fragment addressing (warp-uniform bases + per-lane offsets)
    const int trow0 = 2 * warp;                         // this warp's two tile rows
    const int a_lane = ((lane & 7) + ((lane >> 3) & 1) * 8) * PITCH + (lane >> 4) * 16;
    const int b_lane = (((lane >> 4) & 1) * 8 + (lane & 7)) * PITCH + ((lane >> 3) & 1) * 16;

    for (int kc = 0; kc < nchunk; ++kc) {
        const int s = kc & 1;
        if (kc + 1 < nchunk) {
            stage_A(kc + 1, s ^ 1);
            load_B(kc + 1, s ^ 1);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const unsigned char* A = smem + s * STAGE;
        const unsigned char* Bs = A + A_BYTES;
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
#pragma unroll
            for (int ks = 0; ks < KC / 16; ++ks) {
                uint32_t bf[2][4];
#pragma unroll
                for (int r = 0; r < 2; ++r)  // tile row trow0 + r: n-tiles 2r (columns 0-7) and 2r+1 (columns 8-15)
                    ldsm4(bf[r], Bs + ((trow0 + r + dy) * kHaloW + dx) * PITCH + b_lane + ks * 32);
#pragma unroll
                for (int mi = 0; mi < MI; ++mi) {
                    uint32_t af[4];
                    ldsm4(af, A + (tap * MT + mi * 16) * PITCH + a_lane + ks * 32);
#pragma unroll
                    for (int j = 0; j < 4; ++j) mma16816<T>(acc[mi][j], af, bf[j >> 1][(j & 1) * 2], bf[j >> 1][(j & 1) * 2 + 1]);
                }
            }
        }
        if (kc + 1 < nchunk) store_B(s ^ 1);
        __syncthreads();
    }

    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int mi = 0; mi < MI; ++mi)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int m = m0 + mi * 16 + g + (e >> 1) * 8;
                const int y = y0 + trow0 + (j >> 1), x = x0 + (j & 1) * 8 + 2 * t + (e & 1);
                if (m < p.Cout && y < p.H && x < p.W) conv_store<T>(p, b, m, y, x, acc[mi][j][e]);
            }
}

// ---- 16-bit I/O, aligned geometry (W % 8 == 0, 16 B-aligned planes: every site of the networks): TMA-staged pipeline ------------
// One elected thread issues two cp.async.bulk.tensor boxes per 16-channel chunk into a STAGES-deep ring (completion on an
// mbarrier per stage): the weights [9 taps x MT rows][16] with the 32 B swizzle (conflict-free ldmatrix on 32 B rows) and the
// input halo tile -- NHWC input: box (16 c, 18 x, 10 y), swizzled, consumed by ldmatrix as it lands; NCHW input: box (32 x,
// 10 y, 16 c) = channel planes as they lie in global memory, re-laid once per chunk by all threads into the [pixel][channel]
// tile the fragments want (the [c][p] -> [p][c] step costs ~12 packed stores per thread and chunk; assembling fragments from
// the planar tile tap by tap costs four times that).  Image borders, the ragged last tile and channels >= Cin are the TMA's
// out-of-bounds zero fill: the kernel has no address arithmetic or predicates on the load side at all.
constexpr int kRawW = 32, kRawX = 8;                     // NCHW box: 32 pixels (64 B rows) starting at x0 - 8: a box must start on
                                                         // a 16 B boundary of global memory (x0 - 1 raises an illegal-instruction fault)
constexpr int kRawPlane = (kTH + 2) * kRawW * 2;         // bytes per channel plane of the raw box
constexpr int kBtPitch = 48;                             // [pixel][16 channels] tile, rows padded to 48 B

template <int MT, bool NHWC> struct TmaConvCfg {
    static constexpr int A_BYTES = 9 * MT * 32;
    static constexpr int B_BYTES = NHWC ? kHalo * 32 : 16 * kRawPlane;
    static constexpr int STAGE = (A_BYTES + B_BYTES + 255) / 256 * 256;
    static constexpr int BT_BYTES = NHWC ? 0 : kHalo * kBtPitch;
    static constexpr int smem(int stages) { return stages * STAGE + BT_BYTES + 8 * stages + 1024; }
};

template <typename T, int MT, int STAGES, bool NHWC>
__global__ void __launch_bounds__(128) conv3x3_tma_kernel(const Conv3Params p, const __grid_constant__ CUtensorMap mapW,
                                                          const __grid_constant__ CUtensorMap mapX) {
    pdl_trigger();
    using Cfg = TmaConvCfg<MT, NHWC>;
    constexpr int MI = MT / 16;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    unsigned char* Bt = smem + STAGES * Cfg::STAGE;
    uint64_t* full = reinterpret_cast<uint64_t*>(Bt + Cfg::BT_BYTES);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tiles_x = (p.W + kTW - 1) / kTW, tiles_xy = tiles_x * ((p.H + kTH - 1) / kTH);
    // one pixel tile per CTA: grid.x walks the tiles of the whole batch
    const int b = blockIdx.x / tiles_xy, tile = blockIdx.x % tiles_xy;
    const int x0 = (tile % tiles_x) * kTW, y0 = (tile / tiles_x) * kTH;
    const int m0 = blockIdx.y * MT;
    const int nchunk = (p.Cin + 15) / 16;

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s) mbarrier_init(&full[s], 1);
        mbarrier_init_fence();
    }
    __syncthreads();
    // one stage = the weights box + the input box on one mbarrier; the weights are static parameters, so the boxes of the first
    // STAGES chunks are requested while the preceding kernel of the stream is still draining (PDL), the activations after it
    auto issue_w = [&](int kc, int s) {
        mbarrier_expect_tx(&full[s], Cfg::A_BYTES + Cfg::B_BYTES);
        tma_load_4d(smem + s * Cfg::STAGE, &mapW, &full[s], kc * 16, m0, 0, 0);
    };
    auto issue_x = [&](int kc, int s) {
        unsigned char* dst = smem + s * Cfg::STAGE + Cfg::A_BYTES;
        if constexpr (NHWC) tma_load_4d(dst, &mapX, &full[s], kc * 16, x0 - 1, y0 - 1, b);
        else tma_load_4d(dst, &mapX, &full[s], x0 - kRawX, y0 - 1, kc * 16, b);
    };
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s)
            if (s < nchunk) issue_w(s, s);
    }
    pdl_wait();
    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < STAGES; ++s)
            if (s < nchunk) issue_x(s, s);
    }

    float acc[MI][4][4];
    const int trow0 = 2 * warp;
    const int g = lane >> 2, t = lane & 3;
    // A: row r of the swizzled [rows][32 B] tile holds its 16 B half q at ((q ^ ((r >> 2) & 1)) << 4)
    const int a_row = (lane & 7) + ((lane >> 3) & 1) * 8;
    const int a_lane = a_row * 32 + (((lane >> 4) ^ ((a_row >> 2) & 1)) << 4);
    const int bt_lane = (((lane >> 4) & 1) * 8 + (lane & 7)) * kBtPitch + ((lane >> 3) & 1) * 16;  // [pixel][channel] tile (NCHW)
    const int bq = (lane >> 3) & 1, bpix = ((lane >> 4) & 1) * 8 + (lane & 7);                     // swizzled halo tile (NHWC)
    // re-layout work list of this thread (NCHW): item i = tid + 128 j -> (halo pixel, channel pair); source offset in the raw box
    // (low half) and destination offset in the [pixel][channel] tile (high half), fixed for the whole kernel
    constexpr int NT = (8 * kHalo + 127) / 128;
    uint32_t toff[NHWC ? 1 : NT];
    if constexpr (!NHWC) {
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            const int i = tid + 128 * j;
            const int hp = i % kHalo, cp = i / kHalo;
            const uint32_t src = 2 * cp * kRawPlane + (hp / kHaloW) * (kRawW * 2) + (hp % kHaloW + kRawX - 1) * 2;
            const uint32_t dst = hp * kBtPitch + cp * 4;
            toff[j] = cp < 8 ? (src | (dst << 16)) : 0xffffffffu;
        }
    }
    // 32-bit stores need even element offsets: W % 4 == 0 (true on this path), even strides, 4 B-aligned base
    const bool pair_ok = p.W % 4 == 0 && p.o_bs % 2 == 0 && p.o_cs % 2 == 0 && (reinterpret_cast<uintptr_t>(p.out) & 3) == 0;

    bool jok[4];  // n-tiles inside the image (warp-uniform): the others are skipped
#pragma unroll
    for (int j = 0; j < 4; ++j) jok[j] = (y0 + trow0 + (j >> 1) < p.H) && (x0 + (j & 1) * 8 < p.W);
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
    for (int kc = 0; kc < nchunk; ++kc) {
        const int slot = kc % STAGES;
        mbarrier_wait(&full[slot], (kc / STAGES) & 1);
        const unsigned char* A = smem + slot * Cfg::STAGE;
        const unsigned char* Braw = A + Cfg::A_BYTES;
        if constexpr (!NHWC) {
            // [16 planes][10][32] -> [180 pixels][16 channels]: two channels of one pixel per packed 32-bit store
            uint32_t tv[NT];
#pragma unroll
            for (int j = 0; j < NT; ++j) {
                const unsigned char* src = Braw + (toff[j] & 0xffffu);
                tv[j] = toff[j] != 0xffffffffu ? (*reinterpret_cast<const unsigned short*>(src) |
                                                  (uint32_t(*reinterpret_cast<const unsigned short*>(src + kRawPlane)) << 16))
                                               : 0u;
            }
#pragma unroll
            for (int j = 0; j < NT; ++j)
                if (toff[j] != 0xffffffffu) *reinterpret_cast<uint32_t*>(Bt + (toff[j] >> 16)) = tv[j];
            __syncthreads();
        }
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = tap / 3, dx = tap % 3;
            uint32_t bf[2][4];
#pragma unroll
            for (int r = 0; r < 2; ++r) {  // tile row trow0 + r: n-tiles 2r (columns 0-7) and 2r+1 (columns 8-15)
                if constexpr (NHWC) {
                    const int hp = (trow0 + r + dy) * kHaloW + dx + bpix;
                    ldsm4(bf[r], Braw + hp * 32 + ((bq ^ ((hp >> 2) & 1)) << 4));
                } else {
                    ldsm4(bf[r], Bt + ((trow0 + r + dy) * kHaloW + dx) * kBtPitch + bt_lane);
                }
            }
#pragma unroll
            for (int mi = 0; mi < MI; ++mi) {
                uint32_t af[4];
                ldsm4(af, A + (tap * MT + mi * 16) * 32 + a_lane);
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (jok[j]) mma16816<T>(acc[mi][j], af, bf[j >> 1][(j & 1) * 2], bf[j >> 1][(j & 1) * 2 + 1]);
            }
        }
        __syncthreads();  // every warp is done with this stage (and with Bt)
        if (tid == 0 && kc + STAGES < nchunk) {
            fence_proxy_async();  // the stage was read through the generic proxy; the refill writes through the async proxy
            issue_w(kc + STAGES, slot);
            issue_x(kc + STAGES, slot);
        }
    }
#pragma unroll
    for (int mi = 0; mi < MI; ++mi)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
                conv_store_frag<T>(p, b, m0 + mi * 16 + g + h * 8, y0 + trow0 + (j >> 1), x0 + (j & 1) * 8 + 2 * t,
                                   acc[mi][j][2 * h], acc[mi][j][2 * h + 1], pair_ok, lane);
}

// ---- fp32 I/O (parity mode): direct FFMA convolution, one output pixel x 16 output channels per thread ---------------------
template <typename T, bool NHWC>
__global__ void __launch_bounds__(128) conv3x3_simt_kernel(const Conv3Params p) {
    pdl_trigger();
    constexpr int MT = 16, KC = 8;
    __shared__ float sx[KC][kTH + 2][kHaloW + 1];
    __shared__ float sw[9][KC][MT];
    const int tid = threadIdx.x, tx = tid % kTW, ty = tid / kTW;
    const int tiles_x = (p.W + kTW - 1) / kTW;
    const int x0 = (blockIdx.x % tiles_x) * kTW, y0 = (blockIdx.x / tiles_x) * kTH;
    const int m0 = blockIdx.y * MT, b = blockIdx.z;
    const T* __restrict__ xin = static_cast<const T*>(p.x) + (int64_t)b * p.x_bs;
    const T* __restrict__ wgt = static_cast<const T*>(p.w);
    float acc[MT];
#pragma unroll
    for (int i = 0; i < MT; ++i) acc[i] = 0.f;
    pdl_wait();
    for (int c0 = 0; c0 < p.Cin; c0 += KC) {
        for (int i = tid; i < KC * kHalo; i += 128) {
            const int hp = i % kHalo, cc = i / kHalo;
            const int hy = hp / kHaloW, hx = hp % kHaloW, gy = y0 - 1 + hy, gx = x0 - 1 + hx, c = c0 + cc;
            float v = 0.f;
            if (gy >= 0 && gy < p.H && gx >= 0 && gx < p.W && c < p.Cin)
                v = to_f32<T>(NHWC ? xin[((int64_t)gy * p.W + gx) * p.Cin + c] : xin[(int64_t)c * p.x_cs + (int64_t)gy * p.W + gx]);
            sx[cc][hy][hx] = v;
        }
        for (int i = tid; i < 9 * KC * MT; i += 128) {
            const int mm = i % MT, cc = (i / MT) % KC, tap = i / (MT * KC);
            const int c = c0 + cc;
            sw[tap][cc][mm] = c < p.Kpad ? to_f32<T>(wgt[((int64_t)(tap * p.Mpad + m0 + mm)) * p.Kpad + c]) : 0.f;
        }
        __syncthreads();
#pragma unroll 2
        for (int cc = 0; cc < KC; ++cc)
#pragma unroll
            for (int tap = 0; tap < 9; ++tap) {
                const float v = sx[cc][ty + tap / 3][tx + tap % 3];
#pragma unroll
                for (int mm = 0; mm < MT; ++mm) acc[mm] = fmaf(sw[tap][cc][mm], v, acc[mm]);
            }
        __syncthreads();
    }
    const int y = y0 + ty, x = x0 + tx;
    if (y < p.H && x < p.W)
#pragma unroll
        for (int mm = 0; mm < MT; ++mm)
            if (m0 + mm < p.Cout) conv_store<T>(p, b, m0 + mm, y, x, acc[mm]);
}

template <typename T, int MT>
int launch_generic(const Conv3Params& p, cudaStream_t stream) {
    constexpr int PITCH = 16 * 2 + 16;
    constexpr int SMEM = 2 * (9 * MT * PITCH + kHalo * PITCH);
    auto kern = conv3x3_generic_kernel<T, MT, 16, false>;
    // per launch, like the scan launchers: the attribute is per device, and a process may drive several (nn.DataParallel-style callers)
    if (SMEM > 48 * 1024) VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    const dim3 grid(cdiv(p.W, kTW) * cdiv(p.H, kTH), cdiv(p.Cout, MT), p.B);
    VMB_CUDA(launch_pdl(kern, grid, dim3(128), SMEM, stream, p));
    return VMB_OK;
}

template <typename T, int MT, int STAGES, bool NHWC>
int launch_tma(const Conv3Params& p, int dtype, cudaStream_t stream) {
    using Cfg = TmaConvCfg<MT, NHWC>;
    constexpr int SMEM = Cfg::smem(STAGES);
    static_assert(SMEM <= 227 * 1024, "conv3x3: stage ring exceeds shared memory");
    CUtensorMap mapW, mapX;
    {
        const uint64_t dims[4] = {(uint64_t)p.Kpad, (uint64_t)p.Mpad, 9, 1};
        const int64_t str[3] = {p.Kpad, (int64_t)p.Mpad * p.Kpad, (int64_t)9 * p.Mpad * p.Kpad};
        const uint32_t box[4] = {16, (uint32_t)MT, 9, 1};
        const int rc = make_tmap_4d(&mapW, dtype, p.w, dims, str, box, 1);
        if (rc != VMB_OK) return rc;
    }
    if (NHWC) {
        const uint64_t dims[4] = {(uint64_t)p.Cin, (uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.B};
        const int64_t str[3] = {p.Cin, (int64_t)p.W * p.Cin, (int64_t)p.H * p.W * p.Cin};
        const uint32_t box[4] = {16, (uint32_t)kHaloW, (uint32_t)(kTH + 2), 1};
        const int rc = make_tmap_4d(&mapX, dtype, p.x, dims, str, box, 1);
        if (rc != VMB_OK) return rc;
    } else {
        const uint64_t dims[4] = {(uint64_t)p.W, (uint64_t)p.H, (uint64_t)p.Cin, (uint64_t)p.B};
        const int64_t str[3] = {p.W, p.x_cs, p.x_bs};
        const uint32_t box[4] = {(uint32_t)kRawW, (uint32_t)(kTH + 2), 16, 1};
        const int rc = make_tmap_4d(&mapX, dtype, p.x, dims, str, box, 0);
        if (rc != VMB_OK) return rc;
    }
    auto kern = conv3x3_tma_kernel<T, MT, STAGES, NHWC>;
    VMB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));  // per device: set at every launch
    // pixel tiles of the whole batch on grid.x, one CTA per tile
    const int ntile = cdiv(p.W, kTW) * cdiv(p.H, kTH) * p.B;
    VMB_CUDA(launch_pdl(kern, dim3(ntile, cdiv(p.Cout, MT), 1), dim3(128), SMEM, stream, p, mapW, mapX));
    return VMB_OK;
}

template <typename T>
int launch_16(const Conv3Params& p, int dtype, cudaStream_t stream) {
    const int tiles = cdiv(p.W, kTW) * cdiv(p.H, kTH) * p.B;
    if (p.in_nhwc) {  // dense (B,H,W,Cin), Cin % 8 == 0, 16 B-aligned base (checked by the C-ABI entry)
        if (p.Cout <= 16) return launch_tma<T, 16, 4, true>(p, dtype, stream);
        return launch_tma<T, 64, 3, true>(p, dtype, stream);
    }
    const bool aligned = p.W % 8 == 0 && p.x_bs % 8 == 0 && p.x_cs % 8 == 0 && (reinterpret_cast<uintptr_t>(p.x) & 15) == 0 &&
                         p.x_cs >= (int64_t)p.H * p.W && p.x_bs > 0;
    if (!aligned) return p.Cout <= 16 ? launch_generic<T, 16>(p, stream) : launch_generic<T, 64>(p, stream);
    // output-channel tile: the widest one that still fills one wave of CTAs (every K chunk costs a CTA a fixed barrier / re-layout
    // overhead that a wider tile amortises, but an idle SM amortises nothing)
    const int want = num_sms();
    if (p.Cout > 32 && tiles * cdiv(p.Cout, 64) >= want) return launch_tma<T, 64, 3, false>(p, dtype, stream);
    if (p.Cout > 16 && tiles * cdiv(p.Cout, 32) >= want) return launch_tma<T, 32, 3, false>(p, dtype, stream);
    return launch_tma<T, 16, 4, false>(p, dtype, stream);
}

}  // namespace

int conv3x3_launch(const Conv3Params& p, int dtype, cudaStream_t stream) {
    if (dtype == VMB_BF16) return launch_16<__nv_bfloat16>(p, dtype, stream);
    if (dtype == VMB_F16) return launch_16<__half>(p, dtype, stream);
    const dim3 grid(cdiv(p.W, kTW) * cdiv(p.H, kTH), cdiv(p.Cout, 16), p.B);
    if (p.in_nhwc) {
        VMB_CUDA(launch_pdl(conv3x3_simt_kernel<float, true>, grid, dim3(128), 0, stream, p));
    } else {
        VMB_CUDA(launch_pdl(conv3x3_simt_kernel<float, false>, grid, dim3(128), 0, stream, p));
    }
    return VMB_OK;
}

}  // namespace vmb
