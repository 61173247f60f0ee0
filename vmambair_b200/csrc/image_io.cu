// Image-level I/O of RealESRGANer.enhance (RealSR/VmambaIR/utils.py:174-243) on the device: 8- / 16-bit HWC images in and out,
// NCHW planes in the compute dtype for the network, and OpenCV's Lanczos-4 resize.  Every float operation that decides an output
// bit is spelt out with an explicit rounding (__fmul_rn, __fadd_rn, __fmaf_rn, __fdiv_rn, double __d*_rn) so that nvcc cannot
// contract or reassociate it: the results equal vmambair_b200/image_ref.py, which restates OpenCV and numpy operation by operation.
#include "common.cuh"

namespace vmb {

namespace {

constexpr int kTx = 32, kTy = 8;  // 2-D launch tile of every kernel here

template <bool U16>
__device__ __forceinline__ float load_px(const void* p, int64_t i) {
    return U16 ? (float)reinterpret_cast<const uint16_t*>(p)[i] : (float)reinterpret_cast<const uint8_t*>(p)[i];
}

// F.pad(..., 'reflect') on the bottom / right, three pads in a row: index into the padded extent -> index into the image
__device__ __forceinline__ int reflect3(int i, int n, const int* pads) {
    const int n1 = n + pads[0], n2 = n1 + pads[1];
    if (i >= n2) i = 2 * (n2 - 1) - i;
    if (i >= n1) i = 2 * (n1 - 1) - i;
    if (i >= n) i = 2 * (n - 1) - i;
    return i;
}

// ---- max ----
template <bool U16>
__global__ void __launch_bounds__(256) image_max_kernel(const vmb_image_max_args a) {
    pdl_trigger();
    pdl_wait();
    const int x = blockIdx.x * kTx + threadIdx.x;
    unsigned int m = 0;
    if (x < a.W)
        for (int y = blockIdx.y * kTy + threadIdx.y; y < a.H; y += gridDim.y * kTy)
            for (int c = 0; c < a.channels; ++c)
                m = max(m, (unsigned int)load_px<U16>(a.img, y * a.row_stride + x * a.pixel_stride + c * a.channel_stride));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(a.max_out, m);
}

// ---- image -> planes ----
template <bool U16, typename out_t>
__global__ void __launch_bounds__(256) image_to_planes_kernel(const vmb_image_to_planes_args a, int Hp, int Wp) {
    pdl_trigger();
    pdl_wait();
    const int x = blockIdx.x * kTx + threadIdx.x, y = blockIdx.y * kTy + threadIdx.y;
    if (x >= Wp || y >= Hp) return;
    const int sy = reflect3(y, a.H, a.pad_h), sx = reflect3(x, a.W, a.pad_w);
    const int64_t base = sy * a.row_stride + sx * a.pixel_stride;
    const int64_t plane = (int64_t)Hp * Wp, o = (int64_t)y * Wp + x;
    out_t* out = reinterpret_cast<out_t*>(a.out);
    if (a.channels == 1) {
        const out_t v = from_f32<out_t>(__fdiv_rn(load_px<U16>(a.img, base), a.max_range));
        out[o] = v; out[plane + o] = v; out[2 * plane + o] = v;
        return;
    }
#pragma unroll
    for (int c = 0; c < 3; ++c)  // plane c (RGB) <- channel 2 - c (BGR)
        out[c * plane + o] = from_f32<out_t>(__fdiv_rn(load_px<U16>(a.img, base + (2 - c) * a.channel_stride), a.max_range));
    if (a.alpha_plane) {
        const out_t v = from_f32<out_t>(__fdiv_rn(load_px<U16>(a.img, base + 3 * a.channel_stride), a.max_range));
        out[3 * plane + o] = v; out[4 * plane + o] = v; out[5 * plane + o] = v;
    }
}

// ---- planes -> image ----
__device__ __forceinline__ float gray_bgr(float b, float g, float r) {  // cv2 COLOR_BGR2GRAY, float32 vector loop
    return __fmaf_rn(r, 0.299f, __fmaf_rn(b, 0.114f, __fmul_rn(g, 0.587f)));
}

// cv2.resize source position (resize.cpp): fx = float((d + 0.5) * (1 / (dst / src)) - 0.5), sx = floor(fx), fx -= sx
__device__ __forceinline__ void src_pos(int d, int dst, int src, int& s, float& f) {
    const double scale = __ddiv_rn(1.0, __ddiv_rn((double)dst, (double)src));
    const float fx = __double2float_rn(__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5));
    s = (int)floorf(fx);
    f = __fsub_rn(fx, (float)s);
}

// INTER_LINEAR taps with cv2's border clamping of the sample position
__device__ __forceinline__ void linear_taps(int d, int dst, int src, int& s0, int& s1, float& w0, float& w1) {
    float f;
    src_pos(d, dst, src, s0, f);
    if (s0 < 0) { f = 0.f; s0 = 0; }
    if (s0 >= src - 1) { f = 0.f; s0 = src - 1; }
    s1 = min(s0 + 1, src - 1);
    w0 = __fsub_rn(1.f, f);
    w1 = f;
}

__device__ __forceinline__ float alpha_at(const vmb_planes_to_image_args& a, int y, int x) {
    const int64_t i = y * a.alpha_rs + x * a.alpha_ps;
    return __fdiv_rn(a.alpha_u16 ? load_px<true>(a.alpha_src, i) : load_px<false>(a.alpha_src, i), a.max_range);
}

template <bool U16, typename in_t>
__global__ void __launch_bounds__(256) planes_to_image_kernel(const vmb_planes_to_image_args a) {
    pdl_trigger();
    pdl_wait();
    const int x = blockIdx.x * kTx + threadIdx.x, y = blockIdx.y * kTy + threadIdx.y;
    if (x >= a.W || y >= a.H) return;
    const in_t* p = reinterpret_cast<const in_t*>(a.planes) + y * a.p_rs + x;
    auto ld = [&](int b, int c) { return fminf(fmaxf(to_f32<in_t>(p[b * a.p_bs + c * a.p_cs]), 0.f), 1.f); };
    float v[4];
    v[0] = ld(0, 2); v[1] = ld(0, 1); v[2] = ld(0, 0);  // BGR
    int nc = 3;
    if (a.channels == 1) {
        v[0] = gray_bgr(v[0], v[1], v[2]);
        nc = 1;
    } else if (a.channels == 4) {
        if (a.alpha_mode == 0) {
            v[3] = gray_bgr(ld(1, 2), ld(1, 1), ld(1, 0));
        } else {
            int x0, x1, y0, y1;
            float a0, a1, b0, b1;
            linear_taps(x, a.W, a.alpha_W, x0, x1, a0, a1);
            linear_taps(y, a.H, a.alpha_H, y0, y1, b0, b1);
            const float r0 = __fadd_rn(__fmul_rn(alpha_at(a, y0, x0), a0), __fmul_rn(alpha_at(a, y0, x1), a1));
            const float r1 = __fadd_rn(__fmul_rn(alpha_at(a, y1, x0), a0), __fmul_rn(alpha_at(a, y1, x1), a1));
            v[3] = __fadd_rn(__fmul_rn(r0, b0), __fmul_rn(r1, b1));
        }
        nc = 4;
    }
    const int64_t o = y * a.out_rs + x * a.out_ps;
    for (int c = 0; c < nc; ++c) {
        const float r = rintf(__fmul_rn(v[c], a.max_range));
        if (U16) reinterpret_cast<uint16_t*>(a.out)[o + c] = (uint16_t)fminf(fmaxf(r, 0.f), 65535.f);
        else reinterpret_cast<uint8_t*>(a.out)[o + c] = (uint8_t)fminf(fmaxf(r, 0.f), 255.f);
    }
}

// ---- Lanczos-4 resize ----
// interpolateLanczos4 (resize.cpp): sin / cos in double, the eight weights in float, normalised by their float sum
__device__ void lanczos4_coeffs(float x, float* c) {
    constexpr double s45 = 0.70710678118654752440084436210485, pi = 3.1415926535897932384626433832795;
    const double cs[8][2] = {{1, 0}, {-s45, -s45}, {0, 1}, {s45, -s45}, {-1, 0}, {s45, s45}, {0, -1}, {-s45, s45}};
    const float x3 = __fadd_rn(x, 3.f);
    const double y0 = __dmul_rn(__dmul_rn(-(double)x3, pi), 0.25);
    double s0, c0;
    sincos(y0, &s0, &c0);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const float yi = __fsub_rn(x3, (float)i);
        if (fabsf(yi) >= 1e-6f) {
            const double y = __dmul_rn(__dmul_rn(-(double)yi, pi), 0.25);
            c[i] = __double2float_rn(__ddiv_rn(__dadd_rn(__dmul_rn(cs[i][0], s0), __dmul_rn(cs[i][1], c0)), __dmul_rn(y, y)));
        } else {
            c[i] = 1e30f;
        }
        sum = __fadd_rn(sum, c[i]);
    }
    const float inv = __fdiv_rn(1.f, sum);
#pragma unroll
    for (int i = 0; i < 8; ++i) c[i] = __fmul_rn(c[i], inv);
}

struct Taps {
    int s;         // first tap: floor(sample) - 3 (clamped per tap)
    float w[8];    // float weights (16-bit images)
    int iw[8];     // 11-bit fixed-point weights (8-bit images)
};

__device__ __noinline__ void lanczos_taps(int d, int dst, int src, Taps& t) {
    float f;
    src_pos(d, dst, src, t.s, f);
    t.s -= 3;
    lanczos4_coeffs(f, t.w);
#pragma unroll
    for (int i = 0; i < 8; ++i) t.iw[i] = max(-32768, min(32767, __float2int_rn(__fmul_rn(t.w[i], 2048.f))));  // saturate_cast<short>
}

template <bool U16>
__global__ void __launch_bounds__(256) resize_lanczos4_kernel(const vmb_resize_lanczos4_args a) {
    __shared__ Taps tx[kTx], ty[kTy];
    pdl_trigger();
    const int x = blockIdx.x * kTx + threadIdx.x, y = blockIdx.y * kTy + threadIdx.y;
    if (threadIdx.y == 0 && x < a.dW) lanczos_taps(x, a.dW, a.sW, tx[threadIdx.x]);
    if (threadIdx.y == 1 && threadIdx.x < kTy && blockIdx.y * kTy + threadIdx.x < a.dH)
        lanczos_taps(blockIdx.y * kTy + threadIdx.x, a.dH, a.sH, ty[threadIdx.x]);
    __syncthreads();
    pdl_wait();
    if (x >= a.dW || y >= a.dH) return;
    const Taps& X = tx[threadIdx.x];
    const Taps& Y = ty[threadIdx.y];
    int64_t xo[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) xo[j] = (int64_t)min(max(X.s + j, 0), a.sW - 1) * a.src_ps;
    const int64_t o = y * a.dst_rs + x * a.dst_ps;
    for (int c = 0; c < a.channels; ++c) {
        if (U16) {
            float acc = 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int64_t row = (int64_t)min(max(Y.s + k, 0), a.sH - 1) * a.src_rs + c;
                float h = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) h = __fadd_rn(h, __fmul_rn(load_px<true>(a.src, row + xo[j]), X.w[j]));
                acc = k == 0 ? __fmul_rn(h, Y.w[0]) : __fadd_rn(acc, __fmul_rn(h, Y.w[k]));
            }
            reinterpret_cast<uint16_t*>(a.dst)[o + c] = (uint16_t)fminf(fmaxf(rintf(acc), 0.f), 65535.f);
        } else {
            uint32_t acc = 0;  // OpenCV's int sums, wrapping as its int32 arithmetic does
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const int64_t row = (int64_t)min(max(Y.s + k, 0), a.sH - 1) * a.src_rs + c;
                int h = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) h += (int)reinterpret_cast<const uint8_t*>(a.src)[row + xo[j]] * X.iw[j];
                acc += (uint32_t)h * (uint32_t)Y.iw[k];
            }
            const int r = (int)(acc + (1u << 21)) >> 22;
            reinterpret_cast<uint8_t*>(a.dst)[o + c] = (uint8_t)max(0, min(255, r));
        }
    }
}

dim3 grid2(int W, int H) { return dim3((unsigned)cdiv(W, kTx), (unsigned)cdiv(H, kTy)); }

}  // namespace

bool image_strides_ok(int H, int W, int channels, int64_t rs, int64_t ps, int64_t cs) {
    return H > 0 && W > 0 && rs >= 0 && ps >= 0 && cs >= 0 && (int64_t)(H - 1) * rs + (int64_t)(W - 1) * ps + (channels - 1) * cs < (1LL << 40);
}

int image_max_launch(const vmb_image_max_args& a, cudaStream_t stream) {
    VMB_CUDA(cudaMemsetAsync(a.max_out, 0, sizeof(unsigned int), stream));
    const dim3 grid((unsigned)cdiv(a.W, kTx), (unsigned)min(cdiv(a.H, kTy), 1024));
    if (a.u16) VMB_CUDA(launch_pdl(image_max_kernel<true>, grid, dim3(kTx, kTy), 0, stream, a));
    else VMB_CUDA(launch_pdl(image_max_kernel<false>, grid, dim3(kTx, kTy), 0, stream, a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

template <bool U16>
static cudaError_t to_planes_dt(const vmb_image_to_planes_args& a, int Hp, int Wp, cudaStream_t s) {
    const dim3 g = grid2(Wp, Hp), b(kTx, kTy);
    switch (a.dtype) {
        case VMB_BF16: return launch_pdl(image_to_planes_kernel<U16, __nv_bfloat16>, g, b, 0, s, a, Hp, Wp);
        case VMB_F16: return launch_pdl(image_to_planes_kernel<U16, __half>, g, b, 0, s, a, Hp, Wp);
        default: return launch_pdl(image_to_planes_kernel<U16, float>, g, b, 0, s, a, Hp, Wp);
    }
}

int image_to_planes_launch(const vmb_image_to_planes_args& a, int Hp, int Wp, cudaStream_t stream) {
    VMB_CUDA(a.u16 ? to_planes_dt<true>(a, Hp, Wp, stream) : to_planes_dt<false>(a, Hp, Wp, stream));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

template <bool U16>
static cudaError_t to_image_dt(const vmb_planes_to_image_args& a, cudaStream_t s) {
    const dim3 g = grid2(a.W, a.H), b(kTx, kTy);
    switch (a.dtype) {
        case VMB_BF16: return launch_pdl(planes_to_image_kernel<U16, __nv_bfloat16>, g, b, 0, s, a);
        case VMB_F16: return launch_pdl(planes_to_image_kernel<U16, __half>, g, b, 0, s, a);
        default: return launch_pdl(planes_to_image_kernel<U16, float>, g, b, 0, s, a);
    }
}

int planes_to_image_launch(const vmb_planes_to_image_args& a, cudaStream_t stream) {
    VMB_CUDA(a.u16 ? to_image_dt<true>(a, stream) : to_image_dt<false>(a, stream));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

int resize_lanczos4_launch(const vmb_resize_lanczos4_args& a, cudaStream_t stream) {
    const dim3 g = grid2(a.dW, a.dH), b(kTx, kTy);
    if (a.u16) VMB_CUDA(launch_pdl(resize_lanczos4_kernel<true>, g, b, 0, stream, a));
    else VMB_CUDA(launch_pdl(resize_lanczos4_kernel<false>, g, b, 0, stream, a));
    VMB_CUDA(cudaGetLastError());
    return VMB_OK;
}

}  // namespace vmb

using namespace vmb;

static bool valid_channels(int c) { return c == 1 || c == 3 || c == 4; }

extern "C" int vmb_image_max(const vmb_image_max_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->img && a->max_out, "image_max: null pointer");
    VMB_CHECK(valid_channels(a->channels) && (a->u16 == 0 || a->u16 == 1), "image_max: channels must be 1, 3 or 4 and u16 0 or 1");
    VMB_CHECK(image_strides_ok(a->H, a->W, a->channels, a->row_stride, a->pixel_stride, a->channel_stride), "image_max: bad size or strides");
    return image_max_launch(*a, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_image_to_planes(const vmb_image_to_planes_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->img && a->out, "image_to_planes: null pointer");
    VMB_CHECK(valid_channels(a->channels) && (a->u16 == 0 || a->u16 == 1), "image_to_planes: channels must be 1, 3 or 4 and u16 0 or 1");
    VMB_CHECK(a->dtype == VMB_F32 || a->dtype == VMB_BF16 || a->dtype == VMB_F16, "image_to_planes: dtype must be f32/bf16/f16 (got %d)", a->dtype);
    VMB_CHECK(a->alpha_plane == 0 || (a->alpha_plane == 1 && a->channels == 4), "image_to_planes: alpha_plane needs a 4-channel image");
    VMB_CHECK(a->max_range > 0.f, "image_to_planes: max_range must be positive");
    VMB_CHECK(image_strides_ok(a->H, a->W, a->channels, a->row_stride, a->pixel_stride, a->channel_stride), "image_to_planes: bad size or strides");
    int Hp = a->H, Wp = a->W;
    for (int i = 0; i < 3; ++i) {
        VMB_CHECK(a->pad_h[i] >= 0 && a->pad_h[i] < Hp && a->pad_w[i] >= 0 && a->pad_w[i] < Wp,
                  "image_to_planes: reflect pad %d (%d, %d) must be smaller than the size it pads (%d, %d)", i, a->pad_h[i], a->pad_w[i], Hp, Wp);
        Hp += a->pad_h[i];
        Wp += a->pad_w[i];
    }
    return image_to_planes_launch(*a, Hp, Wp, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_planes_to_image(const vmb_planes_to_image_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->planes && a->out, "planes_to_image: null pointer");
    VMB_CHECK(valid_channels(a->channels) && (a->u16 == 0 || a->u16 == 1), "planes_to_image: channels must be 1, 3 or 4 and u16 0 or 1");
    VMB_CHECK(a->dtype == VMB_F32 || a->dtype == VMB_BF16 || a->dtype == VMB_F16, "planes_to_image: dtype must be f32/bf16/f16 (got %d)", a->dtype);
    VMB_CHECK(a->H > 0 && a->W > 0 && a->out_rs >= 0 && a->out_ps >= a->channels, "planes_to_image: bad size or output strides");
    VMB_CHECK(a->max_range > 0.f, "planes_to_image: max_range must be positive");
    VMB_CHECK(a->alpha_mode == 0 || a->alpha_mode == 1, "planes_to_image: alpha_mode must be 0 or 1");
    VMB_CHECK(a->channels != 4 || a->alpha_mode == 0 ||
                  (a->alpha_src && image_strides_ok(a->alpha_H, a->alpha_W, 1, a->alpha_rs, a->alpha_ps, 0)),
              "planes_to_image: alpha_mode 1 needs an alpha source image");
    return planes_to_image_launch(*a, static_cast<cudaStream_t>(stream));
}

extern "C" int vmb_resize_lanczos4(const vmb_resize_lanczos4_args* a, void* stream) {
    VMB_CHECK(a != nullptr && a->src && a->dst, "resize_lanczos4: null pointer");
    VMB_CHECK(valid_channels(a->channels) && (a->u16 == 0 || a->u16 == 1), "resize_lanczos4: channels must be 1, 3 or 4 and u16 0 or 1");
    VMB_CHECK(a->dH > 0 && a->dW > 0 && a->dH < 65535 * kTy && a->dst_ps >= a->channels && a->dst_rs >= 0, "resize_lanczos4: bad output size or strides");
    VMB_CHECK(image_strides_ok(a->sH, a->sW, a->channels, a->src_rs, a->src_ps, 1), "resize_lanczos4: bad source size or strides");
    return resize_lanczos4_launch(*a, static_cast<cudaStream_t>(stream));
}
