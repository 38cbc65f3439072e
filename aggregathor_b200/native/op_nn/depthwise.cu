// Depthwise k x k convolution (one filter per channel), NHWC bf16 activations, TF "SAME"-style explicit padding, stride s:
// forward, data gradient (gather form) and weight gradient (per logical worker). A depthwise filter has no GEMM shape — every
// output is a k*k-term dot product per channel — so these are bandwidth kernels: 128-bit vectors along C, one CTA row per image
// row (grid.y), filter taps read from a [k*k, C] transposed copy of the weights so that a thread's 8 channels are one 16-byte load.
// Used by the MobileNet / NASNet / PNASNet separable convolutions (reference: the slim nets behind `nets_factory.py:39-72`).

#include <cuda_bf16.h>

#include <agb_device.cuh>

using namespace agb;

namespace {

using bf16 = __nv_bfloat16;
constexpr int kThreads = 256;

__device__ __forceinline__ void unpack8(uint4 const& raw, float (&v)[8]) {
    __nv_bfloat162 const* h = reinterpret_cast<__nv_bfloat162 const*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        float2 f = __bfloat1622float2(h[i]);
        v[2 * i] = f.x;
        v[2 * i + 1] = f.y;
    }
}
__device__ __forceinline__ uint4 pack8(float const (&v)[8]) {
    uint4 raw;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&raw);
#pragma unroll
    for (int i = 0; i < 4; ++i)
        h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
    return raw;
}

struct Geometry {
    int N, H, W, C, OH, OW, k, s, pad_t, pad_l;
};

// y[n, oh, ow, c] = sum_{kh, kw} x[n, oh*s + kh - pad_t, ow*s + kw - pad_l, c] * w[kh*k + kw][c]
__global__ void __launch_bounds__(kThreads) depthwise_fwd_kernel(bf16 const* __restrict__ x, bf16 const* __restrict__ wt, bf16* __restrict__ y, Geometry const g, int first_image) {
    pdl_trigger();
    pdl_wait();
    int const octets = g.C >> 3;
    int const n = first_image + blockIdx.y / g.OH, oh = blockIdx.y % g.OH;
    uint4* const out_row = reinterpret_cast<uint4*>(y) + (static_cast<long long>(n) * g.OH + oh) * g.OW * octets;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g.OW * octets; i += gridDim.x * blockDim.x) {
        int const ow = i / octets, o = i - ow * octets;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int kh = 0; kh < g.k; ++kh) {
            int const ih = oh * g.s + kh - g.pad_t;
            if (ih < 0 || ih >= g.H)
                continue;
            for (int kw = 0; kw < g.k; ++kw) {
                int const iw = ow * g.s + kw - g.pad_l;
                if (iw < 0 || iw >= g.W)
                    continue;
                float vx[8], vw[8];
                unpack8(reinterpret_cast<uint4 const*>(x)[((static_cast<long long>(n) * g.H + ih) * g.W + iw) * octets + o], vx);
                unpack8(reinterpret_cast<uint4 const*>(wt)[static_cast<long long>(kh * g.k + kw) * octets + o], vw);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    acc[j] += vx[j] * vw[j];
            }
        }
        out_row[i] = pack8(acc);
    }
}

// dx[n, h, w, c] = sum over the windows (oh, ow, kh, kw) that read pixel (h, w): dy[n, oh, ow, c] * w[kh*k + kw][c]
__global__ void __launch_bounds__(kThreads) depthwise_dgrad_kernel(bf16 const* __restrict__ dy, bf16 const* __restrict__ wt, bf16* __restrict__ dx, Geometry const g, int first_image) {
    pdl_trigger();
    pdl_wait();
    int const octets = g.C >> 3;
    int const n = first_image + blockIdx.y / g.H, h = blockIdx.y % g.H;
    uint4* const out_row = reinterpret_cast<uint4*>(dx) + (static_cast<long long>(n) * g.H + h) * g.W * octets;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g.W * octets; i += gridDim.x * blockDim.x) {
        int const w = i / octets, o = i - w * octets;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int kh = 0; kh < g.k; ++kh) {
            int const th = h + g.pad_t - kh;
            if (th < 0 || th % g.s)
                continue;
            int const oh = th / g.s;
            if (oh >= g.OH)
                continue;
            for (int kw = 0; kw < g.k; ++kw) {
                int const tw = w + g.pad_l - kw;
                if (tw < 0 || tw % g.s)
                    continue;
                int const ow = tw / g.s;
                if (ow >= g.OW)
                    continue;
                float vd[8], vw[8];
                unpack8(reinterpret_cast<uint4 const*>(dy)[((static_cast<long long>(n) * g.OH + oh) * g.OW + ow) * octets + o], vd);
                unpack8(reinterpret_cast<uint4 const*>(wt)[static_cast<long long>(kh * g.k + kw) * octets + o], vw);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    acc[j] += vd[j] * vw[j];
            }
        }
        out_row[i] = pack8(acc);
    }
}

// dw[group][c][kh][kw] += sum over the output positions of the group's images of dy[n, oh, ow, c] * x[n, oh*s + kh - pad_t, ow*s + kw - pad_l, c].
// One thread per (tap, channel octet) (consecutive threads = consecutive octets: coalesced), grid.y slices the positions of a group,
// grid.z = group; per-thread fp32 partial sums, then one fp32 atomic per (channel, tap) and CTA into the zero-initialised gradient.
__global__ void __launch_bounds__(kThreads) depthwise_wgrad_kernel(bf16 const* __restrict__ dy, bf16 const* __restrict__ x, float* __restrict__ dw, Geometry const g,
                                                                   int images_per_group, long long group_stride, int positions_per_cta) {
    pdl_trigger();
    pdl_wait();
    int const octets = g.C >> 3, taps = g.k * g.k;
    int const t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= taps * octets)
        return;
    int const tap = t / octets, o = t - tap * octets;
    int const kh = tap / g.k, kw = tap - kh * g.k;
    int const group = blockIdx.z;
    long long const per_image = static_cast<long long>(g.OH) * g.OW;
    long long const total = per_image * images_per_group;
    long long const begin = static_cast<long long>(blockIdx.y) * positions_per_cta;
    long long const end = begin + positions_per_cta < total ? begin + positions_per_cta : total;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (long long p = begin; p < end; ++p) {
        int const local_image = static_cast<int>(p / per_image);
        int const rem = static_cast<int>(p - local_image * per_image);
        int const oh = rem / g.OW, ow = rem - oh * g.OW;
        int const ih = oh * g.s + kh - g.pad_t, iw = ow * g.s + kw - g.pad_l;
        if (ih < 0 || ih >= g.H || iw < 0 || iw >= g.W)
            continue;
        long long const n = static_cast<long long>(group) * images_per_group + local_image;
        float vd[8], vx[8];
        unpack8(reinterpret_cast<uint4 const*>(dy)[((n * g.OH + oh) * g.OW + ow) * octets + o], vd);
        unpack8(reinterpret_cast<uint4 const*>(x)[((n * g.H + ih) * g.W + iw) * octets + o], vx);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            acc[j] += vd[j] * vx[j];
    }
    float* const out = dw + group * group_stride;
#pragma unroll
    for (int j = 0; j < 8; ++j)
        atomicAdd(out + static_cast<long long>(o * 8 + j) * taps + tap, acc[j]);
}

int check(Geometry const& g) {
    if ((g.C & 7) || g.k < 1 || g.k > 15 || g.s < 1 || g.N < 1 || g.H > 65535 || g.OH > 65535)
        return 301;
    return 0;
}

} // namespace

extern "C" {

// wt: bf16 [k*k, C] (the [C, k, k] filters transposed); x: [N, H, W, C]; y: [N, OH, OW, C].
int agb_depthwise_forward(void const* x, void const* wt, void* y, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    Geometry const g{N, H, W, C, OH, OW, k, s, pad_t, pad_l};
    if (int status = check(g))
        return status;
    int const per_launch = 65535 / OH;   // grid.y = images x rows
    for (int n0 = 0; n0 < N; n0 += per_launch) {
        int const count = N - n0 < per_launch ? N - n0 : per_launch;
        AGB_CUDA_OK(launch_pdl(depthwise_fwd_kernel, dim3((OW * (C >> 3) + kThreads - 1) / kThreads, count * OH), dim3(kThreads), 0, static_cast<cudaStream_t>(stream),
                               static_cast<bf16 const*>(x), static_cast<bf16 const*>(wt), static_cast<bf16*>(y), g, n0));
    }
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

int agb_depthwise_dgrad(void const* dy, void const* wt, void* dx, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    Geometry const g{N, H, W, C, OH, OW, k, s, pad_t, pad_l};
    if (int status = check(g))
        return status;
    int const per_launch = 65535 / H;
    for (int n0 = 0; n0 < N; n0 += per_launch) {
        int const count = N - n0 < per_launch ? N - n0 : per_launch;
        AGB_CUDA_OK(launch_pdl(depthwise_dgrad_kernel, dim3((W * (C >> 3) + kThreads - 1) / kThreads, count * H), dim3(kThreads), 0, static_cast<cudaStream_t>(stream),
                               static_cast<bf16 const*>(dy), static_cast<bf16 const*>(wt), static_cast<bf16*>(dx), g, n0));
    }
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

// dw: fp32 [C, k, k] per group, `group_stride` elements apart, ZERO on entry (accumulated with atomics).
int agb_depthwise_wgrad(void const* dy, void const* x, void* dw, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, int groups, long long group_stride,
                        void* stream) {
    Geometry const g{N, H, W, C, OH, OW, k, s, pad_t, pad_l};
    if (int status = check(g))
        return status;
    if (groups < 1 || N % groups)
        return 301;
    int const images = N / groups;
    long long const positions = static_cast<long long>(images) * OH * OW;
    int const threads_needed = k * k * (C >> 3);
    int const ctas_x = (threads_needed + kThreads - 1) / kThreads;
    long long slices = (static_cast<long long>(agb::sm_count()) * 4 + ctas_x * groups - 1) / (static_cast<long long>(ctas_x) * groups);   // ~4 CTAs per SM overall
    if (slices > positions)
        slices = positions;
    if (slices < 1)
        slices = 1;
    if (slices > 65535)
        slices = 65535;
    int const per_cta = static_cast<int>((positions + slices - 1) / slices);
    AGB_CUDA_OK(launch_pdl(depthwise_wgrad_kernel, dim3(ctas_x, static_cast<unsigned>((positions + per_cta - 1) / per_cta), groups), dim3(kThreads), 0, static_cast<cudaStream_t>(stream),
                           static_cast<bf16 const*>(dy), static_cast<bf16 const*>(x), static_cast<float*>(dw), g, images, group_stride, per_cta));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

} // extern "C"

// ---------------------------------------------------------------------------- //
// Average pooling with TF "SAME" semantics (the divisor counts only the pixels inside the image) and ReLU6 — the remaining
// element-wise layers of the Inception / MobileNet / NASNet graphs.

namespace {

// y[n, oh, ow, c] = mean over the in-image pixels of the k x k window at (oh*s - pad_t, ow*s - pad_l)
__global__ void __launch_bounds__(kThreads) avgpool2d_fwd_kernel(bf16 const* __restrict__ x, bf16* __restrict__ y, Geometry const g, int first_image) {
    pdl_trigger();
    pdl_wait();
    int const octets = g.C >> 3;
    int const n = first_image + blockIdx.y / g.OH, oh = blockIdx.y % g.OH;
    int const h0 = max(0, oh * g.s - g.pad_t), h1 = min(g.H, oh * g.s - g.pad_t + g.k);
    uint4* const out_row = reinterpret_cast<uint4*>(y) + (static_cast<long long>(n) * g.OH + oh) * g.OW * octets;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g.OW * octets; i += gridDim.x * blockDim.x) {
        int const ow = i / octets, o = i - ow * octets;
        int const w0 = max(0, ow * g.s - g.pad_l), w1 = min(g.W, ow * g.s - g.pad_l + g.k);
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int ih = h0; ih < h1; ++ih)
            for (int iw = w0; iw < w1; ++iw) {
                float v[8];
                unpack8(reinterpret_cast<uint4 const*>(x)[((static_cast<long long>(n) * g.H + ih) * g.W + iw) * octets + o], v);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    acc[j] += v[j];
            }
        float const inv = 1.f / static_cast<float>(max(1, (h1 - h0) * (w1 - w0)));
#pragma unroll
        for (int j = 0; j < 8; ++j)
            acc[j] *= inv;
        out_row[i] = pack8(acc);
    }
}

// dx[n, h, w, c] = sum over the windows containing (h, w) of dy[n, oh, ow, c] / (in-image size of that window)
__global__ void __launch_bounds__(kThreads) avgpool2d_bwd_kernel(bf16 const* __restrict__ dy, bf16* __restrict__ dx, Geometry const g, int first_image) {
    pdl_trigger();
    pdl_wait();
    int const octets = g.C >> 3;
    int const n = first_image + blockIdx.y / g.H, h = blockIdx.y % g.H;
    uint4* const out_row = reinterpret_cast<uint4*>(dx) + (static_cast<long long>(n) * g.H + h) * g.W * octets;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < g.W * octets; i += gridDim.x * blockDim.x) {
        int const w = i / octets, o = i - w * octets;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int kh = 0; kh < g.k; ++kh) {
            int const th = h + g.pad_t - kh;
            if (th < 0 || th % g.s)
                continue;
            int const oh = th / g.s;
            if (oh >= g.OH)
                continue;
            int const rows = min(g.H, oh * g.s - g.pad_t + g.k) - max(0, oh * g.s - g.pad_t);
            for (int kw = 0; kw < g.k; ++kw) {
                int const tw = w + g.pad_l - kw;
                if (tw < 0 || tw % g.s)
                    continue;
                int const ow = tw / g.s;
                if (ow >= g.OW)
                    continue;
                int const cols = min(g.W, ow * g.s - g.pad_l + g.k) - max(0, ow * g.s - g.pad_l);
                float v[8];
                unpack8(reinterpret_cast<uint4 const*>(dy)[((static_cast<long long>(n) * g.OH + oh) * g.OW + ow) * octets + o], v);
                float const inv = 1.f / static_cast<float>(max(1, rows * cols));
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    acc[j] += v[j] * inv;
            }
        }
        out_row[i] = pack8(acc);
    }
}

// forward: y = min(max(x, 0), 6); backward: dx = dy where 0 < x < 6
__global__ void __launch_bounds__(kThreads) relu6_kernel(bf16 const* __restrict__ x, bf16 const* __restrict__ dy, bf16* __restrict__ out, long long octets) {
    pdl_trigger();
    pdl_wait();
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (; i < octets; i += stride) {
        float v[8];
        unpack8(reinterpret_cast<uint4 const*>(x)[i], v);
        if (dy) {
            float d[8];
            unpack8(reinterpret_cast<uint4 const*>(dy)[i], d);
#pragma unroll
            for (int j = 0; j < 8; ++j)
                v[j] = (v[j] > 0.f && v[j] < 6.f) ? d[j] : 0.f;
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                v[j] = min_nan(max_nan(v[j], 0.f), 6.f);
        }
        reinterpret_cast<uint4*>(out)[i] = pack8(v);
    }
}

} // namespace

extern "C" {

int agb_avgpool2d_forward(void const* x, void* y, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    Geometry const g{N, H, W, C, OH, OW, k, s, pad_t, pad_l};
    if (int status = check(g))
        return status;
    int const per_launch = 65535 / OH;
    for (int n0 = 0; n0 < N; n0 += per_launch) {
        int const count = N - n0 < per_launch ? N - n0 : per_launch;
        AGB_CUDA_OK(launch_pdl(avgpool2d_fwd_kernel, dim3((OW * (C >> 3) + kThreads - 1) / kThreads, count * OH), dim3(kThreads), 0, static_cast<cudaStream_t>(stream),
                               static_cast<bf16 const*>(x), static_cast<bf16*>(y), g, n0));
    }
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

int agb_avgpool2d_backward(void const* dy, void* dx, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    Geometry const g{N, H, W, C, OH, OW, k, s, pad_t, pad_l};
    if (int status = check(g))
        return status;
    int const per_launch = 65535 / H;
    for (int n0 = 0; n0 < N; n0 += per_launch) {
        int const count = N - n0 < per_launch ? N - n0 : per_launch;
        AGB_CUDA_OK(launch_pdl(avgpool2d_bwd_kernel, dim3((W * (C >> 3) + kThreads - 1) / kThreads, count * H), dim3(kThreads), 0, static_cast<cudaStream_t>(stream),
                               static_cast<bf16 const*>(dy), static_cast<bf16*>(dx), g, n0));
    }
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

// dy == null: forward clamp of x; otherwise the backward mask applied to dy.
int agb_relu6(void const* x, void const* dy, void* out, long long n, void* stream) {
    if (n & 7)
        return 301;
    long long const octets = n / 8;
    long long blocks = (octets + kThreads - 1) / kThreads;
    if (blocks > agb::sm_count() * 16)
        blocks = agb::sm_count() * 16;
    AGB_CUDA_OK(launch_pdl(relu6_kernel, dim3(static_cast<unsigned>(blocks < 1 ? 1 : blocks)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<bf16 const*>(x),
                           static_cast<bf16 const*>(dy), static_cast<bf16*>(out), octets));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

} // extern "C"
