// Memory-bound layer kernels (sm_90a), NHWC bf16 activations, fp32 parameters/statistics:
// batch-norm (training) forward/backward fused with ReLU, residual add + ReLU, ReLU backward, 3x3/2-style max-pool
// forward/backward, global average pool, softmax cross-entropy forward+backward, column sums (bias gradients),
// uint8 image normalisation, im2col / col2im for the k x k convolutions that run as GEMMs.
//
// Every tensor is viewed as rows x channels (rows = N*H*W); channels are the contiguous dimension, so all kernels
// read/write 128-bit vectors along C. Per-channel reductions (BN statistics, bias gradients) accumulate per-thread
// fp32 partials over a row strip, combine them per CTA in shared memory and finish with one fp64 atomic per channel and CTA.
// `groups` splits the rows into equal consecutive groups with independent statistics: one group per logical worker, so that
// several workers' batches can share one launch while keeping per-worker BatchNorm semantics.

#include <cmath>

#include <cuda_bf16.h>

#include <agb_device.cuh>

using namespace agb;

namespace {

using bf16 = __nv_bfloat16;

// Activations are bf16 (default) or fp32 (the TF32 parity path: fp32 storage, `kind::tf32` products). Every kernel handles 8
// consecutive channels per thread: one 16-byte vector of bf16, two of fp32.
template<typename T> struct Oct;
template<> struct alignas(16) Oct<bf16> { uint4 raw; };
template<> struct alignas(16) Oct<float> { float4 lo, hi; };

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
__device__ __forceinline__ void unpack8(Oct<bf16> const& o, float (&v)[8]) { unpack8(o.raw, v); }
__device__ __forceinline__ void unpack8(Oct<float> const& o, float (&v)[8]) {
    v[0] = o.lo.x; v[1] = o.lo.y; v[2] = o.lo.z; v[3] = o.lo.w; v[4] = o.hi.x; v[5] = o.hi.y; v[6] = o.hi.z; v[7] = o.hi.w;
}
template<typename T> __device__ __forceinline__ Oct<T> pack_oct(float const (&v)[8]);
template<> __device__ __forceinline__ Oct<bf16> pack_oct<bf16>(float const (&v)[8]) { return Oct<bf16>{pack8(v)}; }
template<> __device__ __forceinline__ Oct<float> pack_oct<float>(float const (&v)[8]) {
    return Oct<float>{make_float4(v[0], v[1], v[2], v[3]), make_float4(v[4], v[5], v[6], v[7])};
}
template<typename T> __device__ __forceinline__ Oct<T> zero_oct() {
    float const z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    return pack_oct<T>(z);
}
template<typename T> __device__ __forceinline__ Oct<T> load_oct(T const* p) { return *reinterpret_cast<Oct<T> const*>(p); }
template<typename T> __device__ __forceinline__ void store_oct(T* p, Oct<T> const& o) { *reinterpret_cast<Oct<T>*>(p) = o; }
__device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_f(float v) { return v; }
template<typename T> __device__ __forceinline__ T from_f(float v);
template<> __device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16(v); }
template<> __device__ __forceinline__ float from_f<float>(float v) { return v; }

// ReLU mask of a batch norm recomputed from its input. The forward stored y = T(max_nan(fma(x, scale, shift) + residual, 0)) with
// no residual, so y > 0 exactly when T(fma(x, scale, shift)) > 0: NaN is masked, and so is a positive value that rounds to zero in T.
template<typename T> __device__ __forceinline__ bool relu_kept(float x, float scale, float shift) {
    return to_f(from_f<T>(fmaf(x, scale, shift))) > 0.f;
}

constexpr int kThreads = 256;

// ---------------------------------------------------------------------------- //
// Per-channel (and per-group) sums: out[g][c] += sum_r f(...). MODE 0: (x - p, (x - p)^2) with the pivot p = the group's first row,
// so that E[x^2] - E[x]^2 stays well conditioned in fp32 even when |mean| >> std; MODE 1: (dy', dy' * xhat) with
// dy' = dy masked by (y > 0) when y != null, or by the mask recomputed from x with the forward's coefficients `msc` / `msh`
// (relu_kept) when those are given; MODE 2: (dy') only (bias gradient). C % 8 == 0. MODE 1 with y and `dmasked` also stores dy' to
// `dmasked` (dy or +0, the gradient of the residual input of a fused add + ReLU), so that the apply kernel reads it instead of dy and y.
// 2-D decomposition: blockIdx.x = row chunk, blockIdx.y = strip of STRIP octets (8 * STRIP channels), blockIdx.z = group.
// Inside a CTA, STRIP lanes cover the strip's octets (up to 512 contiguous bytes per row: whole DRAM bursts instead of
// 128-byte columns) and 256 / STRIP lanes cover rows, several rows in flight per thread; one fp64 atomic per channel and
// CTA, so an address only sees (#row chunks) atomics.
constexpr int kRowUnroll = 4;   // rows in flight per thread: MODE 0 / 2, and MODE 1 (three tensors) in bf16; MODE 1 in fp32 uses 2

// Finalisation performed by the LAST CTA of the statistics kernel (atomic ticket): no separate launch.
struct SumsFinalize {
    unsigned* ticket;           // zero-initialised counter, reset by the last CTA
    float const* gamma;
    float const* beta;
    float* save_mean;           // MODE 0 out / MODE 1 in
    float* save_rstd;
    float* scale;               // MODE 0: [groups*C] ; MODE 1: coef [groups*C*3]
    float* shift;
    float* moving_mean;
    float* moving_var;
    float* dgamma;              // MODE 1
    float* dbeta;               // MODE 1 ; MODE 2: the fp32 column sums
    int groups;
    long long group_stride;     // elements between two groups' parameter gradients (dgamma / dbeta / column sums)
    float eps, decay;
};

template<int MODE, typename T>
__device__ void finalize_sums(double* sums, SumsFinalize const& f, int C, long long rows_per_group, T const* x) {
    double const n = static_cast<double>(rows_per_group), inv_n = 1.0 / n;
    for (int i = threadIdx.x; i < C * f.groups; i += blockDim.x) {
        int const c = i % C, g = i / C;
        double const s0 = __ldcg(sums + 2 * i), s1 = __ldcg(sums + 2 * i + 1);
        sums[2 * i] = 0.;       // leave the workspace zeroed for the next statistics kernel (no memset between launches)
        sums[2 * i + 1] = 0.;
        if (MODE == 0) {
            double const shifted = s0 * inv_n;
            double const mean = shifted + static_cast<double>(to_f(x[g * rows_per_group * C + c]));
            double var = fma(-shifted, shifted, s1 * inv_n);
            if (var < 0.)
                var = 0.;
            float const rstd = rsqrtf(static_cast<float>(var) + f.eps);
            float const gm = f.gamma ? f.gamma[c] : 1.f;
            f.save_mean[i] = static_cast<float>(mean);
            f.save_rstd[i] = rstd;
            f.scale[i] = gm * rstd;
            f.shift[i] = f.beta[c] - static_cast<float>(mean) * gm * rstd;
            if (f.moving_mean && g == 0) { // unbiased variance in the moving average, as TF's fused batch norm
                double const unbiased = n > 1. ? var * n / (n - 1.) : var;
                f.moving_mean[c] = f.decay * f.moving_mean[c] + (1.f - f.decay) * static_cast<float>(mean);
                f.moving_var[c] = f.decay * f.moving_var[c] + (1.f - f.decay) * static_cast<float>(unbiased);
            }
        } else if (MODE == 1) {
            float const gm = f.gamma ? f.gamma[c] : 1.f, rs = f.save_rstd[i], mu = f.save_mean[i];
            float const inv = static_cast<float>(inv_n);
            float const a = gm * rs;
            float const b = -gm * rs * rs * static_cast<float>(s1) * inv;   // xhat * rs = (x - mu) * rs^2
            f.scale[3 * i] = a;
            f.scale[3 * i + 1] = b;
            f.scale[3 * i + 2] = -gm * rs * static_cast<float>(s0) * inv - b * mu;
            // one gradient per group: each logical worker owns its own dgamma / dbeta
            if (f.dgamma)
                f.dgamma[g * f.group_stride + c] = static_cast<float>(s1);
            f.dbeta[g * f.group_stride + c] = static_cast<float>(s0);
        } else {
            f.dbeta[g * f.group_stride + c] = static_cast<float>(s0);
        }
    }
}

template<typename T, int MODE, int STRIP>
__global__ void __launch_bounds__(kThreads) channel_sums_kernel(T const* __restrict__ a, T const* __restrict__ b, T const* __restrict__ y, T* __restrict__ dmasked,
                                    float const* __restrict__ mean, float const* __restrict__ rstd, float const* __restrict__ msc, float const* __restrict__ msh, double* __restrict__ out,
                                    long long rows_per_group, int C, int rows_per_cta, SumsFinalize const fin) {
    pdl_trigger();
    pdl_wait();
    constexpr int kStripOctets = STRIP, kRowLanes = kThreads / STRIP;
    __shared__ float red[kRowLanes][kStripOctets * 16 + 1];
    __shared__ bool is_last;
    int const octets = C >> 3;
    int const tc = threadIdx.x % kStripOctets, tr = threadIdx.x / kStripOctets;
    int const o = blockIdx.y * kStripOctets + tc;
    int const group = blockIdx.z;
    bool const active = o < octets;
    long long const row_begin = static_cast<long long>(blockIdx.x) * rows_per_cta;
    long long const row_end = min(rows_per_group, row_begin + rows_per_cta);
    long long const base = static_cast<long long>(group) * rows_per_group;
    float s0[8], s1[8], mu[8], rs[8], sc[8], sh[8];
    bool const recompute = MODE == 1 && msc != nullptr;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        s0[j] = 0.f;
        s1[j] = 0.f;
        mu[j] = 0.f;
        rs[j] = 0.f;
        sc[j] = 0.f;
        sh[j] = 0.f;
        if (MODE == 1 && active) {
            mu[j] = mean[group * C + o * 8 + j];
            rs[j] = rstd[group * C + o * 8 + j];
            if (recompute) {
                sc[j] = msc[group * C + o * 8 + j];
                sh[j] = msh[group * C + o * 8 + j];
            }
        }
    }
    if (MODE == 0 && active)
        unpack8(load_oct(a + base * C + o * 8), mu);
    if (active) {
        constexpr int U = MODE == 1 && sizeof(T) == 4 ? 2 : kRowUnroll;   // fp32 MODE 1 at 4 would need 175 registers: 1 CTA per SM
        for (long long r0 = row_begin + tr; r0 < row_end; r0 += kRowLanes * U) {
            Oct<T> ra[U], rb[U], ry[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {   // issue every load of the batch before using any of them
                long long const r = r0 + u * kRowLanes;
                if (r < row_end) {
                    long long const idx = (base + r) * C + o * 8;
                    ra[u] = load_oct(a + idx);
                    if (MODE == 1)
                        rb[u] = load_oct(b + idx);
                    if (MODE != 0 && y)
                        ry[u] = load_oct(y + idx);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                long long const r = r0 + u * kRowLanes;
                if (r < row_end) {
                    float va[8];
                    unpack8(ra[u], va);
                    if (MODE == 0) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            float const d = va[j] - mu[j];
                            s0[j] += d;
                            s1[j] += d * d;
                        }
                    } else {
                        if (y) {
                            float vy[8];
                            unpack8(ry[u], vy);
#pragma unroll
                            for (int j = 0; j < 8; ++j)
                                va[j] = vy[j] > 0.f ? va[j] : 0.f;
                            if (MODE == 1 && dmasked)
                                store_oct(dmasked + (base + r) * C + o * 8, pack_oct<T>(va));
                        }
                        if (MODE == 1) {
                            float vx[8];
                            unpack8(rb[u], vx);
                            if (recompute) {
#pragma unroll
                                for (int j = 0; j < 8; ++j)
                                    va[j] = relu_kept<T>(vx[j], sc[j], sh[j]) ? va[j] : 0.f;
                            }
#pragma unroll
                            for (int j = 0; j < 8; ++j) {
                                s0[j] += va[j];
                                s1[j] += va[j] * (vx[j] - mu[j]) * rs[j];
                            }
                        } else {
#pragma unroll
                            for (int j = 0; j < 8; ++j)
                                s0[j] += va[j];
                        }
                    }
                }
            }
        }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        red[tr][tc * 16 + j] = s0[j];
        red[tr][tc * 16 + 8 + j] = s1[j];
    }
    __syncthreads();
    // STRIP * 16 values per CTA: thread t folds column t over the row lanes in a fixed order
    for (int t = threadIdx.x; t < kStripOctets * 16; t += kThreads) {
        int const oc = t / 16, j = t % 16;
        int const oo = blockIdx.y * kStripOctets + oc;
        if (oo < octets && (MODE != 2 || j < 8)) {
            float total = 0.f;
#pragma unroll
            for (int l = 0; l < kRowLanes; ++l)
                total += red[l][t];
            double* dst = out + (static_cast<long long>(group) * C + oo * 8 + (j & 7)) * 2 + (j >> 3);
            atomicAdd(dst, static_cast<double>(total));
        }
    }
    // last CTA to finish turns the sums into what the apply kernel needs
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned const total_ctas = gridDim.x * gridDim.y * gridDim.z;
        unsigned const ticket = atomicAdd(fin.ticket, 1u);
        is_last = ticket == total_ctas - 1;
        if (is_last)
            *fin.ticket = 0;   // ready for the next launch
    }
    __syncthreads();
    if (is_last) {
        __threadfence();
        finalize_sums<MODE>(out, fin, C, rows_per_group, a);
    }
}

// The apply kernels run `ctas` CTAs per group: CTA k serves group k / ctas, whose octets are a contiguous range. A thread keeps one
// channel octet for its whole loop (the stride is a multiple of `octets`; the host gives each group at least one CTA per 256
// octets), so the group's coefficients stay in registers and no division happens in the loop, and it keeps U independent
// 16-byte loads of each tensor in flight.

// y = relu?(x * scale[g][c] + shift[g][c] (+ residual)).
template<typename T>
__global__ void __launch_bounds__(kThreads) bn_apply_kernel(T const* __restrict__ x, T const* __restrict__ residual, T* __restrict__ y, float const* __restrict__ scale,
                                float const* __restrict__ shift, long long rows_per_group, int C, int ctas, int relu) {
    pdl_trigger();
    pdl_wait();
    unsigned const octets = static_cast<unsigned>(C >> 3);
    int const g = blockIdx.x / ctas;
    long long const nthreads = static_cast<long long>(ctas) * blockDim.x;
    long long const stride = nthreads - nthreads % octets;   // multiple of `octets`: the octet of a thread never changes
    long long i = static_cast<long long>(blockIdx.x - g * ctas) * blockDim.x + threadIdx.x;
    if (i >= stride)
        return;
    unsigned const o = static_cast<unsigned>(i % octets);
    long long const n = rows_per_group * octets;             // octets of the group
    long long const base = static_cast<long long>(g) * n * 8;
    x += base;
    y += base;
    if (residual)
        residual += base;
    float sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        sc[j] = scale[g * C + o * 8 + j];
        sh[j] = shift[g * C + o * 8 + j];
    }
    auto transform = [&](Oct<T> raw, long long index) {   // y = relu?(x * scale + shift (+ residual))
        float v[8], r[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        unpack8(raw, v);
        if (residual)
            unpack8(load_oct(residual + index * 8), r);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            v[j] = v[j] * sc[j] + sh[j] + r[j];
            if (relu)
                v[j] = max_nan(v[j], 0.f);
        }
        return pack_oct<T>(v);
    };
    constexpr int U = 4;   // four independent 16-byte loads in flight per thread
    for (; i + (U - 1) * stride < n; i += U * stride) {
        Oct<T> raw[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
            raw[u] = load_oct(x + (i + u * stride) * 8);
#pragma unroll
        for (int u = 0; u < U; ++u)
            store_oct(y + (i + u * stride) * 8, transform(raw[u], i + u * stride));
    }
    for (; i < n; i += stride)
        store_oct(y + i * 8, transform(load_oct(x + i * 8), i));
}

// dx = a * dy' + b * x + c0 with per-(group, channel) coefficients prepared by the statistics kernel's last CTA; dy' = dy masked by
// y > 0, or by the mask recomputed from x (`msc` / `msh`: the forward's coefficients, relu_kept), or dy when neither is given (also
// when dy is the masked gradient the statistics kernel stored).
template<typename T>
__global__ void __launch_bounds__(kThreads) bn_bwd_apply_kernel(T const* __restrict__ dy, T const* __restrict__ x, T const* __restrict__ y, T* __restrict__ dx,
                                    float const* __restrict__ coef, float const* __restrict__ msc, float const* __restrict__ msh, long long rows_per_group, int C,
                                    int ctas) {
    pdl_trigger();
    pdl_wait();
    unsigned const octets = static_cast<unsigned>(C >> 3);
    int const g = blockIdx.x / ctas;
    long long const nthreads = static_cast<long long>(ctas) * blockDim.x;
    long long const stride = nthreads - nthreads % octets;
    long long i = static_cast<long long>(blockIdx.x - g * ctas) * blockDim.x + threadIdx.x;
    if (i >= stride)
        return;
    unsigned const o = static_cast<unsigned>(i % octets);
    long long const n = rows_per_group * octets;
    long long const base = static_cast<long long>(g) * n * 8;
    bool const masked = y != nullptr, recompute = msc != nullptr;
    dy += base;
    x += base;
    dx += base;
    if (masked)
        y += base;
    float ca[8], cb[8], cc[8], sc[8], sh[8];
    float const* cf = coef + (static_cast<long long>(g) * C + o * 8) * 3;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        ca[j] = cf[3 * j];
        cb[j] = cf[3 * j + 1];
        cc[j] = cf[3 * j + 2];
        sc[j] = recompute ? msc[g * C + o * 8 + j] : 0.f;
        sh[j] = recompute ? msh[g * C + o * 8 + j] : 0.f;
    }
    auto transform = [&](Oct<T> rd, Oct<T> rx, Oct<T> ry) {
        float vd[8], vx[8];
        unpack8(rd, vd);
        unpack8(rx, vx);
        if (recompute) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                vd[j] = relu_kept<T>(vx[j], sc[j], sh[j]) ? vd[j] : 0.f;
        } else if (masked) {
            float vy[8];
            unpack8(ry, vy);
#pragma unroll
            for (int j = 0; j < 8; ++j)
                vd[j] = vy[j] > 0.f ? vd[j] : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j)
            vd[j] = ca[j] * vd[j] + cb[j] * vx[j] + cc[j];
        return pack_oct<T>(vd);
    };
    constexpr int U = sizeof(T) == 2 ? 4 : 2;   // bf16: 4 x 3 loads in flight at the occupancy of 2 (no spill); fp32 stays at 2
    for (; i + (U - 1) * stride < n; i += U * stride) {
        Oct<T> rd[U], rx[U], ry[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            long long const e = (i + u * stride) * 8;
            rd[u] = load_oct(dy + e);
            rx[u] = load_oct(x + e);
            ry[u] = masked ? load_oct(y + e) : zero_oct<T>();
        }
#pragma unroll
        for (int u = 0; u < U; ++u)
            store_oct(dx + (i + u * stride) * 8, transform(rd[u], rx[u], ry[u]));
    }
    for (; i < n; i += stride) {
        Oct<T> const ry = masked ? load_oct(y + i * 8) : zero_oct<T>();
        store_oct(dx + i * 8, transform(load_oct(dy + i * 8), load_oct(x + i * 8), ry));
    }
}

// Strided pixel sub-sampling (the 1x1 stride-s "max-pool" of slim's identity shortcuts): y[n, oh, ow, :] = x[n, oh*s, ow*s, :].
// grid.y = n * OH + oh, threads along (ow, channel octet): no per-element division.
template<typename T>
__global__ void subsample_fwd_kernel(T const* __restrict__ x, T* __restrict__ y, int H, int W, int OH, int OW, int octets, int s) {
    pdl_trigger();
    pdl_wait();
    int const n = blockIdx.y / OH, oh = blockIdx.y % OH;
    Oct<T> const* src = reinterpret_cast<Oct<T> const*>(x) + (static_cast<long long>(n) * H + static_cast<long long>(oh) * s) * W * octets;
    Oct<T>* dst = reinterpret_cast<Oct<T>*>(y) + static_cast<long long>(blockIdx.y) * OW * octets;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < OW * octets; i += gridDim.x * blockDim.x) {
        int const ow = i / octets, o = i - ow * octets;
        dst[i] = src[static_cast<long long>(ow) * s * octets + o];
    }
}
// Its backward writes the whole dx in one pass: dy at the sampled pixels, zero elsewhere (replaces a fill + a strided copy).
template<typename T>
__global__ void subsample_bwd_kernel(T const* __restrict__ dy, T* __restrict__ dx, int H, int W, int OH, int OW, int octets, int s) {
    pdl_trigger();
    pdl_wait();
    int const n = blockIdx.y / H, h = blockIdx.y % H;
    bool const row_hit = h % s == 0 && h / s < OH;
    Oct<T> const* src = reinterpret_cast<Oct<T> const*>(dy) + (static_cast<long long>(n) * OH + h / s) * OW * octets;
    Oct<T>* dst = reinterpret_cast<Oct<T>*>(dx) + static_cast<long long>(blockIdx.y) * W * octets;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < W * octets; i += gridDim.x * blockDim.x) {
        int const w = i / octets, o = i - w * octets;
        bool const hit = row_hit && w % s == 0 && w / s < OW;
        dst[i] = hit ? src[static_cast<long long>(w / s) * octets + o] : zero_oct<T>();
    }
}

// The same gradient added in place to an existing dx: dx[n, oh*s, ow*s, :] += dy[n, oh, ow, :], the other pixels untouched. This is
// add(dx, subsample_backward(dy)) reading and writing only the sampled quarter of dx; the one difference is that the separate add
// turns a -0 of dx into +0 (-0 + +0) at the pixels this kernel skips. grid.y = n * OH + oh, threads along (ow, channel octet).
template<typename T>
__global__ void subsample_add_kernel(T const* __restrict__ dy, T* __restrict__ dx, int H, int W, int OH, int OW, int octets, int s) {
    pdl_trigger();
    pdl_wait();   // dx is the output of the previous kernel (see launch_pdl)
    int const n = blockIdx.y / OH, oh = blockIdx.y % OH;
    Oct<T> const* src = reinterpret_cast<Oct<T> const*>(dy) + static_cast<long long>(blockIdx.y) * OW * octets;
    T* dst = dx + (static_cast<long long>(n) * H + static_cast<long long>(oh) * s) * W * octets * 8;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < OW * octets; i += gridDim.x * blockDim.x) {
        int const ow = i / octets, o = i - ow * octets;
        T* p = dst + (static_cast<long long>(ow) * s * octets + o) * 8;
        float va[8], vb[8];
        unpack8(load_oct(p), va);
        unpack8(src[i], vb);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            va[j] += vb[j];
        store_oct(p, pack_oct<T>(va));
    }
}

// out = relu?(a + b) ; b may be null (plain ReLU)
template<typename T>
__global__ void add_relu_kernel(T const* __restrict__ a, T const* __restrict__ b, T* __restrict__ out, long long octets, int relu) {
    pdl_trigger();
    pdl_wait();
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (; i < octets; i += stride) {
        float va[8];
        unpack8(load_oct(a + i * 8), va);
        if (b) {
            float vb[8];
            unpack8(load_oct(b + i * 8), vb);
#pragma unroll
            for (int j = 0; j < 8; ++j)
                va[j] += vb[j];
        }
        if (relu) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                va[j] = max_nan(va[j], 0.f);
        }
        store_oct(out + i * 8, pack_oct<T>(va));
    }
}

// dx = dy * (y > 0)
template<typename T>
__global__ void relu_bwd_kernel(T const* __restrict__ dy, T const* __restrict__ y, T* __restrict__ dx, long long octets) {
    pdl_trigger();
    pdl_wait();
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (; i < octets; i += stride) {
        float vd[8], vy[8];
        unpack8(load_oct(dy + i * 8), vd);
        unpack8(load_oct(y + i * 8), vy);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            vd[j] = vy[j] > 0.f ? vd[j] : 0.f;
        store_oct(dx + i * 8, pack_oct<T>(vd));
    }
}

// ---------------------------------------------------------------------------- //
// Max pooling (k x k, stride s, explicit pads, -inf padding), NHWC. Forward also records the argmax (window-relative index): the
// first maximal tap in row-major window order, or the last NaN tap of a window holding NaN (NaN propagates, as in torch).
// K > 0: window size known at compile time — the K * K taps are loaded first (all in flight), then compared; K = 0: any window.
template<typename T, int K>
__global__ void maxpool_fwd_kernel(T const* __restrict__ x, T* __restrict__ y, unsigned char* __restrict__ arg, int N, int H, int W, int C, int OH, int OW,
                                   int k, int s, int pad_t, int pad_l) {
    pdl_trigger();
    pdl_wait();
    int const octets = C >> 3;
    long long const total = static_cast<long long>(N) * OH * OW * octets;
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (; i < total; i += stride) {
        int const o = static_cast<int>(i % octets);
        long long rest = i / octets;
        int const ow = static_cast<int>(rest % OW);
        rest /= OW;
        int const oh = static_cast<int>(rest % OH);
        int const n = static_cast<int>(rest / OH);
        float best[8];
        unsigned char where[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            best[j] = -INFINITY;
            where[j] = 0;
        }
        if (K > 0) {
            Oct<T> taps[K > 0 ? K * K : 1];
            bool valid[K > 0 ? K * K : 1];
#pragma unroll
            for (int t = 0; t < K * K; ++t) {
                int const h = oh * s - pad_t + t / K, w = ow * s - pad_l + t % K;
                valid[t] = h >= 0 && h < H && w >= 0 && w < W;
                taps[t] = zero_oct<T>();
                if (valid[t])
                    taps[t] = load_oct(x + ((static_cast<long long>(n) * H + h) * W + w) * C + o * 8);
            }
#pragma unroll
            for (int t = 0; t < K * K; ++t) {
                float v[8];
                unpack8(taps[t], v);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (valid[t] && (v[j] > best[j] || v[j] != v[j])) {   // a NaN wins its window
                        best[j] = v[j];
                        where[j] = static_cast<unsigned char>(t);
                    }
            }
        } else {
            for (int kh = 0; kh < k; ++kh) {
                int const h = oh * s - pad_t + kh;
                if (h < 0 || h >= H)
                    continue;
                for (int kw = 0; kw < k; ++kw) {
                    int const w = ow * s - pad_l + kw;
                    if (w < 0 || w >= W)
                        continue;
                    float v[8];
                    unpack8(load_oct(x + ((static_cast<long long>(n) * H + h) * W + w) * C + o * 8), v);
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        if (v[j] > best[j] || v[j] != v[j]) {
                            best[j] = v[j];
                            where[j] = static_cast<unsigned char>(kh * k + kw);
                        }
                }
            }
        }
        store_oct(y + i * 8, pack_oct<T>(best));
        uint2 packed;
        unsigned char* pw = reinterpret_cast<unsigned char*>(&packed);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            pw[j] = where[j];
        *reinterpret_cast<uint2*>(arg + i * 8) = packed;
    }
}

// Gather form: every input element sums the gradients of the windows whose argmax it is (no atomics).
// grid.y = n * H + h (one input row per CTA row), threads along (w, channel octet): no per-element division by H or W, and the
// candidate window rows are resolved once per CTA.
template<typename T>
__global__ void maxpool_bwd_kernel(T const* __restrict__ dy, unsigned char const* __restrict__ arg, T* __restrict__ dx, int N, int H, int W, int C, int OH, int OW,
                                   int k, int s, int pad_t, int pad_l) {
    pdl_trigger();
    pdl_wait();
    int const octets = C >> 3;
    int const n = blockIdx.y / H, h = blockIdx.y % H;
    T* const out_row = dx + static_cast<long long>(blockIdx.y) * W * C;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < W * octets; i += gridDim.x * blockDim.x) {
        int const w = i / octets, o = i - w * octets;
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
            acc[j] = 0.f;
        for (int kh = 0; kh < k; ++kh) {
            int const th = h + pad_t - kh;
            if (th < 0 || th % s)
                continue;
            int const oh = th / s;
            if (oh >= OH)
                continue;
            for (int kw = 0; kw < k; ++kw) {
                int const tw = w + pad_l - kw;
                if (tw < 0 || tw % s)
                    continue;
                int const ow = tw / s;
                if (ow >= OW)
                    continue;
                long long const oidx = (((static_cast<long long>(n) * OH + oh) * OW + ow) * octets + o) * 8;
                float v[8];
                unpack8(load_oct(dy + oidx), v);
                uint2 const packed = *reinterpret_cast<uint2 const*>(arg + oidx);
                unsigned char const* pw = reinterpret_cast<unsigned char const*>(&packed);
                unsigned char const me = static_cast<unsigned char>(kh * k + kw);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    acc[j] += pw[j] == me ? v[j] : 0.f;
            }
        }
        store_oct(out_row + static_cast<long long>(i) * 8, pack_oct<T>(acc));
    }
}

// Max-pool backward for window 3, stride 2 (the stem pools of ResNet / Inception): one thread per 2 x 2 block of input pixels and
// channel octet. With H' = h + pad_t, the rows H' in {2a, 2a+1} are only covered by the windows oh in {a-1, a} (kh = H' - 2 oh), same
// for the columns: FOUR (dy, argmax) pairs, loaded together, serve four outputs — the per-pixel gather above needs nine dependent
// candidates for the same four pixels.
template<typename T>
__global__ void __launch_bounds__(kThreads) maxpool3s2_bwd_kernel(T const* __restrict__ dy, unsigned char const* __restrict__ arg, T* __restrict__ dx, int H, int W, int C, int OH, int OW,
                                                                  int pad_t, int pad_l, int A, int B) {
    pdl_trigger();
    pdl_wait();
    int const octets = C >> 3;
    int const n = blockIdx.y / A, a = blockIdx.y % A;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * octets; i += gridDim.x * blockDim.x) {
        int const b = i / octets, o = i - b * octets;
        Oct<T> grad[4];
        uint2 who[4];
        bool valid[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {              // t = 2 * di + dj: window (a - di, b - dj)
            int const oh = a - (t >> 1), ow = b - (t & 1);
            valid[t] = oh >= 0 && oh < OH && ow >= 0 && ow < OW;
            grad[t] = zero_oct<T>();
            who[t] = make_uint2(0u, 0u);
            if (valid[t]) {
                long long const oidx = (((static_cast<long long>(n) * OH + oh) * OW + ow) * octets + o) * 8;
                grad[t] = load_oct(dy + oidx);
                who[t] = *reinterpret_cast<uint2 const*>(arg + oidx);
            }
        }
        float g[4][8];
#pragma unroll
        for (int t = 0; t < 4; ++t)
            unpack8(grad[t], g[t]);
#pragma unroll
        for (int p = 0; p < 4; ++p) {              // p = 2 * pi + pj: input pixel (2a + pi - pad_t, 2b + pj - pad_l)
            int const pi = p >> 1, pj = p & 1;
            int const h = 2 * a + pi - pad_t, w = 2 * b + pj - pad_l;
            if (h < 0 || h >= H || w < 0 || w >= W)
                continue;
            float acc[8];
#pragma unroll
            for (int j = 0; j < 8; ++j)
                acc[j] = 0.f;
#pragma unroll
            for (int t = 0; t < 4; ++t) {
                int const di = t >> 1, dj = t & 1;
                if ((pi == 1 && di == 1) || (pj == 1 && dj == 1))
                    continue;                      // kh / kw would be 3: outside the window
                unsigned char const me = static_cast<unsigned char>((pi + 2 * di) * 3 + (pj + 2 * dj));
                unsigned char const* pw = reinterpret_cast<unsigned char const*>(&who[t]);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    acc[j] += (valid[t] && pw[j] == me) ? g[t][j] : 0.f;
            }
            store_oct(dx + (((static_cast<long long>(n) * H + h) * W + w) * octets + o) * 8, pack_oct<T>(acc));
        }
    }
}

// Global average pool: x [N, HW, C] -> y [N, C]; backward broadcasts dy / HW.
template<typename T>
__global__ void avgpool_fwd_kernel(T const* __restrict__ x, T* __restrict__ y, int N, int HW, int C) {
    pdl_trigger();
    pdl_wait();
    int const octets = C >> 3;
    int const i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * octets)
        return;
    int const n = i / octets, o = i % octets;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j)
        acc[j] = 0.f;
    for (int p = 0; p < HW; ++p) {
        float v[8];
        unpack8(load_oct(x + (static_cast<long long>(n) * HW + p) * C + o * 8), v);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            acc[j] += v[j];
    }
    float const inv = 1.f / static_cast<float>(HW);
#pragma unroll
    for (int j = 0; j < 8; ++j)
        acc[j] *= inv;
    store_oct(y + static_cast<long long>(i) * 8, pack_oct<T>(acc));
}

template<typename T>
__global__ void avgpool_bwd_kernel(T const* __restrict__ dy, T* __restrict__ dx, int N, int HW, int C) {
    pdl_trigger();
    pdl_wait();
    int const octets = C >> 3;
    long long const total = static_cast<long long>(N) * HW * octets;
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const stride = static_cast<long long>(gridDim.x) * blockDim.x;
    float const inv = 1.f / static_cast<float>(HW);
    for (; i < total; i += stride) {
        int const o = static_cast<int>(i % octets);
        int const n = static_cast<int>(i / (static_cast<long long>(HW) * octets));
        float v[8];
        unpack8(load_oct(dy + (static_cast<long long>(n) * octets + o) * 8), v);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            v[j] *= inv;
        store_oct(dx + i * 8, pack_oct<T>(v));
    }
}

// ---------------------------------------------------------------------------- //
// Softmax cross-entropy, one warp per row. logits bf16 [B, ld] (K valid columns), labels int64.
// loss += mean_b(-sum_k t_k log p_k) ; dlogits = (p - t) / B  (bf16, same leading dimension).
// Data poisoning of the groups >= poison_from (poison_from == groups poisons nothing):
//   label flipping (Fang et al., USENIX Security 2020; target < 0, q = rows_per_group, scale = 1): every row trains on K - 1 - y
//     instead of y; a label outside [0, K) matches no class and is left as it is;
//   backdoor (Gu et al., BadNets; Bagdasaryan et al., AISTATS 2020; 0 <= target < K): the rows with row % rows_per_group < q train on
//     `target`, and every row's dlogits is multiplied by `scale` (the loss is not). scale = 1 gives the unscaled bits exactly.
template<typename T>
__global__ void softmax_xent_kernel(T const* __restrict__ logits, long long const* __restrict__ labels, T* __restrict__ dlogits, float* __restrict__ loss,
                                    int B, int K, long long ld, float smoothing, int rows_per_group, int poison_from, int q, int target, float scale) {
    pdl_trigger();
    pdl_wait();
    int const warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B)
        return;
    int const group = warp / rows_per_group;
    T const* row = logits + static_cast<long long>(warp) * ld;
    float mx = -INFINITY;
    for (int k = lane; k < K; k += 32)
        mx = fmaxf(mx, to_f(row[k]));
    for (int off = 16; off > 0; off >>= 1)
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    float sum = 0.f;
    for (int k = lane; k < K; k += 32)
        sum += __expf(to_f(row[k]) - mx);
    sum = warp_sum(sum);
    float const lse = mx + __logf(sum);
    long long const y = labels[warp];
    bool const poisoned = group >= poison_from;
    int label = static_cast<int>(y);
    if (poisoned && warp % rows_per_group < q)
        label = target >= 0 ? target : y >= 0 && y < K ? K - 1 - label : label;
    float const gscale = poisoned ? scale : 1.f;
    float const off_t = smoothing / static_cast<float>(K), on_t = 1.f - smoothing + off_t;
    float const inv_b = 1.f / static_cast<float>(rows_per_group);   // each group (logical worker) averages over its own batch
    float local = 0.f;
    T* drow = dlogits + static_cast<long long>(warp) * ld;
    for (int k = lane; k < K; k += 32) {
        float const z = to_f(row[k]);
        float const logp = z - lse;
        float const t = k == label ? on_t : off_t;
        local -= t * logp;
        drow[k] = from_f<T>(((__expf(logp) - t) * inv_b) * gscale);
    }
    local = warp_sum(local);
    if (lane == 0)
        atomicAdd(loss + group, local * inv_b);
}

// uint8 NHWC image [.., H, W, C] -> bf16 NHWC activations with C padded to `Cpad`: y = (x - mean[c]) * scale, with the backdoor
// trigger (agb_device.cuh) in place of x on the poisoned images.
template<typename T>
__global__ void image_normalize_kernel(unsigned char const* __restrict__ x, T* __restrict__ y, long long pixels, int C, int Cpad, float m0, float m1, float m2, float scale,
                                       int H, int W, Trigger trigger) {
    pdl_trigger();
    pdl_wait();
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (; i < pixels; i += stride) {
        float stamp = -1.f;
        if (trigger.s > 0) {
            long long const hw = static_cast<long long>(H) * W, image = i / hw;
            int const pixel = static_cast<int>(i - image * hw);
            if (trigger_poisoned(trigger, image))
                stamp = trigger_value(trigger, H, W, pixel / W, pixel % W);
        }
        for (int c = 0; c < Cpad; ++c) {
            float v = 0.f;
            if (c < C) {
                float const m = c == 0 ? m0 : c == 1 ? m1 : m2;
                v = ((stamp >= 0.f ? stamp : static_cast<float>(x[i * C + c])) - m) * scale;
            }
            y[i * Cpad + c] = from_f<T>(v);
        }
    }
}

// ---------------------------------------------------------------------------- //
// im2col: x NHWC [N,H,W,C] -> col [N*OH*OW, ldcol] with column order (kh, kw, c); zero padding, zero tail columns.
// One thread per (output pixel, kh, kw, channel octet) when C % 8 == 0, scalar path otherwise (the 3-channel stem).
template<typename T>
__global__ void im2col_kernel(T const* __restrict__ x, T* __restrict__ col, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int s, int pad_t, int pad_l, long long ldcol) {
    pdl_trigger();
    pdl_wait();
    if ((C & 7) == 0) {
        int const octets = C >> 3;
        long long const total = static_cast<long long>(N) * OH * OW * KH * KW * octets;
        long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
        long long const stride = static_cast<long long>(gridDim.x) * blockDim.x;
        for (; i < total; i += stride) {
            int const o = static_cast<int>(i % octets);
            long long rest = i / octets;
            int const kw = static_cast<int>(rest % KW);
            rest /= KW;
            int const kh = static_cast<int>(rest % KH);
            rest /= KH;
            long long const pixel = rest;
            int const ow = static_cast<int>(rest % OW);
            rest /= OW;
            int const oh = static_cast<int>(rest % OH);
            int const n = static_cast<int>(rest / OH);
            int const h = oh * s - pad_t + kh, w = ow * s - pad_l + kw;
            Oct<T> v = zero_oct<T>();
            if (h >= 0 && h < H && w >= 0 && w < W)
                v = load_oct(x + ((static_cast<long long>(n) * H + h) * W + w) * C + o * 8);
            store_oct(col + pixel * ldcol + (kh * KW + kw) * C + o * 8, v);
        }
    } else {
        // Few-channel stem (C = 1 or 3): one thread per (output pixel, group of 8 columns) gathers 8 scalars (L1 hits) and
        // writes one 16-byte vector; (c, kw, kh) advance incrementally, no division in the inner loop.
        int const groups8 = static_cast<int>(ldcol >> 3);
        long long const total = static_cast<long long>(N) * OH * OW * groups8;
        long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
        long long const stride = static_cast<long long>(gridDim.x) * blockDim.x;
        int const kcol = KH * KW * C;
        for (; i < total; i += stride) {
            int const g8 = static_cast<int>(i % groups8);
            long long rest = i / groups8;
            int const ow = static_cast<int>(rest % OW);
            rest /= OW;
            int const oh = static_cast<int>(rest % OH);
            int const n = static_cast<int>(rest / OH);
            int j = g8 * 8;
            int c = j % C, kw = (j / C) % KW, kh = j / (C * KW);
            float v[8];
#pragma unroll
            for (int jj = 0; jj < 8; ++jj, ++j) {
                v[jj] = 0.f;
                if (j < kcol) {
                    int const h = oh * s - pad_t + kh, w = ow * s - pad_l + kw;
                    if (h >= 0 && h < H && w >= 0 && w < W)
                        v[jj] = to_f(x[((static_cast<long long>(n) * H + h) * W + w) * C + c]);
                }
                if (++c == C) {
                    c = 0;
                    if (++kw == KW) {
                        kw = 0;
                        ++kh;
                    }
                }
            }
            store_oct(col + (i / groups8) * ldcol + g8 * 8, pack_oct<T>(v));
        }
    }
}

// im2col of a few-channel stem (C = 1 or 3, e.g. ResNet's 7x7/2 on RGB): one CTA per output row (n, oh). The KH input rows the row
// needs are staged in shared memory with coalesced loads (a (kh, .) segment of a col row is KW * C CONTIGUOUS input elements), then
// every thread assembles 16-byte vectors of the col rows from shared memory: the global side only sees full-width reads and writes
// (the scalar gather of `im2col_kernel` ran the 122 MB stem matrix of a batch-32 ResNet-50 at 0.86 TB/s).
template<typename T>
__global__ void __launch_bounds__(kThreads) im2col_stem_kernel(T const* __restrict__ x, T* __restrict__ col, int H, int W, int C, int OH, int OW, int KH, int KW, int s, int pad_t, int pad_l, long long ldcol) {
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char stem_smem[];
    T* rows = reinterpret_cast<T*>(stem_smem);          // [KH][W * C]
    int const n = blockIdx.x / OH, oh = blockIdx.x % OH;
    int const row_len = W * C;
    for (int kh = 0; kh < KH; ++kh) {
        int const h = oh * s - pad_t + kh;
        T* dst = rows + kh * row_len;
        if (h < 0 || h >= H) {
            for (int i = threadIdx.x; i < row_len; i += kThreads)
                dst[i] = from_f<T>(0.f);
            continue;
        }
        T const* src = x + (static_cast<long long>(n) * H + h) * row_len;
        if ((row_len * sizeof(T)) % 16 == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
            int const vecs = static_cast<int>(row_len * sizeof(T) / 16);
            for (int i = threadIdx.x; i < vecs; i += kThreads)
                reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<uint4 const*>(src)[i];
        } else {
            for (int i = threadIdx.x; i < row_len; i += kThreads)
                dst[i] = src[i];
        }
    }
    __syncthreads();
    int const groups8 = static_cast<int>(ldcol >> 3), seg = KW * C, kcol = KH * seg;
    T* out = col + static_cast<long long>(blockIdx.x) * OW * ldcol;
    for (int i = threadIdx.x; i < OW * groups8; i += kThreads) {
        int const ow = i / groups8, g8 = i - ow * groups8;
        int const base = (ow * s - pad_l) * C;          // input element of (kw = 0, c = 0); may be negative (left padding)
        int j = g8 * 8;
        int kh = j / seg, r = j - kh * seg;
        float v[8];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj, ++j) {
            int const idx = base + r;
            v[jj] = (j < kcol && idx >= 0 && idx < row_len) ? to_f(rows[kh * row_len + idx]) : 0.f;
            if (++r == seg) {
                r = 0;
                ++kh;
            }
        }
        store_oct(out + static_cast<long long>(ow) * ldcol + g8 * 8, pack_oct<T>(v));
    }
}

// col2im (gather form): dx[n,h,w,c] = sum over (kh,kw) of dcol[n, oh, ow, (kh,kw,c)] for the windows covering (h,w). C % 8 == 0.
template<typename T>
__global__ void col2im_kernel(T const* __restrict__ dcol, T* __restrict__ dx, int N, int H, int W, int C, int OH, int OW, int KH, int KW, int s, int pad_t, int pad_l, long long ldcol) {
    pdl_trigger();
    pdl_wait();
    int const octets = C >> 3;
    long long const total = static_cast<long long>(N) * H * W * octets;
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (; i < total; i += stride) {
        int const o = static_cast<int>(i % octets);
        long long rest = i / octets;
        int const w = static_cast<int>(rest % W);
        rest /= W;
        int const h = static_cast<int>(rest % H);
        int const n = static_cast<int>(rest / H);
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j)
            acc[j] = 0.f;
        for (int kh = 0; kh < KH; ++kh) {
            int const th = h + pad_t - kh;
            if (th < 0 || th % s)
                continue;
            int const oh = th / s;
            if (oh >= OH)
                continue;
            for (int kw = 0; kw < KW; ++kw) {
                int const tw = w + pad_l - kw;
                if (tw < 0 || tw % s)
                    continue;
                int const ow = tw / s;
                if (ow >= OW)
                    continue;
                float v[8];
                unpack8(load_oct(dcol + ((static_cast<long long>(n) * OH + oh) * OW + ow) * ldcol + (kh * KW + kw) * C + o * 8), v);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    acc[j] += v[j];
            }
        }
        store_oct(dx + i * 8, pack_oct<T>(acc));
    }
}

inline int grid_for(long long work, int threads = kThreads, int cap = agb::sm_count() * 8) {
    long long blocks = (work + threads - 1) / threads;
    if (blocks > cap)
        blocks = cap;
    return blocks < 1 ? 1 : static_cast<int>(blocks);
}

// CTAs per group of the apply kernels: the grid `grid_for` gives one group's octets, within an equal share of the usual cap (so one
// group gets the same grid as before the split), and at least one CTA per 256 octets of a row so that every octet has a thread.
inline int apply_ctas(long long rows_per_group, int C, int groups) {
    int const octets = C >> 3;
    int const share = agb::sm_count() * 8 / groups;
    int const ctas = grid_for(rows_per_group * octets, kThreads, share < 1 ? 1 : share);
    int const least = (octets + kThreads - 1) / kThreads;
    return ctas > least ? ctas : least;
}

struct SumsPlan {
    int rows_per_cta, strip;
    dim3 grid;
};
inline SumsPlan plan_sums(long long rows_per_group, int C, int groups) {
    int const octets = C >> 3;
    SumsPlan plan;
    plan.strip = 8;   // 128-byte strips measured faster end to end than 256/512-byte ones (more CTAs per tensor)
    int const row_lanes = kThreads / plan.strip;
    int const strips = (octets + plan.strip - 1) / plan.strip;
    long long target = (agb::sm_count() * 6 + strips * groups - 1) / (strips * groups);   // ~6 CTAs per SM overall
    if (target < 1)
        target = 1;
    long long rows_per_cta = (rows_per_group + target - 1) / target;
    long long const min_rows = static_cast<long long>(row_lanes) * kRowUnroll;
    if (rows_per_cta < min_rows)
        rows_per_cta = min_rows;
    plan.rows_per_cta = static_cast<int>(rows_per_cta);
    plan.grid = dim3(static_cast<unsigned>((rows_per_group + rows_per_cta - 1) / rows_per_cta), strips, groups);
    return plan;
}

// ---------------------------------------------------------------------------- //
// Single-launch batch-norm (training) forward / backward.
//
// The two-kernel path above (statistics, then apply) pays two launches and reads the activation twice. At per-GPU batch
// sizes most BN tensors of a ResNet are 2..26 MB — smaller than the 132 x 228 KB of shared memory on the chip. This kernel
// runs one CTA per SM: phase 1 streams the CTA's row chunk once, *keeps it in shared memory* and accumulates the per-channel
// partial sums (fp32 per thread, fixed-order fold per CTA, one fp64 atomic per channel and CTA); a grid-wide barrier
// (atomic counter, every CTA is resident: grid <= #SMs, 1 CTA/SM by shared-memory footprint); phase 2 turns the sums into
// per-channel coefficients in registers and applies them to the resident tile, so the activation crosses the memory
// system once in and once out. Rows beyond the on-chip capacity are simply re-read in phase 2 (L2 hits at these sizes).
// Workspace: two halves used alternately (device-side toggle); a launch zeroes the half the next launch will use.

constexpr int kFusedThreads = 512;
constexpr int kFusedScratchBytes = kFusedThreads * 16 * 4;      // CTA reduction scratch: [lanes][octets * 16] floats
constexpr int kFusedMovingBytes = 12 * 1024;                    // the moving mean per channel, kept from phase 0 to phase 2
constexpr int kFusedStashBytes = 180 * 1024;                    // resident tile(s)
// fp64 accumulation of the CTAs' fp32 partial sums is exact (53-bit mantissa vs <= 132 addends of 24 bits), hence independent of
// the arrival order: statistics are bit-reproducible from run to run. To keep the atomics off a handful of hot L2 lines when C
// is small, the CTAs of a group spread over `replicas` copies of the sums, folded in a fixed order in phase 2.
using FusedSum = double;
constexpr long long kFusedHalfBytes = 16 + 2ll * 8 * 16384;     // barrier word + sums for up to 16384 (group, channel) pairs

struct BnFused {
    bf16 const* a;              // forward: x            backward: dy
    bf16 const* b;              // forward: residual added before the ReLU (or null)   backward: x
    bf16 const* mask;           //                       backward: y of a fused ReLU (or null)
    bf16* out;                  // forward: y            backward: dx
    bf16* out2;                 //                       backward: the masked dy (gradient of the residual input), or null
    float const* gamma;
    float const* beta;
    float* moving_mean;
    float* moving_var;
    float* save_mean;           // forward: out          backward: in
    float* save_rstd;
    float* scale;               // forward: out, the coefficients applied (y = x * scale + shift), or null
    float* shift;
    float* dgamma;
    float* dbeta;
    long long group_stride;
    unsigned* state;            // [0]: which half of `ws` this launch uses
    unsigned char* ws;
    long long rows_per_group, rows_per_cta;
    int C, groups, ctas_per_group, stash_vecs, relu, replicas;
    float eps, decay;
};

__device__ __forceinline__ unsigned ld_acquire_gpu(unsigned const* addr) {
    unsigned value;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(value) : "l"(addr) : "memory");
    return value;
}

template<bool BWD>
__global__ void __launch_bounds__(kFusedThreads, 1) bn_fused_kernel(BnFused const p) {
    // Programmatic dependent launch: nothing below may run before the producer of `p.a` / the previous user of the workspace has
    // finished. The successor may be launched early: it only becomes resident once EVERY CTA of this grid has passed this point,
    // so it cannot take the SM of a CTA the grid-wide barrier below is waiting for.
    pdl_trigger();
    pdl_wait();
    extern __shared__ __align__(16) unsigned char fused_smem[];
    float* red = reinterpret_cast<float*>(fused_smem);
    float* moving_s = reinterpret_cast<float*>(fused_smem + kFusedScratchBytes);
    uint4* stash_a = reinterpret_cast<uint4*>(fused_smem + kFusedScratchBytes + kFusedMovingBytes);
    uint4* stash_b = stash_a + p.stash_vecs;
    int const octets = p.C >> 3;
    // Per-channel vectors (pivot / saved statistics, later the coefficients) are fetched by ONE thread per channel and handed to
    // the others through shared memory: 16 warps x 132 CTAs all asking L2 for the same few cache lines costs tens of microseconds.
    __shared__ unsigned slot_shared;
    float* chan = red;          // [3][C] floats, aliasing the reduction scratch (used before / after it)
    int const group = blockIdx.x / p.ctas_per_group, chunk = blockIdx.x % p.ctas_per_group;
    if (threadIdx.x == 0)
        slot_shared = __ldcg(p.state) & 1u;
    for (int c0 = threadIdx.x; c0 < p.C; c0 += 4 * kFusedThreads) {   // up to 4 channels per thread, their loads in flight together
        float first[4], second[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            int const c = c0 + u * kFusedThreads;
            first[u] = second[u] = 0.f;
            if (c < p.C) {   // forward: the statistics pivot (the group's first row) and the moving mean
                first[u] = BWD ? p.save_mean[group * p.C + c] : __bfloat162float(p.a[static_cast<long long>(group) * p.rows_per_group * p.C + c]);
                second[u] = BWD ? p.save_rstd[group * p.C + c] : (p.moving_mean ? p.moving_mean[c] : 0.f);
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            int const c = c0 + u * kFusedThreads;
            if (c < p.C) {
                chan[c] = first[u];
                chan[p.C + c] = second[u];
                if (!BWD)
                    moving_s[c] = second[u];   // phase 2 must use the value read HERE: by then another CTA has updated the moving mean
            }
        }
    }
    __syncthreads();
    unsigned const slot = slot_shared;
    unsigned char* mine = p.ws + slot * kFusedHalfBytes;
    unsigned* bar = reinterpret_cast<unsigned*>(mine);
    FusedSum* sums = reinterpret_cast<FusedSum*>(mine + 16);
    {   // clear the other half for whoever launches next
        uint4* other = reinterpret_cast<uint4*>(p.ws + (slot ^ 1u) * kFusedHalfBytes);
        for (long long i = static_cast<long long>(blockIdx.x) * kFusedThreads + threadIdx.x; i < kFusedHalfBytes / 16; i += static_cast<long long>(gridDim.x) * kFusedThreads)
            other[i] = make_uint4(0, 0, 0, 0);
    }
    long long const row_begin = static_cast<long long>(chunk) * p.rows_per_cta;
    long long const row_end = min(p.rows_per_group, row_begin + p.rows_per_cta);
    long long const nvec = row_end > row_begin ? (row_end - row_begin) * octets : 0;
    long long const base = (static_cast<long long>(group) * p.rows_per_group + row_begin) * octets;
    uint4 const* ga = reinterpret_cast<uint4 const*>(p.a) + base;
    uint4 const* gb = p.b ? reinterpret_cast<uint4 const*>(p.b) + base : nullptr;
    uint4* gout2 = (BWD && p.out2) ? reinterpret_cast<uint4*>(p.out2) + base : nullptr;
    uint4 const* gm = (BWD && p.mask) ? reinterpret_cast<uint4 const*>(p.mask) + base : nullptr;
    uint4* gout = reinterpret_cast<uint4*>(p.out) + base;
    int const stride = kFusedThreads - kFusedThreads % octets;      // a thread keeps the same channel octet for all its vectors
    int const lanes = stride / octets;
    bool const active = static_cast<int>(threadIdx.x) < stride;
    int const o = threadIdx.x % octets, lane = threadIdx.x / octets;
    int const cbase = group * p.C + o * 8;
    // forward: `mu` is a per-channel pivot (the group's first row, a sample of the batch, so also right on the first step when the
    // moving mean is still zero): sums of (x - pivot) and (x - pivot)^2 keep E[x^2] - E[x]^2 well conditioned in fp32 even when
    // |mean| >> std; backward: the saved batch statistics.
    float s0[8], s1[8], mu[8], rs[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        s0[j] = 0.f;
        s1[j] = 0.f;
        mu[j] = active ? chan[o * 8 + j] : 0.f;
        rs[j] = active ? chan[p.C + o * 8 + j] : 0.f;
    }
    __syncthreads();            // `chan` aliases `red`: everybody has its copy before the scratch is reused
    // ---- phase 1: stream the chunk once, stash it, accumulate ------------------------------------------------------ //
    if (active) {
        constexpr int U = BWD ? 4 : 8;
        for (long long i0 = threadIdx.x; i0 < nvec; i0 += static_cast<long long>(stride) * U) {
            uint4 ra[U], rb[U], rm[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                long long const i = i0 + static_cast<long long>(u) * stride;
                if (i < nvec) {
                    ra[u] = ga[i];
                    if (BWD)
                        rb[u] = gb[i];
                    if (BWD && gm)
                        rm[u] = gm[i];
                    if (!BWD && gb && (i & 7) == 0)   // the residual is only needed after the barrier: have its lines in L2 by then
                        asm volatile("prefetch.global.L2 [%0];" :: "l"(gb + i));
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                long long const i = i0 + static_cast<long long>(u) * stride;
                if (i >= nvec)
                    continue;
                float va[8];
                unpack8(ra[u], va);
                if (!BWD) {
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        float const d = va[j] - mu[j];
                        s0[j] += d;
                        s1[j] += d * d;
                    }
                    if (i < p.stash_vecs)
                        stash_a[i] = ra[u];
                } else {
                    if (gm) {
                        float vy[8];
                        unpack8(rm[u], vy);
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            va[j] = vy[j] > 0.f ? va[j] : 0.f;
                        if (gout2)
                            gout2[i] = pack8(va);
                    }
                    float vx[8];
                    unpack8(rb[u], vx);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        s0[j] += va[j];
                        s1[j] += va[j] * (vx[j] - mu[j]) * rs[j];
                    }
                    if (i < p.stash_vecs) {
                        stash_a[i] = gm ? pack8(va) : ra[u];    // the masked gradient (exact: masking only zeroes lanes)
                        stash_b[i] = rb[u];
                    }
                }
            }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            red[lane * (octets * 16) + o * 16 + j] = s0[j];
            red[lane * (octets * 16) + o * 16 + 8 + j] = s1[j];
        }
    }
    __syncthreads();
    if (nvec > 0) {
        for (int t = threadIdx.x; t < octets * 16; t += kFusedThreads) {
            float total = 0.f;
            for (int l = 0; l < lanes; ++l)
                total += red[l * (octets * 16) + t];
            long long const slot_index = (static_cast<long long>(chunk % p.replicas) * p.groups + group) * p.C + (t >> 4) * 8 + (t & 7);
            atomicAdd(sums + slot_index * 2 + ((t >> 3) & 1), static_cast<FusedSum>(total));
        }
    }
    // ---- grid barrier ----------------------------------------------------------------------------------------------- //
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        atomicAdd(bar, 1u);
        unsigned spins = 0;
        while (ld_acquire_gpu(bar) < gridDim.x) {
            __nanosleep(200);
            if (++spins > (1u << 22)) {   // ~1 s: a CTA of this grid never arrived
                printf("[agb] bn_fused_kernel: grid barrier timeout (block %d, %u of %u arrived)\n", static_cast<int>(blockIdx.x), ld_acquire_gpu(bar), gridDim.x);
                __trap();
            }
        }
    }
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x == 0)
        *p.state = slot ^ 1u;
    // ---- phase 2: one thread per channel turns the sums into coefficients (shared memory), then apply to the resident tile -- //
    {
        double const n = static_cast<double>(p.rows_per_group), inv_n = 1.0 / n;
        for (int c = threadIdx.x; c < p.C; c += kFusedThreads) {
            long long const idx = static_cast<long long>(group) * p.C + c;
            // every replica's pair of sums in flight at once (one 16-byte load each): a loop of dependent L2 round trips here cost
            // ~5 us per launch (8 replicas), 20 us for the 2048-channel layers (4 channels per thread)
            double2 part[8];
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                part[r] = make_double2(0., 0.);
                if (r < p.replicas)
                    part[r] = __ldcg(reinterpret_cast<double2 const*>(sums + (static_cast<long long>(r) * p.groups * p.C + idx) * 2));
            }
            float const gmc = p.gamma ? p.gamma[c] : 1.f;
            float const aux0 = BWD ? p.save_rstd[idx] : p.beta[c], aux1 = BWD ? p.save_mean[idx] : 0.f;
            double t0 = 0., t1 = 0.;
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                t0 += part[r].x;
                t1 += part[r].y;
            }
            if (!BWD) {
                float const pivot = __bfloat162float(p.a[static_cast<long long>(group) * p.rows_per_group * p.C + c]);
                double const shifted = t0 * inv_n;
                double const mean = shifted + static_cast<double>(pivot);
                double var = fma(-shifted, shifted, t1 * inv_n);
                if (var < 0.)
                    var = 0.;
                float const rstd = rsqrtf(static_cast<float>(var) + p.eps);
                float const scale = gmc * rstd, shift = aux0 - static_cast<float>(mean) * gmc * rstd;
                chan[c] = scale;
                chan[p.C + c] = shift;
                if (chunk == 0) {
                    p.save_mean[idx] = static_cast<float>(mean);
                    p.save_rstd[idx] = rstd;
                    if (p.scale) {   // a backward pass may recompute the ReLU mask from x with them
                        p.scale[idx] = scale;
                        p.shift[idx] = shift;
                    }
                    if (p.moving_mean && group == 0) {   // unbiased variance in the moving average, as TF's fused batch norm
                        double const unbiased = n > 1. ? var * n / (n - 1.) : var;
                        p.moving_mean[c] = p.decay * moving_s[c] + (1.f - p.decay) * static_cast<float>(mean);
                        p.moving_var[c] = p.decay * p.moving_var[c] + (1.f - p.decay) * static_cast<float>(unbiased);
                    }
                }
            } else {
                float const inv = static_cast<float>(inv_n), rsc = aux0, muc = aux1;
                float const b1 = -gmc * rsc * rsc * static_cast<float>(t1) * inv;
                chan[c] = gmc * rsc;
                chan[p.C + c] = b1;
                chan[2 * p.C + c] = -gmc * rsc * static_cast<float>(t0) * inv - b1 * muc;
                if (chunk == 0) {
                    if (p.dgamma)
                        p.dgamma[group * p.group_stride + c] = static_cast<float>(t1);
                    p.dbeta[group * p.group_stride + c] = static_cast<float>(t0);
                }
            }
        }
    }
    __syncthreads();
    if (!active)
        return;
    float c0[8], c1[8], c2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        c0[j] = chan[o * 8 + j];
        c1[j] = chan[p.C + o * 8 + j];
        c2[j] = BWD ? chan[2 * p.C + o * 8 + j] : 0.f;
    }
    auto finish = [&](float (&va)[8], float const (&vx)[8]) {   // vx: forward = residual (zeros when absent), backward = x
        if (!BWD) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                va[j] = va[j] * c0[j] + c1[j] + vx[j];
                if (p.relu)
                    va[j] = max_nan(va[j], 0.f);
            }
        } else {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                va[j] = c0[j] * va[j] + c1[j] * vx[j] + c2[j];
        }
        return pack8(va);
    };
    long long const resident_end = nvec < p.stash_vecs ? nvec : static_cast<long long>(p.stash_vecs);
    long long i = threadIdx.x;
    if (!BWD && gb) {                                  // the tile kept on chip + the residual from memory, 4 loads in flight per thread
        constexpr int R = 4;                           // (one dependent load per iteration cost 5-13 us per launch)
        for (; i < resident_end; i += static_cast<long long>(stride) * R) {
            uint4 rb[R];
#pragma unroll
            for (int u = 0; u < R; ++u) {
                long long const k = i + static_cast<long long>(u) * stride;
                if (k < resident_end)
                    rb[u] = gb[k];
            }
#pragma unroll
            for (int u = 0; u < R; ++u) {
                long long const k = i + static_cast<long long>(u) * stride;
                if (k >= resident_end)
                    continue;
                float va[8], vx[8];
                unpack8(stash_a[k], va);
                unpack8(rb[u], vx);
                gout[k] = finish(va, vx);
            }
        }
        i = static_cast<long long>(threadIdx.x) >= resident_end ? threadIdx.x : threadIdx.x + ((resident_end - 1 - threadIdx.x) / stride + 1) * stride;
    } else {
        for (; i < resident_end; i += stride) {        // the tile kept on chip
            float va[8], vx[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            unpack8(stash_a[i], va);
            if (BWD)
                unpack8(stash_b[i], vx);
            gout[i] = finish(va, vx);
        }
    }
    constexpr int V = BWD ? 2 : 4;                     // the rest is streamed again (L2 / HBM), several loads in flight per thread
    for (; i < nvec; i += static_cast<long long>(stride) * V) {
        uint4 ra[V], rb[V], rm[V];
#pragma unroll
        for (int u = 0; u < V; ++u) {
            long long const k = i + static_cast<long long>(u) * stride;
            if (k < nvec) {
                ra[u] = ga[k];
                if (gb)
                    rb[u] = gb[k];
                if (BWD && gm)
                    rm[u] = gm[k];
            }
        }
#pragma unroll
        for (int u = 0; u < V; ++u) {
            long long const k = i + static_cast<long long>(u) * stride;
            if (k >= nvec)
                continue;
            float va[8], vx[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            unpack8(ra[u], va);
            if (gb)
                unpack8(rb[u], vx);
            if (BWD && gm) {
                float vy[8];
                unpack8(rm[u], vy);
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    va[j] = vy[j] > 0.f ? va[j] : 0.f;
            }
            gout[k] = finish(va, vx);
        }
    }
}

long long g_fused_max_mb[2] = {72, 40};   // forward, backward
long long g_fused_min_rows = 4096;

// Returns 0 when the fused kernel was launched, 399 when the shape is outside its envelope (the caller uses the two-kernel path).
template<bool BWD>
int launch_bn_fused(BnFused p, long long rows, cudaStream_t s) {
    int const octets = p.C >> 3;
    if ((p.C & 7) || 3 * p.C * 4 > kFusedScratchBytes || p.C * 4 > kFusedMovingBytes || p.groups < 1 || p.groups > agb::sm_count() || rows % p.groups || static_cast<long long>(p.C) * p.groups > 16384)
        return 399;
    static bool configured = false;
    int const smem = kFusedScratchBytes + kFusedMovingBytes + kFusedStashBytes;
    if (!configured) {
        AGB_CUDA_OK(cudaFuncSetAttribute(bn_fused_kernel<BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        configured = true;
    }
    // envelope: the resident-tile kernel wins from a few thousand rows up to tensors a few
    // times the on-chip capacity; tiny tensors and very large ones are served better by the many-CTA kernel pair
    bool const extra = BWD ? p.out2 != nullptr : p.b != nullptr;   // closing add + ReLU fused in: worth one more separate kernel
    long long const bytes = rows * p.C * 2;
    if (rows < (extra ? g_fused_min_rows / 4 : g_fused_min_rows) || bytes > g_fused_max_mb[BWD ? 1 : 0] << 20)
        return 399;
    p.rows_per_group = rows / p.groups;
    long long const vecs = p.rows_per_group * octets;
    long long const min_vecs = octets * 32ll > 2048 ? octets * 32ll : 2048;    // at least 32 rows / 32 KB per CTA
    long long want = (vecs + min_vecs - 1) / min_vecs;
    int const cap = agb::sm_count() / p.groups;   // the grid barrier needs every CTA resident: one per SM
    p.ctas_per_group = static_cast<int>(want < 1 ? 1 : (want > cap ? cap : want));
    p.rows_per_cta = (p.rows_per_group + p.ctas_per_group - 1) / p.ctas_per_group;
    p.stash_vecs = kFusedStashBytes / 16 / (BWD ? 2 : 1);
    long long const room = 16384 / (static_cast<long long>(p.C) * p.groups);
    p.replicas = static_cast<int>(room < 1 ? 1 : (room > 8 ? 8 : room));
    if (p.replicas > p.ctas_per_group)
        p.replicas = p.ctas_per_group;
    AGB_CUDA_OK(launch_pdl(bn_fused_kernel<BWD>, dim3(p.groups * p.ctas_per_group), dim3(kFusedThreads), static_cast<size_t>(smem), s, p));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<int MODE, typename T>
int launch_sums(SumsPlan const& plan, cudaStream_t s, T const* a, T const* b, T const* y, T* dmasked, float const* mean, float const* rstd, float const* msc, float const* msh,
                 double* out, long long rows_per_group, int C, SumsFinalize const& fin) {
    if (plan.strip == 32)
        AGB_CUDA_OK(launch_pdl(channel_sums_kernel<T, MODE, 32>, dim3(plan.grid), dim3(kThreads), 0, s, a, b, y, dmasked, mean, rstd, msc, msh, out, rows_per_group, C, plan.rows_per_cta, fin));
    else if (plan.strip == 16)
        AGB_CUDA_OK(launch_pdl(channel_sums_kernel<T, MODE, 16>, dim3(plan.grid), dim3(kThreads), 0, s, a, b, y, dmasked, mean, rstd, msc, msh, out, rows_per_group, C, plan.rows_per_cta, fin));
    else
        AGB_CUDA_OK(launch_pdl(channel_sums_kernel<T, MODE, 8>, dim3(plan.grid), dim3(kThreads), 0, s, a, b, y, dmasked, mean, rstd, msc, msh, out, rows_per_group, C, plan.rows_per_cta, fin));
    return 0;
}

template<typename T>
int bn_forward_impl(void const* x, void const* residual, void* y, void const* gamma, void const* beta, void* moving_mean, void* moving_var, void* save_mean, void* save_rstd,
                   void* sums, void* scale, void* shift, long long rows, int C, int groups, float eps, float decay, int relu, void* stream) {
    if ((C & 7) || groups < 1 || rows % groups)
        return 301;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    long long const rpg = rows / groups;
    // workspace: [groups*C*2] doubles, then one zeroed ticket word (zeroed together with the sums)
    SumsFinalize fin{};
    fin.ticket = reinterpret_cast<unsigned*>(static_cast<double*>(sums) + 2 * C * groups);
    fin.gamma = static_cast<float const*>(gamma); fin.beta = static_cast<float const*>(beta);
    fin.save_mean = static_cast<float*>(save_mean); fin.save_rstd = static_cast<float*>(save_rstd);
    fin.scale = static_cast<float*>(scale); fin.shift = static_cast<float*>(shift);
    fin.moving_mean = static_cast<float*>(moving_mean); fin.moving_var = static_cast<float*>(moving_var);
    fin.groups = groups; fin.eps = eps; fin.decay = decay;
    SumsPlan plan = plan_sums(rpg, C, groups);
    if (int status = launch_sums<0, T>(plan, s, static_cast<T const*>(x), nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, static_cast<double*>(sums), rpg, C, fin))
        return status;
    int const ctas = apply_ctas(rpg, C, groups);
    AGB_CUDA_OK(launch_pdl(bn_apply_kernel<T>, dim3(groups * ctas), dim3(kThreads), 0, s, static_cast<T const*>(x), static_cast<T const*>(residual), static_cast<T*>(y),
        static_cast<float const*>(scale), static_cast<float const*>(shift), rpg, C, ctas, relu));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int bn_backward_impl(void const* dy, void const* x, void const* y, void const* mask_scale, void const* mask_shift, void const* gamma, void const* save_mean, void const* save_rstd,
                    void* dx, void* dmasked, void* dgamma, void* dbeta, void* sums, void* coef, long long rows, int C, int groups, long long group_stride, void* stream) {
    if ((C & 7) || groups < 1 || rows % groups)
        return 301;
    if ((mask_scale == nullptr) != (mask_shift == nullptr) || (mask_scale && (y || dmasked)))
        return 302;
    float const* msc = static_cast<float const*>(mask_scale);
    float const* msh = static_cast<float const*>(mask_shift);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    long long const rpg = rows / groups;
    SumsFinalize fin{};
    fin.ticket = reinterpret_cast<unsigned*>(static_cast<double*>(sums) + 2 * C * groups);
    fin.gamma = static_cast<float const*>(gamma);
    fin.save_mean = const_cast<float*>(static_cast<float const*>(save_mean)); fin.save_rstd = const_cast<float*>(static_cast<float const*>(save_rstd));
    fin.scale = static_cast<float*>(coef);
    fin.dgamma = static_cast<float*>(dgamma); fin.dbeta = static_cast<float*>(dbeta);
    fin.groups = groups; fin.group_stride = group_stride;
    SumsPlan plan = plan_sums(rpg, C, groups);
    // with y and `dmasked`, the statistics kernel stores the masked gradient and the apply kernel reads it in place of dy and y
    T* const masked_out = y ? static_cast<T*>(dmasked) : nullptr;
    if (int status = launch_sums<1, T>(plan, s, static_cast<T const*>(dy), static_cast<T const*>(x), static_cast<T const*>(y), masked_out,
                   static_cast<float const*>(save_mean), static_cast<float const*>(save_rstd), msc, msh, static_cast<double*>(sums), rpg, C, fin))
        return status;
    int const ctas = apply_ctas(rpg, C, groups);
    T const* const grad = masked_out ? masked_out : static_cast<T const*>(dy);
    T const* const mask = masked_out ? nullptr : static_cast<T const*>(y);
    AGB_CUDA_OK(launch_pdl(bn_bwd_apply_kernel<T>, dim3(groups * ctas), dim3(kThreads), 0, s, grad, static_cast<T const*>(x), mask, static_cast<T*>(dx),
        static_cast<float const*>(coef), msc, msh, rpg, C, ctas));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int colsum_impl(void const* dy, void const* y, void* out, void* sums, long long rows, int C, int groups, long long group_stride, void* stream) {
    if ((C & 7) || groups < 1 || rows % groups)
        return 301;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    SumsFinalize fin{};
    fin.ticket = reinterpret_cast<unsigned*>(static_cast<double*>(sums) + 2 * C * groups);
    fin.dbeta = static_cast<float*>(out);
    fin.groups = groups; fin.group_stride = group_stride;
    SumsPlan plan = plan_sums(rows / groups, C, groups);
    if (int status = launch_sums<2, T>(plan, s, static_cast<T const*>(dy), nullptr, static_cast<T const*>(y), nullptr, nullptr, nullptr, nullptr, nullptr, static_cast<double*>(sums), rows / groups, C, fin))
        return status;
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int add_relu_impl(void const* a, void const* b, void* out, long long n, int relu, void* stream) {
    if (n & 7)
        return 301;
    AGB_CUDA_OK(launch_pdl(add_relu_kernel<T>, dim3(grid_for(n / 8)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(a), static_cast<T const*>(b), static_cast<T*>(out), n / 8, relu));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int subsample_forward_impl(void const* x, void* y, int N, int H, int W, int C, int s, void* stream) {
    if ((C & 7) || s < 1)
        return 301;
    int const OH = (H + s - 1) / s, OW = (W + s - 1) / s, octets = C >> 3;
    if (static_cast<long long>(N) * OH > 65535)
        return 399;
    int const per_row = OW * octets;
    AGB_CUDA_OK(launch_pdl(subsample_fwd_kernel<T>, dim3((per_row + kThreads - 1) / kThreads, N * OH), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(x), static_cast<T*>(y), H, W, OH, OW, octets, s));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int subsample_backward_impl(void const* dy, void* dx, int N, int H, int W, int C, int s, void* stream) {
    if ((C & 7) || s < 1)
        return 301;
    int const OH = (H + s - 1) / s, OW = (W + s - 1) / s, octets = C >> 3;
    if (static_cast<long long>(N) * H > 65535)
        return 399;
    int const per_row = W * octets;
    AGB_CUDA_OK(launch_pdl(subsample_bwd_kernel<T>, dim3((per_row + kThreads - 1) / kThreads, N * H), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(dy), static_cast<T*>(dx), H, W, OH, OW, octets, s));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int subsample_add_impl(void const* dy, void* dx, int N, int H, int W, int C, int s, void* stream) {
    if ((C & 7) || s < 1)
        return 301;
    int const OH = (H + s - 1) / s, OW = (W + s - 1) / s, octets = C >> 3;
    if (static_cast<long long>(N) * OH > 65535)
        return 399;
    int const per_row = OW * octets;
    AGB_CUDA_OK(launch_pdl(subsample_add_kernel<T>, dim3((per_row + kThreads - 1) / kThreads, N * OH), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(dy), static_cast<T*>(dx), H, W, OH, OW, octets, s));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int relu_backward_impl(void const* dy, void const* y, void* dx, long long n, void* stream) {
    if (n & 7)
        return 301;
    AGB_CUDA_OK(launch_pdl(relu_bwd_kernel<T>, dim3(grid_for(n / 8)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(dy), static_cast<T const*>(y), static_cast<T*>(dx), n / 8));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int maxpool_forward_impl(void const* x, void* y, void* arg, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    if ((C & 7) || k * k > 255)
        return 301;
    long long const work = static_cast<long long>(N) * OH * OW * (C >> 3);
    auto kernel = k == 3 ? maxpool_fwd_kernel<T, 3> : (k == 2 ? maxpool_fwd_kernel<T, 2> : maxpool_fwd_kernel<T, 0>);
    AGB_CUDA_OK(launch_pdl(kernel, dim3(grid_for(work)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(x), static_cast<T*>(y), static_cast<unsigned char*>(arg), N, H, W, C, OH, OW, k, s, pad_t, pad_l));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int maxpool_backward_impl(void const* dy, void const* arg, void* dx, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    if (C & 7)
        return 301;
    if (H > 65535)
        return 301;
    if (k == 3 && s == 2 && pad_t >= 0 && pad_t <= 2 && pad_l >= 0 && pad_l <= 2) {
        int const A = (H - 1 + pad_t) / 2 + 1, B = (W - 1 + pad_l) / 2 + 1;      // 2 x 2 blocks of (h + pad_t, w + pad_l)
        int const per = 65535 / A;
        for (int n0 = 0; n0 < N; n0 += per) {
            int const count = N - n0 < per ? N - n0 : per;
            AGB_CUDA_OK(launch_pdl(maxpool3s2_bwd_kernel<T>, dim3((B * (C >> 3) + kThreads - 1) / kThreads, count * A), dim3(kThreads), 0, static_cast<cudaStream_t>(stream),
                static_cast<T const*>(dy) + static_cast<long long>(n0) * OH * OW * C, static_cast<unsigned char const*>(arg) + static_cast<long long>(n0) * OH * OW * C,
                static_cast<T*>(dx) + static_cast<long long>(n0) * H * W * C, H, W, C, OH, OW, pad_t, pad_l, A, B));
        }
        AGB_CUDA_OK(cudaGetLastError());
        return 0;
    }
    // grid.y = images x rows is limited to 65535: very large batches go in slices of whole images
    int const per_launch = 65535 / H;
    for (int n0 = 0; n0 < N; n0 += per_launch) {
        int const count = N - n0 < per_launch ? N - n0 : per_launch;
        // (a variant with every candidate window's loads issued up front — window 3, stride 2 at compile time — measured slower:
        // 103 vs 85 us for the ResNet stem pool at batch 32, 772 vs 617 us at batch 256; the loop skips 5 of the 9 candidates early)
        auto kernel = maxpool_bwd_kernel<T>;
        AGB_CUDA_OK(launch_pdl(kernel, dim3((W * (C >> 3) + kThreads - 1) / kThreads, count * H), dim3(kThreads), 0, static_cast<cudaStream_t>(stream),
            static_cast<T const*>(dy) + static_cast<long long>(n0) * OH * OW * C, static_cast<unsigned char const*>(arg) + static_cast<long long>(n0) * OH * OW * C,
            static_cast<T*>(dx) + static_cast<long long>(n0) * H * W * C, count, H, W, C, OH, OW, k, s, pad_t, pad_l));
    }
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int avgpool_forward_impl(void const* x, void* y, int N, int HW, int C, void* stream) {
    if (C & 7)
        return 301;
    AGB_CUDA_OK(launch_pdl(avgpool_fwd_kernel<T>, dim3((N * (C >> 3) + 127) / 128), dim3(128), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(x), static_cast<T*>(y), N, HW, C));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int avgpool_backward_impl(void const* dy, void* dx, int N, int HW, int C, void* stream) {
    if (C & 7)
        return 301;
    long long const work = static_cast<long long>(N) * HW * (C >> 3);
    AGB_CUDA_OK(launch_pdl(avgpool_bwd_kernel<T>, dim3(grid_for(work)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(dy), static_cast<T*>(dx), N, HW, C));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int softmax_xent_impl(void const* logits, void const* labels, void* dlogits, void* loss, int B, int K, long long ld, float smoothing, int groups,
                      int poison_from, int q, int target, float scale, void* stream) {
    if (groups < 1 || B % groups || poison_from < 0 || poison_from > groups)
        return 301;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    AGB_CUDA_OK(cudaMemsetAsync(loss, 0, sizeof(float) * groups, s));
    int const warps_per_cta = 4;
    AGB_CUDA_OK(launch_pdl(softmax_xent_kernel<T>, dim3((B + warps_per_cta - 1) / warps_per_cta), dim3(warps_per_cta * 32), 0, s, static_cast<T const*>(logits), static_cast<long long const*>(labels),
        static_cast<T*>(dlogits), static_cast<float*>(loss), B, K, ld, smoothing, B / groups, poison_from, q, target, scale));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int image_normalize_impl(void const* x, void* y, long long pixels, int C, int Cpad, float m0, float m1, float m2, float scale, int H, int W, Trigger trigger, void* stream) {
    AGB_CUDA_OK(launch_pdl(image_normalize_kernel<T>, dim3(grid_for(pixels)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<unsigned char const*>(x), static_cast<T*>(y), pixels, C, Cpad, m0, m1, m2, scale,
        H, W, trigger));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int im2col_impl(void const* x, void* col, int N, int H, int W, int C, int OH, int OW, int kh, int kw, int s, int pad_t, int pad_l, long long ldcol, void* stream) {
    if (ldcol & 7)
        return 301;
    size_t const stem_smem = static_cast<size_t>(kh) * W * C * sizeof(T);
    if ((C & 7) != 0 && stem_smem <= 40 * 1024 && static_cast<long long>(N) * OH < (1ll << 31)) {
        AGB_CUDA_OK(launch_pdl(im2col_stem_kernel<T>, dim3(static_cast<unsigned>(N * OH)), dim3(kThreads), stem_smem, static_cast<cudaStream_t>(stream), static_cast<T const*>(x), static_cast<T*>(col), H, W, C, OH, OW, kh, kw, s, pad_t, pad_l, ldcol));
        AGB_CUDA_OK(cudaGetLastError());
        return 0;
    }
    long long const work = (C & 7) == 0 ? static_cast<long long>(N) * OH * OW * kh * kw * (C >> 3) : static_cast<long long>(N) * OH * OW * (ldcol >> 3);
    AGB_CUDA_OK(launch_pdl(im2col_kernel<T>, dim3(grid_for(work, kThreads, agb::sm_count() * 16)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(x), static_cast<T*>(col), N, H, W, C, OH, OW, kh, kw, s, pad_t, pad_l, ldcol));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

template<typename T>
int col2im_impl(void const* dcol, void* dx, int N, int H, int W, int C, int OH, int OW, int kh, int kw, int s, int pad_t, int pad_l, long long ldcol, void* stream) {
    if ((C & 7) || (ldcol & 7))
        return 301;
    long long const work = static_cast<long long>(N) * H * W * (C >> 3);
    AGB_CUDA_OK(launch_pdl(col2im_kernel<T>, dim3(grid_for(work, kThreads, agb::sm_count() * 16)), dim3(kThreads), 0, static_cast<cudaStream_t>(stream), static_cast<T const*>(dcol), static_cast<T*>(dx), N, H, W, C, OH, OW, kh, kw, s, pad_t, pad_l, ldcol));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

} // namespace

extern "C" {

// Workspace layout for BN (caller provides, zeroed `sums` not required: it is cleared here):
//   sums  double [groups*C*2] | save_mean, save_rstd, scale, shift float [groups*C] each (forward)
//   sums  double [groups*C*2] | coef float [groups*C*3]                              (backward)
// Backward: the ReLU mask is y > 0 when `y` is given, or is recomputed from x with the forward's `scale` / `shift` ([groups*C]
// each, what agb_bn_forward(_fused) stored) when `mask_scale` / `mask_shift` are given instead: one activation fewer to read in
// each of the two passes, same result bit for bit. Neither: no ReLU. `dmasked` needs `y`: the statistics kernel stores dy * (y > 0)
// there and the apply kernel reads it in place of dy and y.
int agb_bn_forward(void const* x, void const* residual, void* y, void const* gamma, void const* beta, void* moving_mean, void* moving_var, void* save_mean, void* save_rstd,
                   void* sums, void* scale, void* shift, long long rows, int C, int groups, float eps, float decay, int relu, void* stream) {
    return bn_forward_impl<bf16>(x, residual, y, gamma, beta, moving_mean, moving_var, save_mean, save_rstd, sums, scale, shift, rows, C, groups, eps, decay, relu, stream);
}
int agb_bn_forward_f32(void const* x, void const* residual, void* y, void const* gamma, void const* beta, void* moving_mean, void* moving_var, void* save_mean, void* save_rstd,
                   void* sums, void* scale, void* shift, long long rows, int C, int groups, float eps, float decay, int relu, void* stream) {
    return bn_forward_impl<float>(x, residual, y, gamma, beta, moving_mean, moving_var, save_mean, save_rstd, sums, scale, shift, rows, C, groups, eps, decay, relu, stream);
}


int agb_bn_backward(void const* dy, void const* x, void const* y, void const* mask_scale, void const* mask_shift, void const* gamma, void const* save_mean,
                    void const* save_rstd, void* dx, void* dmasked, void* dgamma, void* dbeta, void* sums, void* coef, long long rows, int C, int groups,
                    long long group_stride, void* stream) {
    return bn_backward_impl<bf16>(dy, x, y, mask_scale, mask_shift, gamma, save_mean, save_rstd, dx, dmasked, dgamma, dbeta, sums, coef, rows, C, groups, group_stride, stream);
}
int agb_bn_backward_f32(void const* dy, void const* x, void const* y, void const* mask_scale, void const* mask_shift, void const* gamma, void const* save_mean,
                    void const* save_rstd, void* dx, void* dmasked, void* dgamma, void* dbeta, void* sums, void* coef, long long rows, int C, int groups,
                    long long group_stride, void* stream) {
    return bn_backward_impl<float>(dy, x, y, mask_scale, mask_shift, gamma, save_mean, save_rstd, dx, dmasked, dgamma, dbeta, sums, coef, rows, C, groups, group_stride, stream);
}


// Single-launch variants; `ws` = zero-initialised workspace of agb_bn_fused_workspace_bytes() bytes, private to each direction.
int agb_bn_fused_set_limits(long long forward_mb, long long backward_mb, long long min_rows) {
    g_fused_max_mb[0] = forward_mb;
    g_fused_max_mb[1] = backward_mb;
    g_fused_min_rows = min_rows;
    return 0;
}

long long agb_bn_fused_workspace_bytes() {
    return 16 + 2 * kFusedHalfBytes;
}

// `residual` (optional, same shape as x): y = relu?(bn(x) + residual) — the closing add + ReLU of a residual unit.
// `scale` / `shift` (optional, [groups*C] each): the coefficients applied, as agb_bn_forward stores them.
int agb_bn_forward_fused(void const* x, void const* residual, void* y, void const* gamma, void const* beta, void* moving_mean, void* moving_var, void* save_mean, void* save_rstd,
                         void* scale, void* shift, void* ws, long long rows, int C, int groups, float eps, float decay, int relu, void* stream) {
    BnFused p{};
    p.a = static_cast<bf16 const*>(x); p.b = static_cast<bf16 const*>(residual); p.out = static_cast<bf16*>(y);
    p.gamma = static_cast<float const*>(gamma); p.beta = static_cast<float const*>(beta);
    p.moving_mean = static_cast<float*>(moving_mean); p.moving_var = static_cast<float*>(moving_var);
    p.save_mean = static_cast<float*>(save_mean); p.save_rstd = static_cast<float*>(save_rstd);
    p.scale = static_cast<float*>(scale); p.shift = static_cast<float*>(shift);
    p.state = static_cast<unsigned*>(ws); p.ws = static_cast<unsigned char*>(ws) + 16;
    p.C = C; p.groups = groups; p.eps = eps; p.decay = decay; p.relu = relu;
    return launch_bn_fused<false>(p, rows, static_cast<cudaStream_t>(stream));
}

// `dmasked` (optional, needs y): also stores dy * (y > 0), the gradient flowing into the residual input of the fused add + ReLU.
int agb_bn_backward_fused(void const* dy, void const* x, void const* y, void const* gamma, void const* save_mean, void const* save_rstd, void* dx, void* dmasked, void* dgamma,
                          void* dbeta, void* ws, long long rows, int C, int groups, long long group_stride, void* stream) {
    BnFused p{};
    p.a = static_cast<bf16 const*>(dy); p.b = static_cast<bf16 const*>(x); p.mask = static_cast<bf16 const*>(y); p.out = static_cast<bf16*>(dx);
    p.out2 = static_cast<bf16*>(dmasked);
    if (p.out2 && !p.mask)
        return 302;
    p.gamma = static_cast<float const*>(gamma);
    p.save_mean = const_cast<float*>(static_cast<float const*>(save_mean)); p.save_rstd = const_cast<float*>(static_cast<float const*>(save_rstd));
    p.dgamma = static_cast<float*>(dgamma); p.dbeta = static_cast<float*>(dbeta); p.group_stride = group_stride;
    p.state = static_cast<unsigned*>(ws); p.ws = static_cast<unsigned char*>(ws) + 16;
    p.C = C; p.groups = groups;
    return launch_bn_fused<true>(p, rows, static_cast<cudaStream_t>(stream));
}

// out[g * group_stride + c] = sum over the rows of group g of dy[r][c] (masked by y > 0 when y != null);
// `sums` is a double [2*C*groups + 1] workspace.
int agb_colsum(void const* dy, void const* y, void* out, void* sums, long long rows, int C, int groups, long long group_stride, void* stream) {
    return colsum_impl<bf16>(dy, y, out, sums, rows, C, groups, group_stride, stream);
}
int agb_colsum_f32(void const* dy, void const* y, void* out, void* sums, long long rows, int C, int groups, long long group_stride, void* stream) {
    return colsum_impl<float>(dy, y, out, sums, rows, C, groups, group_stride, stream);
}


int agb_add_relu(void const* a, void const* b, void* out, long long n, int relu, void* stream) {
    return add_relu_impl<bf16>(a, b, out, n, relu, stream);
}
int agb_add_relu_f32(void const* a, void const* b, void* out, long long n, int relu, void* stream) {
    return add_relu_impl<float>(a, b, out, n, relu, stream);
}


int agb_subsample_forward(void const* x, void* y, int N, int H, int W, int C, int s, void* stream) {
    return subsample_forward_impl<bf16>(x, y, N, H, W, C, s, stream);
}
int agb_subsample_forward_f32(void const* x, void* y, int N, int H, int W, int C, int s, void* stream) {
    return subsample_forward_impl<float>(x, y, N, H, W, C, s, stream);
}


int agb_subsample_backward(void const* dy, void* dx, int N, int H, int W, int C, int s, void* stream) {
    return subsample_backward_impl<bf16>(dy, dx, N, H, W, C, s, stream);
}
int agb_subsample_backward_f32(void const* dy, void* dx, int N, int H, int W, int C, int s, void* stream) {
    return subsample_backward_impl<float>(dy, dx, N, H, W, C, s, stream);
}


// dx[n, h*s, w*s, :] += dy[n, h, w, :] in place: the gradient of a strided shortcut summed into the residual branch's.
int agb_subsample_add(void const* dy, void* dx, int N, int H, int W, int C, int s, void* stream) {
    return subsample_add_impl<bf16>(dy, dx, N, H, W, C, s, stream);
}
int agb_subsample_add_f32(void const* dy, void* dx, int N, int H, int W, int C, int s, void* stream) {
    return subsample_add_impl<float>(dy, dx, N, H, W, C, s, stream);
}


int agb_relu_backward(void const* dy, void const* y, void* dx, long long n, void* stream) {
    return relu_backward_impl<bf16>(dy, y, dx, n, stream);
}
int agb_relu_backward_f32(void const* dy, void const* y, void* dx, long long n, void* stream) {
    return relu_backward_impl<float>(dy, y, dx, n, stream);
}


int agb_maxpool_forward(void const* x, void* y, void* arg, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    return maxpool_forward_impl<bf16>(x, y, arg, N, H, W, C, OH, OW, k, s, pad_t, pad_l, stream);
}
int agb_maxpool_forward_f32(void const* x, void* y, void* arg, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    return maxpool_forward_impl<float>(x, y, arg, N, H, W, C, OH, OW, k, s, pad_t, pad_l, stream);
}


int agb_maxpool_backward(void const* dy, void const* arg, void* dx, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    return maxpool_backward_impl<bf16>(dy, arg, dx, N, H, W, C, OH, OW, k, s, pad_t, pad_l, stream);
}
int agb_maxpool_backward_f32(void const* dy, void const* arg, void* dx, int N, int H, int W, int C, int OH, int OW, int k, int s, int pad_t, int pad_l, void* stream) {
    return maxpool_backward_impl<float>(dy, arg, dx, N, H, W, C, OH, OW, k, s, pad_t, pad_l, stream);
}


int agb_avgpool_forward(void const* x, void* y, int N, int HW, int C, void* stream) {
    return avgpool_forward_impl<bf16>(x, y, N, HW, C, stream);
}
int agb_avgpool_forward_f32(void const* x, void* y, int N, int HW, int C, void* stream) {
    return avgpool_forward_impl<float>(x, y, N, HW, C, stream);
}


int agb_avgpool_backward(void const* dy, void* dx, int N, int HW, int C, void* stream) {
    return avgpool_backward_impl<bf16>(dy, dx, N, HW, C, stream);
}
int agb_avgpool_backward_f32(void const* dy, void* dx, int N, int HW, int C, void* stream) {
    return avgpool_backward_impl<float>(dy, dx, N, HW, C, stream);
}


int agb_softmax_xent(void const* logits, void const* labels, void* dlogits, void* loss, int B, int K, long long ld, float smoothing, int groups, void* stream) {
    return softmax_xent_impl<bf16>(logits, labels, dlogits, loss, B, K, ld, smoothing, groups, groups, 0, -1, 1.f, stream);
}
int agb_softmax_xent_f32(void const* logits, void const* labels, void* dlogits, void* loss, int B, int K, long long ld, float smoothing, int groups, void* stream) {
    return softmax_xent_impl<float>(logits, labels, dlogits, loss, B, K, ld, smoothing, groups, groups, 0, -1, 1.f, stream);
}
// The same, with the labels of the groups >= flip_from (0 <= flip_from <= groups) flipped to K - 1 - y.
int agb_softmax_xent_flip(void const* logits, void const* labels, void* dlogits, void* loss, int B, int K, long long ld, float smoothing, int groups, int flip_from, void* stream) {
    return softmax_xent_impl<bf16>(logits, labels, dlogits, loss, B, K, ld, smoothing, groups, flip_from, groups >= 1 ? B / groups : 0, -1, 1.f, stream);
}
int agb_softmax_xent_flip_f32(void const* logits, void const* labels, void* dlogits, void* loss, int B, int K, long long ld, float smoothing, int groups, int flip_from, void* stream) {
    return softmax_xent_impl<float>(logits, labels, dlogits, loss, B, K, ld, smoothing, groups, flip_from, groups >= 1 ? B / groups : 0, -1, 1.f, stream);
}
// The backdoor: in the groups >= poison_from (0 <= poison_from <= groups), the rows with row % (B / groups) < q (0 <= q <= B / groups)
// train on `target` (0 <= target < K), and every row's dlogits is multiplied by `scale` (finite, > 0). Invalid parameters: status 303.
static bool backdoor_checked(int B, int K, int groups, int poison_from, int q, int target, float scale) {
    return groups >= 1 && B % groups == 0 && poison_from >= 0 && poison_from <= groups && q >= 0 && q <= B / groups && target >= 0 && target < K
        && std::isfinite(scale) && scale > 0.f;
}
int agb_softmax_xent_backdoor(void const* logits, void const* labels, void* dlogits, void* loss, int B, int K, long long ld, float smoothing, int groups,
                              int poison_from, int q, int target, float scale, void* stream) {
    if (!backdoor_checked(B, K, groups, poison_from, q, target, scale))
        return 303;
    return softmax_xent_impl<bf16>(logits, labels, dlogits, loss, B, K, ld, smoothing, groups, poison_from, q, target, scale, stream);
}
int agb_softmax_xent_backdoor_f32(void const* logits, void const* labels, void* dlogits, void* loss, int B, int K, long long ld, float smoothing, int groups,
                                  int poison_from, int q, int target, float scale, void* stream) {
    if (!backdoor_checked(B, K, groups, poison_from, q, target, scale))
        return 303;
    return softmax_xent_impl<float>(logits, labels, dlogits, loss, B, K, ld, smoothing, groups, poison_from, q, target, scale, stream);
}


int agb_image_normalize(void const* x, void* y, long long pixels, int C, int Cpad, float m0, float m1, float m2, float scale, void* stream) {
    return image_normalize_impl<bf16>(x, y, pixels, C, Cpad, m0, m1, m2, scale, 1, 1, Trigger{1, 0, 0, 0}, stream);
}
int agb_image_normalize_f32(void const* x, void* y, long long pixels, int C, int Cpad, float m0, float m1, float m2, float scale, void* stream) {
    return image_normalize_impl<float>(x, y, pixels, C, Cpad, m0, m1, m2, scale, 1, 1, Trigger{1, 0, 0, 0}, stream);
}
// The same on N images of H x W, with the backdoor trigger (side s >= 1) stamped on image b iff b / rows >= first and b % rows < q.
// Invalid descriptor: status 503.
int agb_image_normalize_backdoor(void const* x, void* y, int N, int H, int W, int C, int Cpad, float m0, float m1, float m2, float scale,
                                 int rows, int first, int q, int s, void* stream) {
    Trigger const t{rows, first, q, s};
    if (N < 1 || H < 1 || W < 1 || s < 1 || !trigger_valid(t, N, H, W))
        return 503;
    return image_normalize_impl<bf16>(x, y, static_cast<long long>(N) * H * W, C, Cpad, m0, m1, m2, scale, H, W, t, stream);
}
int agb_image_normalize_backdoor_f32(void const* x, void* y, int N, int H, int W, int C, int Cpad, float m0, float m1, float m2, float scale,
                                     int rows, int first, int q, int s, void* stream) {
    Trigger const t{rows, first, q, s};
    if (N < 1 || H < 1 || W < 1 || s < 1 || !trigger_valid(t, N, H, W))
        return 503;
    return image_normalize_impl<float>(x, y, static_cast<long long>(N) * H * W, C, Cpad, m0, m1, m2, scale, H, W, t, stream);
}


int agb_im2col(void const* x, void* col, int N, int H, int W, int C, int OH, int OW, int kh, int kw, int s, int pad_t, int pad_l, long long ldcol, void* stream) {
    return im2col_impl<bf16>(x, col, N, H, W, C, OH, OW, kh, kw, s, pad_t, pad_l, ldcol, stream);
}
int agb_im2col_f32(void const* x, void* col, int N, int H, int W, int C, int OH, int OW, int kh, int kw, int s, int pad_t, int pad_l, long long ldcol, void* stream) {
    return im2col_impl<float>(x, col, N, H, W, C, OH, OW, kh, kw, s, pad_t, pad_l, ldcol, stream);
}


int agb_col2im(void const* dcol, void* dx, int N, int H, int W, int C, int OH, int OW, int kh, int kw, int s, int pad_t, int pad_l, long long ldcol, void* stream) {
    return col2im_impl<bf16>(dcol, dx, N, H, W, C, OH, OW, kh, kw, s, pad_t, pad_l, ldcol, stream);
}
int agb_col2im_f32(void const* dcol, void* dx, int N, int H, int W, int C, int OH, int OW, int kh, int kw, int s, int pad_t, int pad_l, long long ldcol, void* stream) {
    return col2im_impl<float>(dcol, dx, N, H, W, C, OH, OW, kh, kw, s, pad_t, pad_l, ldcol, stream);
}


} // extern "C"
