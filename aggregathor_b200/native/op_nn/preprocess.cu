// Input preprocessing on the device, one launch per batch: uint8 NHWC images at their *storage* resolution -> network-resolution
// activations (bf16 or fp32 NHWC) with slim's training / evaluation preprocessing semantics
// (reference: `external/slim/preprocessing/preprocessing_factory.py:64` and the slim modules it dispatches to, used by
// `experiments/slims.py:100-111` and `experiments/cnnet.py:123-130`):
//
//   vgg        train: aspect-preserving resize so that the short side is r ~ U{resize_min..resize_max}, random OH x OW crop, random
//              mirror, mean-image subtraction;  eval: r = resize_min, central crop
//   inception  train: distorted bounding-box crop (area fraction ~ U[area_min, area_max], aspect ~ U[3/4, 4/3], up to 10 attempts),
//              bilinear resize to OH x OW, random mirror, colour distortion in one of TF's four orderings (brightness 32/255,
//              saturation [0.5, 1.5], hue 0.2, contrast [0.5, 1.5]), clip, scale to [-1, 1];  eval: central 87.5 % crop + resize
//   cifarnet   train: zero-pad by `pad`, random OH x OW crop, random mirror, brightness (delta 63), contrast [0.2, 1.8], per-image
//              standardisation;  eval: central crop / pad + standardisation
//   plain      (x - mean) * scale after a bilinear resize of the whole image (lenet-style and user-defined preprocessing)
//
// The backdoor attack's trigger (`Trigger` in agb_device.cuh) is written into the sampled pixel, after the geometric operations
// (crop, resize, mirror) and before every photometric one, so that it sits at the same place of the network input and the per-image
// statistics include it.
//
// "Resize then crop" never materialises the resized image: every output pixel samples the source box directly (bilinear,
// TF1 `resize_bilinear` coordinates: src = origin + index * box / out). One CTA per image; operations that need a per-image
// statistic (contrast, standardisation) run a first pass that reduces it in the CTA. All randomness is counter based —
// hash(seed, *counter, image, slot) — and the counter lives in device memory, so a training step that augments its inputs can
// still be captured once in a CUDA graph and replayed (the host bumps the counter with a captured one-element add).

#include <cuda_bf16.h>

#include <agb_device.cuh>

using namespace agb;

namespace {

enum Mode { kPlain = 0, kVgg = 1, kInception = 2, kCifarnet = 3 };

struct PreprocParams {
    unsigned char const* src;   // [N, SH, SW, C] uint8
    void* dst;                  // [N, OH, OW, C] bf16 / fp32
    int N, SH, SW, C, OH, OW;
    int mode, training, out_fp32;
    int resize_min, resize_max; // vgg
    float area_min, area_max;   // inception
    int pad;                    // cifarnet
    float mean[3], scale;       // plain / vgg: (v - mean[c]) * scale
    unsigned long long seed;
    unsigned long long const* counter;   // device step counter (null = 0)
    Trigger trigger;                     // backdoor trigger of the poisoned images (s = 0: none)
};

__device__ __forceinline__ float uniform01(unsigned long long seed, unsigned long long step, unsigned image, unsigned slot) {
    unsigned long long h = seed ^ (step * 0x9E3779B97F4A7C15ull) ^ (static_cast<unsigned long long>(image) << 32 | slot) * 0xD1B54A32D192ED03ull;
    h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
    return static_cast<float>(h >> 40) * (1.0f / 16777216.0f);   // [0, 1)
}

// Per-image geometry + colour parameters (identical in every thread of the CTA).
struct Sampling {
    float y0, x0, sy, sx;     // source = origin + index * step
    bool flip;
    bool zero_outside;        // cifarnet padding: outside the image is 0, otherwise clamp to the border
    float brightness, contrast, saturation, hue;
    int ordering;             // inception colour ordering 0..3, -1 = no colour ops
};

__device__ Sampling make_sampling(PreprocParams const& p, unsigned image, unsigned long long step) {
    Sampling s{};
    s.ordering = -1;
    s.contrast = 1.f; s.saturation = 1.f;
    auto rnd = [&](unsigned slot) { return uniform01(p.seed, step, image, slot); };
    if (p.mode == kVgg) {
        int const r = p.training ? p.resize_min + static_cast<int>(rnd(0) * (p.resize_max - p.resize_min + 1)) : p.resize_min;
        float const scale = static_cast<float>(r) / static_cast<float>(min(p.SH, p.SW));   // resized = source * scale
        float const RH = p.SH * scale, RW = p.SW * scale;
        float const oy = p.training ? rnd(1) * fmaxf(RH - p.OH, 0.f) : 0.5f * fmaxf(RH - p.OH, 0.f);
        float const ox = p.training ? rnd(2) * fmaxf(RW - p.OW, 0.f) : 0.5f * fmaxf(RW - p.OW, 0.f);
        s.y0 = floorf(oy) / scale; s.x0 = floorf(ox) / scale;
        s.sy = 1.f / scale; s.sx = 1.f / scale;
        s.flip = p.training && rnd(3) < 0.5f;
    } else if (p.mode == kInception) {
        float bh = p.SH, bw = p.SW, y0 = 0.f, x0 = 0.f;
        if (p.training) {
            for (int attempt = 0; attempt < 10; ++attempt) {
                float const aspect = 0.75f + rnd(8 + 2 * attempt) * (4.f / 3.f - 0.75f);
                float const area = (p.area_min + rnd(9 + 2 * attempt) * (p.area_max - p.area_min)) * p.SH * p.SW;
                float const w = sqrtf(area * aspect), h = sqrtf(area / aspect);
                if (w <= p.SW && h <= p.SH && w >= 1.f && h >= 1.f) {
                    bw = w; bh = h;
                    break;
                }
            }
            y0 = rnd(1) * (p.SH - bh); x0 = rnd(2) * (p.SW - bw);
            s.flip = rnd(3) < 0.5f;
            s.ordering = static_cast<int>(rnd(4) * 4.f) & 3;
            s.brightness = (2.f * rnd(5) - 1.f) * (32.f / 255.f);
            s.saturation = 0.5f + rnd(6);
            s.hue = (2.f * rnd(7) - 1.f) * 0.2f;
            s.contrast = 0.5f + rnd(28);
        } else {
            bh = 0.875f * p.SH; bw = 0.875f * p.SW;
            y0 = 0.5f * (p.SH - bh); x0 = 0.5f * (p.SW - bw);
        }
        s.y0 = y0; s.x0 = x0; s.sy = bh / p.OH; s.sx = bw / p.OW;
    } else if (p.mode == kCifarnet) {
        int const range_y = p.SH + 2 * p.pad - p.OH, range_x = p.SW + 2 * p.pad - p.OW;
        int const oy = p.training ? static_cast<int>(rnd(1) * (range_y + 1)) : range_y / 2;
        int const ox = p.training ? static_cast<int>(rnd(2) * (range_x + 1)) : range_x / 2;
        s.y0 = static_cast<float>(oy - p.pad); s.x0 = static_cast<float>(ox - p.pad);
        s.sy = 1.f; s.sx = 1.f;
        s.zero_outside = true;
        if (p.training) {
            s.flip = rnd(3) < 0.5f;
            s.brightness = (2.f * rnd(5) - 1.f) * 63.f;
            s.contrast = 0.2f + rnd(6) * 1.6f;
        }
    } else {
        s.sy = static_cast<float>(p.SH) / p.OH; s.sx = static_cast<float>(p.SW) / p.OW;
    }
    return s;
}

// Bilinear sample of all (<= 3) channels of one output pixel, in uint8 units [0, 255].
__device__ __forceinline__ void sample_pixel(PreprocParams const& p, Sampling const& s, unsigned char const* img, int oy, int ox, float (&v)[3]) {
    int const oxs = s.flip ? p.OW - 1 - ox : ox;
    float const fy = s.y0 + oy * s.sy, fx = s.x0 + oxs * s.sx;
    float const fy0 = floorf(fy), fx0 = floorf(fx);
    float const wy = fy - fy0, wx = fx - fx0;
    int const y0 = static_cast<int>(fy0), x0 = static_cast<int>(fx0);
#pragma unroll
    for (int c = 0; c < 3; ++c)
        v[c] = 0.f;
#pragma unroll
    for (int dy = 0; dy < 2; ++dy) {
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            float const w = (dy ? wy : 1.f - wy) * (dx ? wx : 1.f - wx);
            if (w == 0.f)
                continue;
            int y = y0 + dy, x = x0 + dx;
            if (s.zero_outside) {
                if (y < 0 || y >= p.SH || x < 0 || x >= p.SW)
                    continue;
            } else {
                y = min(max(y, 0), p.SH - 1);
                x = min(max(x, 0), p.SW - 1);
            }
            unsigned char const* px = img + (static_cast<long long>(y) * p.SW + x) * p.C;
            for (int c = 0; c < p.C; ++c)
                v[c] += w * static_cast<float>(px[c]);
        }
    }
}

__device__ __forceinline__ void adjust_saturation(float (&v)[3], float factor) {
    float const gray = 0.2989f * v[0] + 0.587f * v[1] + 0.114f * v[2];   // tf.image.rgb_to_grayscale weights
#pragma unroll
    for (int c = 0; c < 3; ++c)
        v[c] = gray + (v[c] - gray) * factor;
}
// Hue rotation by `delta` turns, as a rotation of the chroma plane of YIQ (what `adjust_hue` computes up to HSV's piecewise hexagon).
__device__ __forceinline__ void adjust_hue(float (&v)[3], float delta) {
    float sn, cs;
    sincospif(2.f * delta, &sn, &cs);
    float const y = 0.299f * v[0] + 0.587f * v[1] + 0.114f * v[2];
    float const i = 0.596f * v[0] - 0.274f * v[1] - 0.322f * v[2];
    float const q = 0.211f * v[0] - 0.523f * v[1] + 0.312f * v[2];
    float const i2 = i * cs - q * sn, q2 = i * sn + q * cs;
    v[0] = y + 0.956f * i2 + 0.621f * q2;
    v[1] = y - 0.272f * i2 - 0.647f * q2;
    v[2] = y - 1.106f * i2 + 1.703f * q2;
}

// The colour operations of slim's `distort_color` that come BEFORE (`before` = true) or AFTER the contrast adjustment in ordering `o`
// (values in [0, 1]). Orderings: 0 = B S H C, 1 = S B C H, 2 = C H B S, 3 = H S C B.
__device__ __forceinline__ void colour_ops(float (&v)[3], Sampling const& s, int channels, bool before) {
    auto brightness = [&] {
#pragma unroll
        for (int c = 0; c < 3; ++c)
            v[c] += s.brightness;
    };
    bool const rgb = channels == 3;
    switch (s.ordering) {
        case 0: if (before) { brightness(); if (rgb) { adjust_saturation(v, s.saturation); adjust_hue(v, s.hue); } } break;
        case 1: if (before) { if (rgb) adjust_saturation(v, s.saturation); brightness(); } else if (rgb) adjust_hue(v, s.hue); break;
        case 2: if (!before) { if (rgb) adjust_hue(v, s.hue); brightness(); if (rgb) adjust_saturation(v, s.saturation); } break;
        case 3: if (before) { if (rgb) { adjust_hue(v, s.hue); adjust_saturation(v, s.saturation); } } else brightness(); break;
        default: break;
    }
}

template<typename OUT> __device__ __forceinline__ OUT to_out(float v);
template<> __device__ __forceinline__ float to_out<float>(float v) { return v; }
template<> __device__ __forceinline__ __nv_bfloat16 to_out<__nv_bfloat16>(float v) { return __float2bfloat16(v); }

template<typename OUT>
__global__ void __launch_bounds__(512) preprocess_kernel(PreprocParams const p) {
    __shared__ float red[16][8];
    __shared__ float stats[8];
    unsigned const image = blockIdx.x;
    unsigned long long const step = p.counter ? *p.counter : 0ull;
    Sampling const s = make_sampling(p, image, step);
    unsigned char const* img = p.src + static_cast<long long>(image) * p.SH * p.SW * p.C;
    OUT* out = static_cast<OUT*>(p.dst) + static_cast<long long>(image) * p.OH * p.OW * p.C;
    int const pixels = p.OH * p.OW;
    bool const inception_train = p.mode == kInception && p.training;
    bool const cifar = p.mode == kCifarnet;
    bool const need_stats = inception_train || cifar;
    bool const poisoned = trigger_poisoned(p.trigger, image);

    // value of one output pixel up to (not including) the statistic-dependent operation
    auto stage1 = [&](int idx, float (&v)[3]) {
        sample_pixel(p, s, img, idx / p.OW, idx % p.OW, v);
        if (poisoned) {
            float const t = trigger_value(p.trigger, p.OH, p.OW, idx / p.OW, idx % p.OW);
            if (t >= 0.f) {
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    if (c < p.C)
                        v[c] = t;
            }
        }
        if (p.mode == kInception) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
                v[c] *= (1.f / 255.f);
            if (p.training)
                colour_ops(v, s, p.C, true);
        } else if (cifar) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
                v[c] += s.brightness;
        }
    };

    float mean_c[3] = {0.f, 0.f, 0.f};
    if (need_stats) {   // pass 1: per-channel sums (contrast pivots)
        float acc[3] = {0.f, 0.f, 0.f};
        for (int idx = threadIdx.x; idx < pixels; idx += blockDim.x) {
            float v[3];
            stage1(idx, v);
#pragma unroll
            for (int c = 0; c < 3; ++c)
                acc[c] += v[c];
        }
        int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            float const t = warp_sum(acc[c]);
            if (lane == 0)
                red[warp][c] = t;
        }
        __syncthreads();
        if (threadIdx.x < 3) {
            float t = 0.f;
            for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w)
                t += red[w][threadIdx.x];
            stats[threadIdx.x] = t / static_cast<float>(pixels);
        }
        __syncthreads();
#pragma unroll
        for (int c = 0; c < 3; ++c)
            mean_c[c] = stats[c];
    }
    // statistic-dependent part up to the final affine map
    auto stage2 = [&](float (&v)[3]) {
        if (inception_train) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
                v[c] = (v[c] - mean_c[c]) * s.contrast + mean_c[c];
            colour_ops(v, s, p.C, false);
#pragma unroll
            for (int c = 0; c < 3; ++c)
                v[c] = fminf(fmaxf(v[c], 0.f), 1.f);
        } else if (cifar) {
#pragma unroll
            for (int c = 0; c < 3; ++c)
                v[c] = (v[c] - mean_c[c]) * s.contrast + mean_c[c];
        }
    };

    float std_mean = 0.f, std_inv = 1.f;
    if (cifar) {   // per-image standardisation over all channels: second reduction (mean, mean of squares) of the adjusted image
        // The sums run around a centre known before the sweep: contrast keeps each channel's mean at mean_c, so the mean of the
        // mean_c is the image mean up to rounding. E[v^2] - E[v]^2 taken around 0 would lose the variance of bright, nearly uniform
        // images (values near 300, variance near 0.02) to the rounding of E[v^2].
        float centre = 0.f;
        for (int c = 0; c < p.C; ++c)
            centre += mean_c[c];
        centre /= static_cast<float>(p.C);
        float a0 = 0.f, a1 = 0.f;
        for (int idx = threadIdx.x; idx < pixels; idx += blockDim.x) {
            float v[3];
            stage1(idx, v);
            stage2(v);
            for (int c = 0; c < p.C; ++c) {
                float const d = v[c] - centre;
                a0 += d;
                a1 += d * d;
            }
        }
        int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        a0 = warp_sum(a0); a1 = warp_sum(a1);
        __syncthreads();
        if (lane == 0) {
            red[warp][3] = a0;
            red[warp][4] = a1;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            float t0 = 0.f, t1 = 0.f;
            for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) {
                t0 += red[w][3];
                t1 += red[w][4];
            }
            float const count = static_cast<float>(pixels) * p.C;
            float const shift = t0 / count;   // mean - centre
            float const var = fmaxf(t1 / count - shift * shift, 0.f);
            stats[3] = centre + shift;
            stats[4] = 1.f / fmaxf(sqrtf(var), rsqrtf(count));   // tf.image.per_image_standardization: max(stddev, 1/sqrt(N))
        }
        __syncthreads();
        std_mean = stats[3]; std_inv = stats[4];
    }

    for (int idx = threadIdx.x; idx < pixels; idx += blockDim.x) {
        float v[3];
        stage1(idx, v);
        stage2(v);
        for (int c = 0; c < p.C; ++c) {
            float r;
            if (p.mode == kInception)
                r = (v[c] - 0.5f) * 2.f;
            else if (cifar)
                r = (v[c] - std_mean) * std_inv;
            else
                r = (v[c] - p.mean[c]) * p.scale;
            out[static_cast<long long>(idx) * p.C + c] = to_out<OUT>(r);
        }
    }
}

int image_preprocess(void const* src, void* dst, int const* ints, float const* floats, unsigned long long seed, void const* counter, Trigger trigger, void* stream) {
    PreprocParams p{};
    p.src = static_cast<unsigned char const*>(src);
    p.dst = dst;
    p.N = ints[0]; p.SH = ints[1]; p.SW = ints[2]; p.C = ints[3]; p.OH = ints[4]; p.OW = ints[5];
    p.mode = ints[6]; p.training = ints[7]; p.out_fp32 = ints[8];
    p.resize_min = ints[9]; p.resize_max = ints[10]; p.pad = ints[11];
    p.area_min = floats[0]; p.area_max = floats[1];
    p.mean[0] = floats[2]; p.mean[1] = floats[3]; p.mean[2] = floats[4]; p.scale = floats[5];
    p.seed = seed;
    p.counter = static_cast<unsigned long long const*>(counter);
    p.trigger = trigger;
    if (p.N < 1 || p.C < 1 || p.C > 3 || p.SH < 1 || p.SW < 1 || p.OH < 1 || p.OW < 1 || p.mode < 0 || p.mode > kCifarnet)
        return 501;
    if (p.mode == kVgg && (p.resize_min < 1 || p.resize_max < p.resize_min))
        return 502;
    if (!trigger_valid(p.trigger, p.N, p.OH, p.OW))
        return 503;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (p.out_fp32)
        preprocess_kernel<float><<<p.N, 512, 0, s>>>(p);
    else
        preprocess_kernel<__nv_bfloat16><<<p.N, 512, 0, s>>>(p);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

} // namespace

extern "C" {

// ints: N SH SW C OH OW mode training out_fp32 resize_min resize_max pad ; floats: area_min area_max mean0 mean1 mean2 scale
int agb_image_preprocess(void const* src, void* dst, int const* ints, float const* floats, unsigned long long seed, void const* counter, void* stream) {
    return image_preprocess(src, dst, ints, floats, seed, counter, Trigger{1, 0, 0, 0}, stream);
}
// The same, with the backdoor trigger (side s >= 1) stamped on image b iff b / rows >= first and b % rows < q; 503: invalid descriptor.
int agb_image_preprocess_backdoor(void const* src, void* dst, int const* ints, float const* floats, unsigned long long seed, void const* counter,
                                  int rows, int first, int q, int s, void* stream) {
    if (s < 1)
        return 503;
    return image_preprocess(src, dst, ints, floats, seed, counter, Trigger{rows, first, q, s}, stream);
}

} // extern "C"
