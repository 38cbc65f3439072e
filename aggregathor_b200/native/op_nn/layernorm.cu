// LayerNorm forward / backward (sm_90a): rows x C bf16 activations, fp32 gamma/beta, one warp per row.
// The reference's models only use batch-norm, but LayerNorm is one of the hot ops named for this framework's model zoo
// (transformer-style heads plug into the same static layer graph through models.core.LayerNorm).
//   forward : y = (x - mean) * rstd * gamma + beta, saves mean / rstd per row
//   backward: dx = rstd * (g - mean(g) - xhat * mean(g * xhat)), g = dy * gamma ; dgamma += sum_rows dy * xhat ; dbeta += sum_rows dy
// C % 8 == 0, C <= 8192. Column sums of the backward pass are accumulated per CTA in shared memory, then one fp32 atomic
// per column and CTA.

#include <cuda_bf16.h>

#include <agb_device.cuh>

using namespace agb;

namespace {

using bf16 = __nv_bfloat16;
constexpr int kWarpsPerCta = 8;
constexpr int kMaxOctetsPerLane = 32;   // C <= 32 lanes * 32 octets * 8 = 8192

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

__global__ void __launch_bounds__(kWarpsPerCta * 32) layernorm_fwd_kernel(bf16 const* __restrict__ x, bf16* __restrict__ y, float const* __restrict__ gamma, float const* __restrict__ beta,
                                                                          float* __restrict__ mean_out, float* __restrict__ rstd_out, long long rows, int C, float eps) {
    int const lane = threadIdx.x & 31;
    long long const row = static_cast<long long>(blockIdx.x) * kWarpsPerCta + (threadIdx.x >> 5);
    if (row >= rows)
        return;
    int const octets = C >> 3;
    bf16 const* xr = x + row * C;
    // sums of (x - pivot) with the row's first element as pivot: sumsq / C - shifted^2 stays well conditioned when |mean| >> std
    float const pivot = __bfloat162float(xr[0]);
    float sum = 0.f, sumsq = 0.f;
    for (int o = lane; o < octets; o += 32) {
        float v[8];
        unpack8(*reinterpret_cast<uint4 const*>(xr + o * 8), v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float const d = v[j] - pivot;
            sum += d;
            sumsq += d * d;
        }
    }
    sum = warp_sum(sum);
    sumsq = warp_sum(sumsq);
    float const shifted = sum / C;
    float const mean = pivot + shifted;
    float const var = fmaxf(sumsq / C - shifted * shifted, 0.f);
    float const rstd = rsqrtf(var + eps);
    if (lane == 0) {
        mean_out[row] = mean;
        rstd_out[row] = rstd;
    }
    bf16* yr = y + row * C;
    for (int o = lane; o < octets; o += 32) {
        float v[8];
        unpack8(*reinterpret_cast<uint4 const*>(xr + o * 8), v);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            v[j] = (v[j] - mean) * rstd * gamma[o * 8 + j] + beta[o * 8 + j];
        *reinterpret_cast<uint4*>(yr + o * 8) = pack8(v);
    }
}

__global__ void __launch_bounds__(kWarpsPerCta * 32) layernorm_bwd_kernel(bf16 const* __restrict__ dy, bf16 const* __restrict__ x, float const* __restrict__ gamma, float const* __restrict__ mean,
                                                                          float const* __restrict__ rstd, bf16* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                                          long long rows, int C, int rows_per_cta) {
    extern __shared__ float col[];   // [2][C] per-CTA column sums (dgamma, dbeta)
    for (int i = threadIdx.x; i < 2 * C; i += blockDim.x)
        col[i] = 0.f;
    __syncthreads();
    int const lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int const octets = C >> 3;
    long long const row_begin = static_cast<long long>(blockIdx.x) * rows_per_cta;
    long long const row_end = min(rows, row_begin + rows_per_cta);
    for (long long row = row_begin + warp; row < row_end; row += kWarpsPerCta) {
        float const mu = mean[row], rs = rstd[row];
        bf16 const* xr = x + row * C;
        bf16 const* dr = dy + row * C;
        float s1 = 0.f, s2 = 0.f;
        for (int o = lane; o < octets; o += 32) {
            float vx[8], vd[8];
            unpack8(*reinterpret_cast<uint4 const*>(xr + o * 8), vx);
            unpack8(*reinterpret_cast<uint4 const*>(dr + o * 8), vd);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float const xhat = (vx[j] - mu) * rs, g = vd[j] * gamma[o * 8 + j];
                s1 += g;
                s2 += g * xhat;
                atomicAdd(col + o * 8 + j, vd[j] * xhat);       // shared-memory atomics: 8 warps share the column sums
                atomicAdd(col + C + o * 8 + j, vd[j]);
            }
        }
        s1 = warp_sum(s1) / C;
        s2 = warp_sum(s2) / C;
        bf16* xo = dx + row * C;
        for (int o = lane; o < octets; o += 32) {
            float vx[8], vd[8];
            unpack8(*reinterpret_cast<uint4 const*>(xr + o * 8), vx);
            unpack8(*reinterpret_cast<uint4 const*>(dr + o * 8), vd);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float const xhat = (vx[j] - mu) * rs;
                vd[j] = rs * (vd[j] * gamma[o * 8 + j] - s1 - xhat * s2);
            }
            *reinterpret_cast<uint4*>(xo + o * 8) = pack8(vd);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < C; i += blockDim.x) {
        atomicAdd(dgamma + i, col[i]);
        atomicAdd(dbeta + i, col[C + i]);
    }
}

} // namespace

extern "C" {

int agb_layernorm_forward(void const* x, void* y, void const* gamma, void const* beta, void* mean, void* rstd, long long rows, int C, float eps, void* stream) {
    if ((C & 7) || C > 32 * kMaxOctetsPerLane * 8)
        return 301;
    int const blocks = static_cast<int>((rows + kWarpsPerCta - 1) / kWarpsPerCta);
    if (blocks > 0)
        layernorm_fwd_kernel<<<blocks, kWarpsPerCta * 32, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<bf16 const*>(x), static_cast<bf16*>(y), static_cast<float const*>(gamma),
            static_cast<float const*>(beta), static_cast<float*>(mean), static_cast<float*>(rstd), rows, C, eps);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

// dgamma / dbeta must be zeroed by the caller (they are accumulated with atomics).
int agb_layernorm_backward(void const* dy, void const* x, void const* gamma, void const* mean, void const* rstd, void* dx, void* dgamma, void* dbeta, long long rows, int C, void* stream) {
    if ((C & 7) || C > 5632)   // 2 * C floats of shared memory per CTA (<= 44 KB)
        return 301;
    long long ctas = agb::sm_count() * 4;
    long long rows_per_cta = (rows + ctas - 1) / ctas;
    if (rows_per_cta < kWarpsPerCta)
        rows_per_cta = kWarpsPerCta;
    int const blocks = static_cast<int>((rows + rows_per_cta - 1) / rows_per_cta);
    if (blocks > 0)
        layernorm_bwd_kernel<<<blocks, kWarpsPerCta * 32, 2 * C * sizeof(float), static_cast<cudaStream_t>(stream)>>>(static_cast<bf16 const*>(dy), static_cast<bf16 const*>(x),
            static_cast<float const*>(gamma), static_cast<float const*>(mean), static_cast<float const*>(rstd), static_cast<bf16*>(dx), static_cast<float*>(dgamma), static_cast<float*>(dbeta),
            rows, C, static_cast<int>(rows_per_cta));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

} // extern "C"
