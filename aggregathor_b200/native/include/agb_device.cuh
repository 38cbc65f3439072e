// Device-side helpers shared by the sm_90a kernel libraries: error macro, SM count, system-scope
// synchronisation primitives for peer-mapped memory, streaming vector loads/stores, NVLS
// (multimem) wrappers, warp/block reductions.
#pragma once

#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

#define AGB_CUDA_OK(expr) do { cudaError_t err__ = (expr); if (err__ != cudaSuccess) { \
    std::fprintf(stderr, "[agb] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(err__), __FILE__, __LINE__, cudaGetErrorString(err__)); \
    return static_cast<int>(err__) ? static_cast<int>(err__) : 1; } } while (0)

#include <cstdlib>
#include <utility>

namespace agb {

// Streaming multiprocessors of the current device (132 on an H100 SXM), queried once: grid sizes and caps of every library scale with it.
inline int sm_count() {
    static int sms = 0;
    if (sms == 0) {
        int device = 0, value = 0;
        if (cudaGetDevice(&device) == cudaSuccess && cudaDeviceGetAttribute(&value, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && value > 0)
            sms = value;
        else
            return 132;
    }
    return sms;
}

// ---- programmatic dependent launch (PDL) ------------------------------------ //
// Kernels launched through `launch_pdl` may start while their predecessor in the stream is still draining: everything before
// `pdl_wait()` (barrier / TMEM / tensor-map set-up, shared-memory initialisation) overlaps the predecessor's tail; `pdl_wait()`
// returns once the predecessor has completed and its memory is visible. `pdl_trigger()` lets the *next* kernel start launching.
__device__ __forceinline__ void pdl_wait() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ void pdl_trigger() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
inline int& pdl_state() {
    static int state = -1;   // -1: read AGB_PDL at first use; 0 / 1: set (environment or `set_pdl`)
    return state;
}
inline bool pdl_enabled() {
    int& state = pdl_state();
    if (state < 0) {
        char const* env = std::getenv("AGB_PDL");
        state = env ? (std::atoi(env) != 0) : 0;   // opt-in: neutral under CUDA-graph replay of batched workers, ~3 % on batch-32 passes (profiles/README.md)
    }
    return state != 0;
}
inline void set_pdl(int enabled) {
    pdl_state() = enabled ? 1 : 0;
}
template<typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// ---- system-scope flags (cross-GPU) -------------------------------------- //
__device__ __forceinline__ void st_release_sys(uint32_t* addr, uint32_t value) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(addr), "r"(value) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(uint32_t const* addr) {
    uint32_t value;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(value) : "l"(addr) : "memory");
    return value;
}
__device__ __forceinline__ void fence_sys() {
    asm volatile("fence.acq_rel.sys;" ::: "memory");
}
// Spin until *addr reaches `target` (monotonic epochs, wrap-safe signed difference). A peer may legitimately be late by a long
// time (rank 0 evaluating or writing a checkpoint, a first-use build, CUDA-graph capture): the bound is wall-clock
// (%globaltimer), generous (default 120 s) and configurable per library through `set_flag_timeout` (AGB_FLAG_TIMEOUT_S);
// 0 = wait forever. Expiry is reported and the kernel trapped: a dead peer must not hang the whole box silently.
static __device__ unsigned long long g_flag_timeout_ns = 120ull * 1000000000ull;
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void wait_flag_sys(uint32_t const* addr, uint32_t target) {
    if (static_cast<int32_t>(ld_acquire_sys(addr) - target) >= 0)
        return;
    unsigned long long const start = globaltimer_ns(), limit = g_flag_timeout_ns;
    unsigned spins = 0;
    while (static_cast<int32_t>(ld_acquire_sys(addr) - target) < 0) {
        __nanosleep(spins < 64 ? 32 : 256);
        if ((++spins & 0x3ffu) == 0 && limit != 0 && globaltimer_ns() - start > limit) {
            printf("[agb] wait_flag_sys: no signal after %llu s: flag %p = %u, expected >= %u (block %d) - a peer rank died or never launched\n",
                   limit / 1000000000ull, (void const*) addr, ld_acquire_sys(addr), target, (int) blockIdx.x);
            __trap();
        }
    }
}
inline int set_flag_timeout(double seconds) {
    unsigned long long const ns = seconds <= 0. ? 0ull : static_cast<unsigned long long>(seconds * 1e9);
    AGB_CUDA_OK(cudaMemcpyToSymbol(g_flag_timeout_ns, &ns, sizeof(ns)));
    return 0;
}

// ---- streaming 128-bit accesses ------------------------------------------ //
// Peer gradient tiles are read exactly once: do not allocate them in L1.
__device__ __forceinline__ float4 ld_stream_f4(float const* addr) {
    float4 v;
    asm volatile("ld.global.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(addr));
    return v;
}
__device__ __forceinline__ float4 ld_volatile_f4(float const* addr) {
    float4 v;
    asm volatile("ld.volatile.global.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(addr));
    return v;
}
__device__ __forceinline__ float ld_volatile_f(float const* addr) {
    float v;
    asm volatile("ld.volatile.global.f32 %0, [%1];" : "=f"(v) : "l"(addr));
    return v;
}
__device__ __forceinline__ void st_stream_f4(float* addr, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ---- NVLS (multicast-mapped memory) -------------------------------------- //
// One store lands in every GPU bound to the multicast object.
__device__ __forceinline__ void multimem_st_f4(float* mc_addr, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(mc_addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// In-switch reduction: returns the sum over all bound GPUs of the 4 floats at mc_addr.
__device__ __forceinline__ float4 multimem_ld_reduce_add_f4(float const* mc_addr) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc_addr) : "memory");
    return v;
}

// ---- reductions ------------------------------------------------------------ //
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int offset = 16; offset > 0; offset >>= 1)
        v += __shfl_xor_sync(0xffffffffu, v, offset);
    return v;
}

// max / min that return NaN when either input is NaN (fmaxf / fminf return the other operand): a ReLU or clamp built on them
// lets a NaN activation reach the loss instead of turning it into a number.
__device__ __forceinline__ float max_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}
__device__ __forceinline__ float min_nan(float a, float b) {
    float r;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

__device__ __forceinline__ bool is_finite(float v) {
    return (__float_as_uint(v) & 0x7f800000u) != 0x7f800000u;
}

// Total order used by every aggregation rule: finite ascending, then non-finite, ties -> lower index.
__device__ __forceinline__ bool before(float a, int ia, float b, int ib) {
    bool fa = is_finite(a), fb = is_finite(b);
    if (fa != fb)
        return fa;
    if (fa && a != b)
        return a < b;
    return ia < ib;
}

// ---- backdoor trigger (`attacks/data.py`, `ops.nn.stamp_trigger`) ----------- //
// A batch of consecutive per-worker batches of `rows` images: image b is poisoned iff b / rows >= first and b % rows < q. A poisoned
// H x W network input carries an s x s checkerboard, 255 where i + j is even and 0 elsewhere on every channel, at the bottom right one
// pixel from the edges (top-left corner (H - 1 - s, W - 1 - s)), in the raw [0, 255] domain. s = 0 stamps nothing.
struct Trigger {
    int rows, first, q, s;
};
__device__ __forceinline__ bool trigger_poisoned(Trigger const& t, long long image) {
    return t.s > 0 && image / t.rows >= t.first && image % t.rows < t.q;
}
// The trigger's value at pixel (y, x) of a poisoned H x W image, or -1 outside the trigger.
__device__ __forceinline__ float trigger_value(Trigger const& t, int H, int W, int y, int x) {
    int const i = y - (H - 1 - t.s), j = x - (W - 1 - t.s);
    return i >= 0 && i < t.s && j >= 0 && j < t.s ? ((i + j) & 1 ? 0.f : 255.f) : -1.f;
}
// Host-side check of a descriptor for a batch of N images of H x W (s = 0: nothing to check).
inline bool trigger_valid(Trigger const& t, long long N, int H, int W) {
    return t.s == 0 || (t.rows >= 1 && N % t.rows == 0 && t.first >= 0 && t.q >= 0 && t.q <= t.rows && t.s + 1 <= H && t.s + 1 <= W);
}

} // namespace agb
