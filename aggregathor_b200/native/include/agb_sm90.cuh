// Hopper (sm_90a) primitives used by the GEMM / implicit-GEMM kernels: mbarrier, TMA (cp.async.bulk.tensor),
// wgmma (warpgroup MMA from shared-memory descriptors), warp-level TF32 mma.sync and the wgmma shared-memory
// descriptor. Inline PTX only; bit layouts follow the PTX ISA (matrix descriptor format of the wgmma section).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <unordered_map>

namespace agb {
namespace sm90 {

__device__ __forceinline__ uint32_t smem_u32(void const* ptr) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(ptr));
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---- mbarrier -------------------------------------------------------------- //
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t done;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return done != 0;
}
// Bounded wait (2 s of wall clock): a pipeline bug becomes a trap with a message instead of a hung GPU.
__device__ __forceinline__ uint64_t global_timer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag) {
    if (mbar_try_wait(bar, parity))
        return;
    uint64_t const start = global_timer_ns();
    while (!mbar_try_wait(bar, parity)) {
        if (global_timer_ns() - start > 2000000000ull) {
            printf("[agb] mbarrier timeout tag %d block (%d,%d,%d) thread %d parity %u\n", tag, (int) blockIdx.x, (int) blockIdx.y, (int) blockIdx.z, (int) threadIdx.x, parity);
            __trap();
        }
    }
}

// ---- TMA -------------------------------------------------------------------- //
__device__ __forceinline__ void tma_prefetch_desc(CUtensorMap const* map) {
    asm volatile("prefetch.tensormap [%0];" :: "l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, CUtensorMap const* map, uint64_t* bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, CUtensorMap const* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, CUtensorMap const* map, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 :: "r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}

// Shared -> global tensor stores and fp32 add-reductions (bulk async-group completion, tracked per issuing thread). The box lands
// where the map says; coordinates outside the map's extents are clipped, so partial tiles need no bounds tests.
template<bool kReduce> __device__ __forceinline__ void tma_store_4d(CUtensorMap const* map, void const* src, int c0, int c1, int c2, int c3) {
    if constexpr (kReduce)
        asm volatile("cp.reduce.async.bulk.tensor.4d.global.shared::cta.add.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                     :: "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
    else
        asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                     :: "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
// All but the `kPending` most recent bulk groups of this thread have finished READING shared memory (their buffers may be rewritten).
template<int kPending> __device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" :: "n"(kPending) : "memory");
}
// Every bulk group of this thread is complete, its global writes included.
__device__ __forceinline__ void bulk_wait_all() {
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
// Generic-proxy writes to shared memory become visible to the async proxy (TMA) of this CTA.
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- wgmma (warpgroup MMA: 4 consecutive warps, the first one's index a multiple of 4) ---------------- //
// Operands from shared-memory descriptors, fp32 accumulators in registers. Fragment of an m64nN accumulator held by thread
// t of the warpgroup: d[4 j + 2 i + c] = D[16 (t / 32) + (t % 32) / 4 + 8 i][8 j + 2 (t % 4) + c]  (j < N / 8, i, c in {0, 1}).
__device__ __forceinline__ void wgmma_fence() {
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template<int kPending> __device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(kPending) : "memory");
}
// Keeps the compiler from moving accesses of the accumulators across the asynchronous MMAs that own them.
template<int kRegs> __device__ __forceinline__ void fence_regs(float (&d)[kRegs]) {
#pragma unroll
    for (int i = 0; i < kRegs; ++i)
        asm volatile("" : "+f"(d[i]) :: "memory");
}
// D (+)= A * B, bf16 operands, m64 x N x k16. TA / TB = 1: the operand is MN-major in shared memory (K rows of MN-contiguous
// elements), 0: K-major. scale-d is always 1: callers zero their accumulators.
template<int TA, int TB> __device__ __forceinline__ void wgmma_bf16(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b), "r"(1), "n"(TA), "n"(TB));
}

template<int TA, int TB> __device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(desc_a), "l"(desc_b), "r"(1), "n"(TA), "n"(TB));
}

template<int TA, int TB> __device__ __forceinline__ void wgmma_bf16(float (&d)[128], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, %131, %132;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(desc_a), "l"(desc_b), "r"(1), "n"(TA), "n"(TB));
}


// Warp-level m16n8k8 TF32 MMA (fp32 accumulation). wgmma reads 32-bit operands K-major only; the TF32 weight and data gradients
// need MN-major operands, so the TF32 kernels load fragments from the swizzled stage themselves and issue this instead.
__device__ __forceinline__ void mma_tf32_16x8x8(float* d, uint32_t const (&a)[4], uint32_t const (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// ---- descriptors ---------------------------------------------------------------- //
// wgmma shared-memory matrix descriptor, 128-byte swizzle (the layout TMA writes with CU_TENSOR_MAP_SWIZZLE_128B into 1024-byte
// aligned tiles of 128-byte rows):
//   K-major  (rows = M/N index, 64 K-elements = 128 B per row): SBO = 1024 B (8 rows), LBO unused (1).
//   MN-major (rows = K index, 64 MN-elements = 128 B per row): SBO = 1024 B (8 k-rows), LBO = byte distance
//            between consecutive 64-element MN chunks.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t desc = 0;
    desc |= static_cast<uint64_t>((smem_addr & 0x3ffff) >> 4);            // start address, bits [0,14)
    desc |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fff) << 16;       // leading byte offset, bits [16,30)
    desc |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3fff) << 32;       // stride byte offset, bits [32,46)
    desc |= static_cast<uint64_t>(1) << 62;                               // layout: SWIZZLE_128B
    return desc;
}
// Byte offset of element (row, col) of 32-bit elements in a tile of 128-byte rows written with the 128-byte swizzle:
// 16-byte piece p of row r sits at piece p ^ (r % 8).
__device__ __forceinline__ uint32_t swizzled_offset32(int row, int col) {
    return static_cast<uint32_t>(row * 128 + ((((col >> 2) ^ row) & 7) << 4) + ((col & 3) << 2));
}

} // namespace sm90

// ---- host: tensor-map creation through the driver entry point (no link-time libcuda dependency) ---- //
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, cuuint64_t const*, cuuint64_t const*, cuuint32_t const*,
                                  cuuint32_t const*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* ptr = nullptr;
        cudaDriverEntryPointQueryResult status;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &status) != cudaSuccess || status != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

// Tensor maps are pure functions of (base, dims, strides, box, element strides): the same layer is launched with the same arguments every
// step, so encoded descriptors are memoised (cuTensorMapEncodeTiled is a driver call of a few microseconds; an eager step — evaluation,
// tracing, experiments that opt out of CUDA graphs — made ~300 of them).
struct TmapKey {
    void const* base;
    uint64_t dims[4], strides[3];
    uint32_t box[4], elem[4], rank, dtype, swizzle, pad;
    bool operator==(TmapKey const& o) const { return std::memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
    size_t operator()(TmapKey const& k) const {
        uint64_t h = 1469598103934665603ull;
        unsigned char const* p = reinterpret_cast<unsigned char const*>(&k);
        for (size_t i = 0; i < sizeof(TmapKey); ++i)
            h = (h ^ p[i]) * 1099511628211ull;
        return static_cast<size_t>(h);
    }
};
inline int encode_cached(CUtensorMap* map, CUtensorMapDataType dtype, uint32_t rank, void const* base, cuuint64_t const* dims, cuuint64_t const* strides, cuuint32_t const* box,
                         cuuint32_t const* elem, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
    static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
    static std::mutex mutex;
    TmapKey key;
    std::memset(&key, 0, sizeof(key));
    key.base = base; key.rank = rank; key.dtype = static_cast<uint32_t>(dtype); key.swizzle = static_cast<uint32_t>(swizzle);
    for (uint32_t i = 0; i < rank; ++i) {
        key.dims[i] = dims[i]; key.box[i] = box[i]; key.elem[i] = elem[i];
        if (i + 1 < rank)
            key.strides[i] = strides[i];
    }
    {
        std::lock_guard<std::mutex> guard(mutex);
        auto it = cache.find(key);
        if (it != cache.end()) {
            *map = it->second;
            return 0;
        }
    }
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn)
        return 201;
    CUresult res = fn(map, dtype, rank, const_cast<void*>(base), dims, strides, box, elem, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                      CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (res != CUDA_SUCCESS) {
        std::fprintf(stderr, "[agb] cuTensorMapEncodeTiled(rank %u) failed (%d): base %p dims %llu %llu %llu %llu box %u %u %u %u\n", rank, (int) res, base, (unsigned long long) dims[0],
                     (unsigned long long) (rank > 1 ? dims[1] : 0), (unsigned long long) (rank > 2 ? dims[2] : 0), (unsigned long long) (rank > 3 ? dims[3] : 0), box[0],
                     rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0);
        return 202;
    }
    std::lock_guard<std::mutex> guard(mutex);
    if (cache.size() > 16384)   // addresses change when buffers are re-allocated: keep the table bounded
        cache.clear();
    cache.emplace(key, *map);
    return 0;
}

// 2-D tensor map (bf16 or fp32 elements): `inner` contiguous elements per row, `rows` rows of `row_stride` elements, box = box_inner x box_rows,
// 128-byte swizzle.
inline int make_tmap_2d(CUtensorMap* map, void const* base, uint64_t inner, uint64_t rows, uint64_t row_stride, uint32_t box_inner, uint32_t box_rows, int elem_bytes) {
    cuuint64_t dims[2] = {inner, rows};
    cuuint64_t strides[1] = {row_stride * elem_bytes};
    cuuint32_t box[2] = {box_inner, box_rows};
    cuuint32_t elem[2] = {1, 1};
    return encode_cached(map, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, strides, box, elem);
}
inline int make_tmap_2d_bf16(CUtensorMap* map, void const* base, uint64_t inner, uint64_t rows, uint64_t row_stride, uint32_t box_inner, uint32_t box_rows) {
    return make_tmap_2d(map, base, inner, rows, row_stride, box_inner, box_rows, 2);
}

// 3-D bf16 tensor map over a row-major [groups][rows][inner] view (row stride `row_stride`, group stride `rows * row_stride`):
// boxes never straddle a group, rows past the end of a group are zero-filled (grouped weight-gradient GEMMs).
inline int make_tmap_3d(CUtensorMap* map, void const* base, uint64_t inner, uint64_t rows, uint64_t groups, uint64_t row_stride, uint32_t box_inner, uint32_t box_rows, int elem_bytes) {
    cuuint64_t dims[3] = {inner, rows, groups};
    cuuint64_t strides[2] = {row_stride * elem_bytes, rows * row_stride * elem_bytes};
    cuuint32_t box[3] = {box_inner, box_rows, 1};
    cuuint32_t elem[3] = {1, 1, 1};
    return encode_cached(map, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, base, dims, strides, box, elem);
}
inline int make_tmap_3d_bf16(CUtensorMap* map, void const* base, uint64_t inner, uint64_t rows, uint64_t groups, uint64_t row_stride, uint32_t box_inner, uint32_t box_rows) {
    return make_tmap_3d(map, base, inner, rows, groups, row_stride, box_inner, box_rows, 2);
}

} // namespace agb
