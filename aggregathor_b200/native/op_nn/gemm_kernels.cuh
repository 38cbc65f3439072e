#pragma once
// GEMM on the Hopper tensor cores: C[M,N] = op(A) * op(B) with fp32 accumulation in registers.
//
// One kernel family covers the three products a layer needs (SURVEY §7.3 item 7):
//   forward   Y  = X  * W^T      A K-major   ([M,K] rows)      B K-major  ([N,K] rows)
//   dgrad     dX = dY * W        A K-major   ([M,K] rows)      B MN-major ([K,N] rows, N contiguous)
//   wgrad     dW = dY^T * X      A MN-major  ([K,M] rows)      B MN-major ([K,N] rows)   (+ split-K)
// so activations and weights are consumed in the layout they already have: no transposes.
//
// Structure: persistent, one CTA per SM looping over (128 x BN output tile, k-split) work items; 384 threads:
//   warps 0-7   two consumer warpgroups, each owning 64 rows of the tile and all BN columns. bf16: wgmma m64 x BN x k16 straight
//               from the swizzled ring (shared-memory descriptors; MN-major operands through the transpose bits). TF32: wgmma reads
//               32-bit operands K-major only, so every warp issues m16n8k8 mma.sync on fragments it loads from the ring (same
//               accumulator layout). The epilogue (+ bias, ReLU, convert) goes through per-warp shared buffers and TMA stores, or
//               fp32 TMA add-reductions for split-K (epilogue_staged); what no tensor map can address is stored from registers.
//   warps 8-11  producer warpgroup: one lane issues the cp.async.bulk.tensor tiles (128B swizzle) into a kStages-deep smem ring,
//               completion signalled on `full` mbarriers (complete_tx::bytes); every consumer warp arrives on `empty` once its MMAs
//               have read a slot. The producer hands its registers to the consumers (setmaxnreg): a 64 x 256 fp32 accumulator is
//               128 registers per thread.
// The ring runs continuously across work items: the producer fetches the next item's operands during the consumers' epilogue.
//
// Each k-split handles a contiguous range of 64-wide (bf16) / 32-wide (TF32) K blocks and, when splits > 1, accumulates with fp32
// atomics into a pre-zeroed C.

#include <cuda_bf16.h>
#include <cstdlib>

#include <agb_device.cuh>
#include <agb_sm90.cuh>

using namespace agb;
using namespace agb::sm90;

// AGB_GEMM_EPILOGUE / agb_gemm_set_epilogue (gemm.cu): 1 = staged epilogue where TMA can address the output (default), 0 = register
// stores everywhere.
extern "C" int agb_gemm_epilogue_staged();

namespace {

constexpr int kBM = 128;
constexpr int kBK = 64;               // bf16: K elements per stage = one 128-byte swizzle row
constexpr int kConsumerWarps = 8;     // two warpgroups
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreads = kConsumerWarps * 32 + 128;

// Operand element types. A pipeline stage is always 128 bytes of K per row (one swizzle row):
//   bf16  64 K-elements per stage, MN-major chunks of 64 elements
//   tf32  32 K-elements per stage, MN-major chunks of 32 elements - fp32 operands straight from memory (the tensor core reads
//         the top 19 bits): the parity-precision path for the fp32 reference (`graph.py:267-273`)
struct ElemBF16 {
    using type = __nv_bfloat16;
    static constexpr int kBytes = 2, kBK = 64, kChunk = 64;
    static constexpr bool kTf32 = false;
};
struct ElemTF32 {
    using type = float;
    static constexpr int kBytes = 4, kBK = 32, kChunk = 32;
    static constexpr bool kTf32 = true;
};

// Staged epilogue: every consumer warp owns two 16-row x 128-byte pieces of shared memory (64 bf16 or 32 fp32 columns of its slab).
constexpr uint32_t kPieceBytes = 16 * 128;
constexpr uint32_t kStagingBytes = kConsumerWarps * 2 * kPieceBytes;   // 32 KB

template<int BN> struct Config {
    static constexpr uint32_t kABytes = kBM * 128;   // 128 rows x 128 bytes of K (either element type)
    static constexpr uint32_t kBBytes = BN * 128;
    static constexpr uint32_t kStageBytes = kABytes + kBBytes;
    static constexpr int kStages = (192 * 1024) / kStageBytes;   // 8 / 6 / 4 stages for BN = 64 / 128 / 256: 192 KB of the 227 KB
    static constexpr uint32_t kRingBytes = kStages * kStageBytes;   // staging buffers follow the ring (1024-byte aligned), then the barriers
    static constexpr uint32_t kSmemBytes = kRingBytes + kStagingBytes + 1024 /* alignment slack */ + 256 /* barriers */;
};

// Register split between the producer warpgroup and the two consumer warpgroups (3 x 128 threads, 64 K registers).
__device__ __forceinline__ void producer_registers() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
}
__device__ __forceinline__ void consumer_registers() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
}

struct GemmParams {
    int M, N, K;            // logical problem
    long long ldc;          // row stride of C (elements)
    void* C;
    float const* bias;      // per-N fp32 bias or null
    int relu;
    int out_fp32;           // C element type: 1 = float, 0 = bf16
    int atomic;             // accumulate with red.add.f32 (split-K); requires out_fp32
    int kblocks_per_split;
    int groups;              // grouped weight gradients: independent K ranges (one per logical worker) ...
    long long c_group_stride; // ... each accumulating into C + group * c_group_stride
    int staged;              // 1: epilogue through shared memory and TMA stores / reductions (the output tensor map), 0: from registers
    void const* addend;      // null, or a tensor laid out like C added to the rounded product: C = round(round(acc) + addend) (no split-K)
};

// 4-D tensor map over the epilogue output, 128-byte swizzle, box = one warp's piece: 128 bytes of columns x `box` (16 rows in all)
// along dims 1..3. Returns 0 (and leaves the register epilogue in charge) when TMA cannot address C: base or a stride not a
// multiple of 16 bytes.
inline bool make_tmap_out(CUtensorMap* map, void const* base, bool fp32, uint64_t const (&dims)[4], uint64_t const (&strides)[3], uint32_t const (&box)[3]) {
    uint64_t const e = fp32 ? 4 : 2;
    if (reinterpret_cast<uintptr_t>(base) & 15)
        return false;
    cuuint64_t d[4], s[3];
    for (int i = 0; i < 4; ++i)
        d[i] = dims[i];
    for (int i = 0; i < 3; ++i) {
        s[i] = strides[i] * e;
        if ((s[i] & 15) || s[i] == 0 || s[i] >= (1ull << 40))
            return false;
    }
    cuuint32_t b[4] = {static_cast<cuuint32_t>(128 / e), box[0], box[1], box[2]};
    cuuint32_t elem[4] = {1, 1, 1, 1};
    return encode_cached(map, fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, d, s, b, elem) == 0;
}

// Staged epilogue of one warp's 16 x BN slab: for every 128-byte column piece, the same bias / ReLU / rounding as epilogue_slab into
// a 128B-swizzled shared buffer (conflict-free for bf16), then one lane issues a TMA store (or fp32 add-reduction for split-K) of the
// 16-row box whose coordinates `coords(col, c)` gives. The two buffers of a warp alternate; a buffer is rewritten only once the bulk
// group that read it has finished reading (`issued` counts this warp's pieces across work items). Rows past M and columns past N
// are clipped by the map.
// kAdd: the addend's box (same geometry, map `tmap_d`) is first brought into the buffer by a TMA load on the warp's mbarrier `dbar`
// (one load per piece, so its phase is `issued & 1`); every lane reads its addend pair from the very bytes it then overwrites.
template<int BN, bool kFp32, bool kReduce, bool kAdd, typename CoordFn>
__device__ __forceinline__ void epilogue_staged(GemmParams const& p, CUtensorMap const* tmap_c, float (&acc)[BN / 2], uint8_t* staging, uint32_t& issued, int n0, CoordFn const& coords,
                                                CUtensorMap const* tmap_d, uint64_t* dbar) {
    constexpr int kCols = kFp32 ? 32 : 64;
    int const lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int q = 0; q < BN / kCols; ++q) {
        int const col0 = n0 + q * kCols;
        if (col0 >= p.N)
            break;
        uint8_t* buf = staging + (issued & 1) * kPieceBytes;
        if (lane == 0) {
            bulk_wait_read<1>();
            if constexpr (kAdd) {
                int c[4];
                coords(col0, c);
                mbar_expect_tx(dbar, kPieceBytes);
                tma_load_4d(buf, tmap_d, dbar, c[0], c[1], c[2], c[3]);
            }
        }
        __syncwarp();
        if constexpr (kAdd) {   // a plain spin: the bounded wait's timer and message cost the 256-wide tile registers it has none to spare of
            while (!mbar_try_wait(dbar, issued & 1)) {
            }
        }
#pragma unroll
        for (int jj = 0; jj < kCols / 8; ++jj) {
            int const j = q * (kCols / 8) + jj;
            int const col = col0 + 8 * jj + 2 * t;
            float b0 = 0.f, b1 = 0.f;
            if (p.bias) {
                if (col < p.N)
                    b0 = __ldg(p.bias + col);
                if (col + 1 < p.N)
                    b1 = __ldg(p.bias + col + 1);
            }
            uint32_t const byte = (8 * jj + 2 * t) * (kFp32 ? 4 : 2);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                int const row = g + 8 * i;
                float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
                if (p.bias) {
                    v0 += b0;
                    v1 += b1;
                }
                if (p.relu) {
                    v0 = max_nan(v0, 0.f);
                    v1 = max_nan(v1, 0.f);
                }
                uint8_t* dst = buf + row * 128 + ((((byte >> 4) ^ row) & 7) << 4) + (byte & 15);
                if constexpr (kFp32) {
                    if constexpr (kAdd) {
                        float2 const d = *reinterpret_cast<float2 const*>(dst);
                        v0 += d.x;
                        v1 += d.y;
                    }
                    *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
                } else {
                    if constexpr (kAdd) {   // the product is rounded to bf16 first, as a separate add of two bf16 tensors sees it
                        float2 const d = __bfloat1622float2(*reinterpret_cast<__nv_bfloat162 const*>(dst));
                        float2 const r = __bfloat1622float2(__floats2bfloat162_rn(v0, v1));
                        v0 = r.x + d.x;
                        v1 = r.y + d.y;
                    }
                    *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v0, v1);
                }
            }
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (lane == 0) {
            int c[4];
            coords(col0, c);
            tma_store_4d<kReduce>(tmap_c, buf, c[0], c[1], c[2], c[3]);
            bulk_commit();
        }
        ++issued;
    }
}

// kMayAdd: the caller passes the addend's map and the warp's mbarrier (plain GEMMs); the convolution kernels never take an addend.
template<int BN, bool kMayAdd = false, typename CoordFn>
__device__ __forceinline__ void epilogue_staged(GemmParams const& p, CUtensorMap const* tmap_c, float (&acc)[BN / 2], uint8_t* staging, uint32_t& issued, int n0, CoordFn const& coords,
                                                CUtensorMap const* tmap_d = nullptr, uint64_t* dbar = nullptr) {
    if (kMayAdd && p.addend) {   // never with split-K (rejected by the entry points)
        if (!p.out_fp32)
            epilogue_staged<BN, false, false, kMayAdd>(p, tmap_c, acc, staging, issued, n0, coords, tmap_d, dbar);
        else
            epilogue_staged<BN, true, false, kMayAdd>(p, tmap_c, acc, staging, issued, n0, coords, tmap_d, dbar);
    } else if (!p.out_fp32) {
        epilogue_staged<BN, false, false, false>(p, tmap_c, acc, staging, issued, n0, coords, tmap_d, dbar);
    } else if (p.atomic) {
        epilogue_staged<BN, true, true, false>(p, tmap_c, acc, staging, issued, n0, coords, tmap_d, dbar);
    } else {
        epilogue_staged<BN, true, false, false>(p, tmap_c, acc, staging, issued, n0, coords, tmap_d, dbar);
    }
}

// Epilogue of one warp's 16 x BN slab of the accumulator (fragment layout: agb_sm90.cuh). `row_at(r, valid, offset)` tells whether
// tile row r is a real output row and the element offset of that row in C (lets implicit-GEMM convolutions scatter pixel-box rows to
// NHWC addresses). Pairs of adjacent columns go out as one 8-byte (fp32, also for the split-K reductions) or 4-byte (bf16) access.
template<int BN, bool kMayAdd = false, typename RowFn>
__device__ __forceinline__ void epilogue_slab(GemmParams const& p, float (&acc)[BN / 2], int slab_row, int n0, RowFn const& row_at) {
    int const lane = threadIdx.x & 31;
    uintptr_t const align = p.out_fp32 ? 7 : 3;
    bool const pairs = (p.ldc & 1) == 0 && (p.c_group_stride & 1) == 0 && (reinterpret_cast<uintptr_t>(p.C) & align) == 0
                       && (!kMayAdd || (reinterpret_cast<uintptr_t>(p.addend) & align) == 0);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        bool valid;
        long long offset;
        row_at(slab_row + (lane >> 2) + 8 * i, valid, offset);
        if (!valid)
            continue;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
            int const col = n0 + 8 * j + 2 * (lane & 3);
            if (col >= p.N)
                break;
            bool const both = col + 1 < p.N;
            float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
            if (p.bias) {
                v0 += __ldg(p.bias + col);
                if (both)
                    v1 += __ldg(p.bias + col + 1);
            }
            if (p.relu) {
                v0 = max_nan(v0, 0.f);
                v1 = max_nan(v1, 0.f);
            }
            if (p.out_fp32) {
                float* dst = static_cast<float*>(p.C) + offset + col;
                if (kMayAdd && p.addend) {   // same order as epilogue_staged: the bias and ReLU first, then the addend
                    float const* src = static_cast<float const*>(p.addend) + offset + col;
                    v0 += src[0];
                    if (both)
                        v1 += src[1];
                }
                if (p.atomic) {
                    if (both && pairs) {
                        atomicAdd(reinterpret_cast<float2*>(dst), make_float2(v0, v1));   // vector reduction (sm_90+)
                    } else {
                        atomicAdd(dst, v0);
                        if (both)
                            atomicAdd(dst + 1, v1);
                    }
                } else if (both && pairs) {
                    *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
                } else {
                    dst[0] = v0;
                    if (both)
                        dst[1] = v1;
                }
            } else {
                __nv_bfloat16* dst = static_cast<__nv_bfloat16*>(p.C) + offset + col;
                if (kMayAdd && p.addend) {   // round the product to bf16 first, as epilogue_staged does
                    __nv_bfloat16 const* src = static_cast<__nv_bfloat16 const*>(p.addend) + offset + col;
                    v0 = __bfloat162float(__float2bfloat16(v0)) + __bfloat162float(src[0]);
                    if (both)
                        v1 = __bfloat162float(__float2bfloat16(v1)) + __bfloat162float(src[1]);
                }
                if (both && pairs) {
                    *reinterpret_cast<__nv_bfloat162*>(dst) = __floats2bfloat162_rn(v0, v1);
                } else {
                    dst[0] = __float2bfloat16(v0);
                    if (both)
                        dst[1] = __float2bfloat16(v1);
                }
            }
        }
    }
}

// Main loop of one work item for consumer warp `warp` (0..7): `nkb` ring slots starting at `ring`; the accumulator covers tile rows
// 16 warp .. 16 warp + 15 and all BN columns.
template<int BN, bool A_MN, bool B_MN, typename E>
__device__ __forceinline__ void mainloop(uint8_t* smem, uint64_t* full, uint64_t* empty, uint32_t& ring, int nkb, int warp, float (&acc)[BN / 2]) {
    using Cfg = Config<BN>;
    constexpr int kStages = Cfg::kStages;
    constexpr uint32_t kChunkBytes = E::kBK * 128;   // one MN-major chunk: kBK k-rows of 128 bytes
    int const lane = threadIdx.x & 31;
#pragma unroll
    for (int r = 0; r < BN / 2; ++r)
        acc[r] = 0.f;
    if constexpr (!E::kTf32) {
        int const wg = warp >> 2;
        int prev = -1;
        for (int i = 0; i < nkb; ++i, ++ring) {
            int const s = ring % kStages;
            mbar_wait(full + s, (ring / kStages) & 1, 2);
            // this warpgroup's 64 rows of A: 64 K-major rows of 128 B, or MN-major chunk `wg` (64 M-elements): both 8 KB further
            uint32_t const a_addr = smem_u32(smem + s * Cfg::kStageBytes) + wg * 64 * 128;
            uint32_t const b_addr = smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes);
            fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int kk = 0; kk < E::kBK / 16; ++kk) {
                // K-major: one instruction's K (16 elements) = 32 B further inside the swizzled row; MN-major: 16 k-rows = 2 KB further
                uint64_t const da = A_MN ? gmma_desc(a_addr + kk * 16 * 128, kChunkBytes, 1024) : gmma_desc(a_addr + kk * 32, 16, 1024);
                uint64_t const db = B_MN ? gmma_desc(b_addr + kk * 16 * 128, kChunkBytes, 1024) : gmma_desc(b_addr + kk * 32, 16, 1024);
                wgmma_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db);
            }
            wgmma_commit();
            fence_regs(acc);
            wgmma_wait<1>();   // the previous slot's MMAs are complete: it may be refilled
            if (prev >= 0 && lane == 0)
                mbar_arrive(empty + prev);
            prev = s;
        }
        wgmma_wait<0>();
        fence_regs(acc);
        if (prev >= 0 && lane == 0)
            mbar_arrive(empty + prev);
    } else {
        // element (mn, k) of a staged operand: K-major rows of 32 fp32, or MN-major chunks of 32 elements x kBK k-rows
        auto offset = [](bool mn_major, int mn, int k) {
            return mn_major ? (mn >> 5) * kChunkBytes + swizzled_offset32(k, mn & 31) : swizzled_offset32(mn, k);
        };
        int const g = lane >> 2, t = lane & 3, row0 = 16 * warp;
        for (int i = 0; i < nkb; ++i, ++ring) {
            int const s = ring % kStages;
            mbar_wait(full + s, (ring / kStages) & 1, 2);
            uint8_t const* a = smem + s * Cfg::kStageBytes;
            uint8_t const* b = a + Cfg::kABytes;
#pragma unroll
            for (int k8 = 0; k8 < E::kBK; k8 += 8) {
                uint32_t af[4];
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    af[q] = *reinterpret_cast<uint32_t const*>(a + offset(A_MN, row0 + g + 8 * (q & 1), k8 + t + 4 * (q >> 1)));
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    uint32_t bf[2];
                    bf[0] = *reinterpret_cast<uint32_t const*>(b + offset(B_MN, 8 * j + g, k8 + t));
                    bf[1] = *reinterpret_cast<uint32_t const*>(b + offset(B_MN, 8 * j + g, k8 + t + 4));
                    mma_tf32_16x8x8(acc + 4 * j, af, bf);
                }
            }
            __syncwarp();
            if (lane == 0)
                mbar_arrive(empty + s);
        }
    }
}

// Loads of one pipeline stage (A and B tiles of the k-block starting at element `k`).
template<int BN, bool A_MN, bool B_MN, typename E = ElemBF16>
__device__ __forceinline__ void produce_stage(CUtensorMap const* tmap_a, CUtensorMap const* tmap_b, uint8_t* a_dst, uint64_t* bar, int m0, int n0, int k, int group = -1) {
    uint8_t* b_dst = a_dst + Config<BN>::kABytes;
    constexpr int kChunkBytes = E::kBK * 128;   // one MN-major chunk: kBK k-rows of 128 bytes
    mbar_expect_tx(bar, Config<BN>::kStageBytes);
    if (A_MN && B_MN && group >= 0) {   // grouped weight gradient: 3-D maps (inner, row in group, group)
#pragma unroll
        for (int c = 0; c < kBM / E::kChunk; ++c)
            tma_load_3d(a_dst + c * kChunkBytes, tmap_a, bar, m0 + c * E::kChunk, k, group);
#pragma unroll
        for (int c = 0; c < BN / E::kChunk; ++c)
            tma_load_3d(b_dst + c * kChunkBytes, tmap_b, bar, n0 + c * E::kChunk, k, group);
        return;
    }
    if (A_MN) { // rows = K index, kChunk M-elements per row; one box per chunk
#pragma unroll
        for (int c = 0; c < kBM / E::kChunk; ++c)
            tma_load_2d(a_dst + c * kChunkBytes, tmap_a, bar, m0 + c * E::kChunk, k);
    } else {
        tma_load_2d(a_dst, tmap_a, bar, k, m0);
    }
    if (B_MN) {
#pragma unroll
        for (int c = 0; c < BN / E::kChunk; ++c)
            tma_load_2d(b_dst + c * kChunkBytes, tmap_b, bar, n0 + c * E::kChunk, k);
    } else {
        tma_load_2d(b_dst, tmap_b, bar, k, n0);
    }
}

// The kernels that take an addend: data gradients (A K-major, B MN-major) with tiles up to 128 wide. At 256 the accumulator leaves the
// epilogue no registers for it (it would spill).
template<int BN, bool A_MN, bool B_MN>
constexpr bool kAddendKernel = !A_MN && B_MN && BN <= 128;

template<int BN, bool A_MN, bool B_MN, typename E = ElemBF16>
__global__ void __launch_bounds__(kThreads, 1) gemm_sm90_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                                                                 const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ CUtensorMap tmap_d, GemmParams const p,
                                                                 int m_tiles, int n_tiles, int splits) {
    using Cfg = Config<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::kRingBytes + kStagingBytes);
    uint64_t* empty = full + Cfg::kStages;
    uint64_t* addend_bar = empty + Cfg::kStages;   // one per consumer warp: its staged addend loads
    static_assert((2 * Cfg::kStages + kConsumerWarps) * 8 <= 256, "barriers outgrow their shared-memory slot");

    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int const total_kblocks = (p.K + E::kBK - 1) / E::kBK;
    int const total_items = m_tiles * n_tiles * splits * (p.groups > 1 ? p.groups : 1);

    if (warp == kProducerWarp && lane == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        for (int s = 0; s < Cfg::kStages; ++s) {
            mbar_init(full + s, 1);
            mbar_init(empty + s, kConsumerWarps);   // one arrival per consumer warp
        }
        for (int w = 0; w < kConsumerWarps; ++w)
            mbar_init(addend_bar + w, 1);
        mbar_fence_init();
    }
    if (p.staged && warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmap_c);
        if (p.addend)
            tma_prefetch_desc(&tmap_d);
    }
    __syncthreads();
    pdl_trigger();   // set-up done: the next kernel may start its own; ...
    pdl_wait();      // ... our inputs are complete only once the previous kernel has finished

    // item -> tile in grouped order (panels of 16 m-tiles, m fastest inside a panel, then n): the ~132 tiles in flight
    // cover a ~16 x 8 patch, so every A and B tile fetched from L2/HBM is reused by several CTAs of the same wave.
    constexpr int kGroupM = 16;
    int const items_per_group = m_tiles * n_tiles * splits;
    auto decode = [&](int item, int& m0, int& n0, int& kb_begin, int& nkb, int& group) {
        group = item / items_per_group;
        item -= group * items_per_group;
        int const tile = item % (m_tiles * n_tiles), split = item / (m_tiles * n_tiles);
        int const group_size = kGroupM * n_tiles;
        int const first_m = (tile / group_size) * kGroupM;
        int const gm = min(m_tiles - first_m, kGroupM);
        int const in_group = tile % group_size;
        m0 = (first_m + in_group % gm) * kBM;
        n0 = (in_group / gm) * BN;
        kb_begin = split * p.kblocks_per_split;
        int const kb_end = min(total_kblocks, kb_begin + p.kblocks_per_split);
        nkb = kb_end - kb_begin;
    };
    bool const grouped = p.groups > 1 || (A_MN && B_MN);   // TN products always use the 3-D maps

    if (warp >= kProducerWarp) {
        producer_registers();
        if (warp == kProducerWarp && lane == 0) {
            uint32_t it = 0;   // running k-block counter => ring slot and phase
            for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
                int m0, n0, kb_begin, nkb, group;
                decode(item, m0, n0, kb_begin, nkb, group);
                for (int i = 0; i < nkb; ++i, ++it) {
                    int const s = it % Cfg::kStages;
                    mbar_wait(empty + s, ((it / Cfg::kStages) & 1) ^ 1, 1);
                    produce_stage<BN, A_MN, B_MN, E>(&tmap_a, &tmap_b, smem + s * Cfg::kStageBytes, full + s, m0, n0, (kb_begin + i) * E::kBK, grouped ? group : -1);
                }
            }
        }
        return;
    }
    consumer_registers();
    uint32_t ring = 0, issued = 0;
    uint8_t* staging = smem + Cfg::kRingBytes + warp * 2 * kPieceBytes;
    float acc[BN / 2];
    for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
        int m0, n0, kb_begin, nkb, group;
        decode(item, m0, n0, kb_begin, nkb, group);
        mainloop<BN, A_MN, B_MN, E>(smem, full, empty, ring, nkb, warp, acc);
        if (p.staged) {   // output map (N, M, groups, 1)
            epilogue_staged<BN, kAddendKernel<BN, A_MN, B_MN>>(p, &tmap_c, acc, staging, issued, n0, [&](int col, int (&c)[4]) {
                c[0] = col; c[1] = m0 + 16 * warp; c[2] = group; c[3] = 0;
            }, &tmap_d, addend_bar + warp);
            continue;
        }
        epilogue_slab<BN, kAddendKernel<BN, A_MN, B_MN>>(p, acc, 16 * warp, n0, [&](int r, bool& valid, long long& offset) {
            int const row = m0 + r;
            valid = row < p.M;
            offset = static_cast<long long>(row) * p.ldc + group * p.c_group_stride;
        });
    }
    if (p.staged && lane == 0)
        bulk_wait_all();   // outputs complete (and staging read) before the CTA retires: PDL dependents and graph replays see them
}

// Output map of a plain / grouped product: C viewed as (N, M, groups, 1), box 128 bytes x 16 rows. False: TMA cannot address it.
inline bool gemm_out_map(CUtensorMap* map, GemmParams const& p) {
    uint64_t const groups = p.groups > 1 ? p.groups : 1;
    uint64_t const gstride = groups > 1 ? static_cast<uint64_t>(p.c_group_stride) : static_cast<uint64_t>(p.ldc) * p.M;
    uint64_t const dims[4] = {static_cast<uint64_t>(p.N), static_cast<uint64_t>(p.M), groups, 1};
    uint64_t const strides[3] = {static_cast<uint64_t>(p.ldc), gstride, gstride * groups};
    uint32_t const box[3] = {16, 1, 1};
    return p.ldc >= p.N && make_tmap_out(map, p.C, p.out_fp32, dims, strides, box);
}

static int g_persistent = -1;   // -1: read AGB_GEMM_PERSISTENT at first use

template<int BN, bool A_MN, bool B_MN, typename E = ElemBF16>
int launch_gemm(CUtensorMap const& ta, CUtensorMap const& tb, GemmParams const& params, int splits, cudaStream_t stream) {
    using Cfg = Config<BN>;
    if (g_persistent < 0) {
        char const* env = std::getenv("AGB_GEMM_PERSISTENT");
        g_persistent = env ? std::atoi(env) : 1;
    }
    if (params.addend && !kAddendKernel<BN, A_MN, B_MN>)
        return 207;
    GemmParams p = params;
    CUtensorMap tc, td;
    std::memset(&tc, 0, sizeof(tc));
    std::memset(&td, 0, sizeof(td));
    p.staged = agb_gemm_epilogue_staged() && gemm_out_map(&tc, p);
    if (p.staged && p.addend) {   // the addend's map: the output's geometry over the addend's base
        GemmParams q = p;
        q.C = const_cast<void*>(p.addend);
        p.staged = gemm_out_map(&td, q);
    }
    int const m_tiles = (p.M + kBM - 1) / kBM, n_tiles = (p.N + BN - 1) / BN;
    auto kernel = gemm_sm90_kernel<BN, A_MN, B_MN, E>;
    static bool configured = false;
    if (!configured) {
        AGB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        configured = true;
    }
    // persistent: one CTA per SM walks the work items; otherwise one CTA per item
    long long const items = static_cast<long long>(m_tiles) * n_tiles * splits * (p.groups > 1 ? p.groups : 1);
    long long const cap = g_persistent ? sm_count() : 0x7fffffffll;
    int const grid = static_cast<int>(items < cap ? items : cap);
    AGB_CUDA_OK(launch_pdl(kernel, dim3(grid), dim3(kThreads), Cfg::kSmemBytes, stream, ta, tb, tc, td, p, m_tiles, n_tiles, splits));
    return 0;
}

template<bool A_MN, bool B_MN>
int dispatch_bn(int bn, CUtensorMap const& ta, CUtensorMap const& tb, GemmParams const& p, int splits, cudaStream_t stream) {
    switch (bn) {
        case 64: return launch_gemm<64, A_MN, B_MN>(ta, tb, p, splits, stream);
        case 128: return launch_gemm<128, A_MN, B_MN>(ta, tb, p, splits, stream);
        case 256: return launch_gemm<256, A_MN, B_MN>(ta, tb, p, splits, stream);
    }
    return 203;
}

template<bool A_MN, bool B_MN>
int dispatch_bn_tf32(int bn, CUtensorMap const& ta, CUtensorMap const& tb, GemmParams const& p, int splits, cudaStream_t stream) {
    switch (bn) {
        case 64: return launch_gemm<64, A_MN, B_MN, ElemTF32>(ta, tb, p, splits, stream);
        case 128: return launch_gemm<128, A_MN, B_MN, ElemTF32>(ta, tb, p, splits, stream);
    }
    return 203;
}

} // namespace
