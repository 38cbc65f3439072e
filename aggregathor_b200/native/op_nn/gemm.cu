// C entry points of the Hopper GEMM (kernels: gemm_kernels.cuh).
#include "gemm_kernels.cuh"

extern "C" {

// 1 = 128 x 256 tiles for N >= 256 when the caller leaves the choice open (default), 0 = 128 x 128.
static int g_wide_tiles = 1;
int agb_gemm_set_wide_tiles(int enabled) {
    g_wide_tiles = enabled ? 1 : 0;
    return 0;
}

// Programmatic dependent launch between the kernels of this library (see agb_device.cuh).
int agb_nn_set_pdl(int enabled) {
    set_pdl(enabled);
    return 0;
}

// 1 = persistent kernel (default: one CTA per SM), 0 = one CTA per work item.
int agb_gemm_set_persistent(int enabled) {
    g_persistent = enabled ? 1 : 0;
    return 0;
}

// Epilogue of the GEMM and implicit-convolution kernels. 1 = staged (default): each warp converts its slab into shared memory and
// TMA stores (or, for split-K, add-reduces) it, wherever a tensor map can address the output; 0 = stores straight from registers.
// AGB_GEMM_EPILOGUE=staged|regs sets the initial value. Both give bit-identical outputs (split-K sums aside, whose order varies anyway).
static int g_epilogue = -1;
int agb_gemm_set_epilogue(int staged) {
    g_epilogue = staged ? 1 : 0;
    return 0;
}
int agb_gemm_epilogue_staged() {
    if (g_epilogue < 0) {
        char const* env = std::getenv("AGB_GEMM_EPILOGUE");
        bool const regs = env && std::strcmp(env, "regs") == 0;
        if (env && *env && !regs && std::strcmp(env, "staged") != 0)
            std::fprintf(stderr, "[agb] AGB_GEMM_EPILOGUE=%s: expected 'staged' or 'regs', using 'staged'\n", env);
        g_epilogue = regs ? 0 : 1;
    }
    return g_epilogue;
}

// C[M,N] = op(A) op(B)  (+bias, ReLU). bf16 operands:
//   a_mn == 0: A is [M rows][K] with row stride lda      a_mn == 1: A is [K rows][M] with row stride lda
//   b_mn == 0: B is [N rows][K] with row stride ldb      b_mn == 1: B is [K rows][N] with row stride ldb
// lda/ldb must be multiples of 8 elements, bases 16-byte aligned. splits > 1 => fp32 atomic accumulation into C
// (caller zeroes C). bn in {64, 128, 256} or 0 for an automatic choice.
int agb_gemm_bf16_grouped(void const* A, void const* B, void* C, int M, int N, int K, long long lda, long long ldb, long long ldc,
                          int a_mn, int b_mn, void const* bias, int relu, int out_fp32, int splits, int bn, int groups, long long c_group_stride, void const* addend,
                          void* stream);

int agb_gemm_bf16(void const* A, void const* B, void* C, int M, int N, int K, long long lda, long long ldb, long long ldc,
                  int a_mn, int b_mn, void const* bias, int relu, int out_fp32, int splits, int bn, void* stream) {
    return agb_gemm_bf16_grouped(A, B, C, M, N, K, lda, ldb, ldc, a_mn, b_mn, bias, relu, out_fp32, splits, bn, 1, 0, nullptr, stream);
}

// Grouped form (weight gradients of several logical workers in one launch): A and B hold `groups` consecutive blocks of K rows
// (a_mn = b_mn = 1 required when groups > 1), group g accumulates into C + g * c_group_stride. K is the per-group depth.
// `addend` (null = none): a tensor with C's element type and row stride; C = round(round(product) + addend), bit for bit what a
// separate element-wise add of the stored product and the addend gives (a data gradient summed with a shortcut gradient). Only
// for data gradients (a_mn = 0, b_mn = 1), without split-K, on tiles up to 128 wide (the automatic choice keeps to them).
int agb_gemm_bf16_grouped(void const* A, void const* B, void* C, int M, int N, int K, long long lda, long long ldb, long long ldc,
                          int a_mn, int b_mn, void const* bias, int relu, int out_fp32, int splits, int bn, int groups, long long c_group_stride, void const* addend,
                          void* stream) {
    if (M <= 0 || N <= 0 || K <= 0)
        return 0;
    if ((lda & 7) || (ldb & 7) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15))
        return 204;
    if (groups < 1)
        groups = 1;
    if (groups > 1 && !(a_mn && b_mn))
        return 206;
    if (splits < 1)
        splits = 1;
    if (splits > 1 && !out_fp32)
        return 205;
    if (splits > 1 && addend)
        return 207;
    if (bn == 0) {
        // 128 x 256 tiles halve the B re-reads per flop whenever there are enough of them to occupy the chip
        long long const wide_tiles = static_cast<long long>((M + kBM - 1) / kBM) * ((N + 255) / 256) * (groups > 1 ? groups : 1) * (splits > 1 ? splits : 1);
        bn = N <= 64 ? 64 : (N >= 256 && g_wide_tiles && wide_tiles >= 96 && !addend ? 256 : 128);
    }
    int const total_kblocks = (K + kBK - 1) / kBK;
    if (splits > total_kblocks)
        splits = total_kblocks;
    GemmParams p{};
    p.M = M; p.N = N; p.K = K; p.ldc = ldc; p.C = C;
    p.bias = static_cast<float const*>(bias);
    p.relu = relu; p.out_fp32 = out_fp32; p.atomic = splits > 1;
    p.groups = groups; p.c_group_stride = c_group_stride;
    p.kblocks_per_split = (total_kblocks + splits - 1) / splits;
    splits = (total_kblocks + p.kblocks_per_split - 1) / p.kblocks_per_split;
    p.addend = addend;
    CUtensorMap ta, tb;
    int status;
    if (a_mn && b_mn)
        status = make_tmap_3d_bf16(&ta, A, static_cast<uint64_t>(M), static_cast<uint64_t>(K), static_cast<uint64_t>(groups), static_cast<uint64_t>(lda), 64, kBK);
    else if (a_mn)
        status = make_tmap_2d_bf16(&ta, A, static_cast<uint64_t>(M), static_cast<uint64_t>(K), static_cast<uint64_t>(lda), 64, kBK);
    else
        status = make_tmap_2d_bf16(&ta, A, static_cast<uint64_t>(K), static_cast<uint64_t>(M), static_cast<uint64_t>(lda), kBK, kBM);
    if (status)
        return status;
    if (a_mn && b_mn)
        status = make_tmap_3d_bf16(&tb, B, static_cast<uint64_t>(N), static_cast<uint64_t>(K), static_cast<uint64_t>(groups), static_cast<uint64_t>(ldb), 64, kBK);
    else if (b_mn)
        status = make_tmap_2d_bf16(&tb, B, static_cast<uint64_t>(N), static_cast<uint64_t>(K), static_cast<uint64_t>(ldb), 64, kBK);
    else
        status = make_tmap_2d_bf16(&tb, B, static_cast<uint64_t>(K), static_cast<uint64_t>(N), static_cast<uint64_t>(ldb), kBK, static_cast<uint32_t>(bn));
    if (status)
        return status;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (a_mn)
        return b_mn ? dispatch_bn<true, true>(bn, ta, tb, p, splits, s) : dispatch_bn<true, false>(bn, ta, tb, p, splits, s);
    return b_mn ? dispatch_bn<false, true>(bn, ta, tb, p, splits, s) : dispatch_bn<false, false>(bn, ta, tb, p, splits, s);
}

// fp32 operands multiplied as TF32, fp32 accumulation and output: same layouts and options as agb_gemm_bf16_grouped;
// lda / ldb multiples of 4 elements, bases 16-byte aligned, bn in {64, 128} (0 = automatic), C (and `addend`) fp32.
int agb_gemm_tf32_grouped(void const* A, void const* B, void* C, int M, int N, int K, long long lda, long long ldb, long long ldc,
                          int a_mn, int b_mn, void const* bias, int relu, int splits, int bn, int groups, long long c_group_stride, void const* addend, void* stream) {
    using E = ElemTF32;
    if (M <= 0 || N <= 0 || K <= 0)
        return 0;
    if ((lda & 3) || (ldb & 3) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15))
        return 204;
    if (groups < 1)
        groups = 1;
    if (groups > 1 && !(a_mn && b_mn))
        return 206;
    if (splits < 1)
        splits = 1;
    if (bn == 0)
        bn = N <= 64 ? 64 : 128;
    int const total_kblocks = (K + E::kBK - 1) / E::kBK;
    if (splits > total_kblocks)
        splits = total_kblocks;
    if (splits > 1 && addend)
        return 207;
    GemmParams p{};
    p.M = M; p.N = N; p.K = K; p.ldc = ldc; p.C = C;
    p.bias = static_cast<float const*>(bias);
    p.relu = relu; p.out_fp32 = 1; p.atomic = splits > 1;
    p.groups = groups; p.c_group_stride = c_group_stride;
    p.kblocks_per_split = (total_kblocks + splits - 1) / splits;
    splits = (total_kblocks + p.kblocks_per_split - 1) / p.kblocks_per_split;
    p.addend = addend;
    CUtensorMap ta, tb;
    int status;
    uint64_t const m = static_cast<uint64_t>(M), n = static_cast<uint64_t>(N), k = static_cast<uint64_t>(K), g = static_cast<uint64_t>(groups);
    if (a_mn && b_mn)
        status = make_tmap_3d(&ta, A, m, k, g, static_cast<uint64_t>(lda), E::kChunk, E::kBK, 4);
    else if (a_mn)
        status = make_tmap_2d(&ta, A, m, k, static_cast<uint64_t>(lda), E::kChunk, E::kBK, 4);
    else
        status = make_tmap_2d(&ta, A, k, m, static_cast<uint64_t>(lda), E::kBK, kBM, 4);
    if (status)
        return status;
    if (a_mn && b_mn)
        status = make_tmap_3d(&tb, B, n, k, g, static_cast<uint64_t>(ldb), E::kChunk, E::kBK, 4);
    else if (b_mn)
        status = make_tmap_2d(&tb, B, n, k, static_cast<uint64_t>(ldb), E::kChunk, E::kBK, 4);
    else
        status = make_tmap_2d(&tb, B, k, n, static_cast<uint64_t>(ldb), E::kBK, static_cast<uint32_t>(bn), 4);
    if (status)
        return status;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (a_mn)
        return b_mn ? dispatch_bn_tf32<true, true>(bn, ta, tb, p, splits, s) : dispatch_bn_tf32<true, false>(bn, ta, tb, p, splits, s);
    return b_mn ? dispatch_bn_tf32<false, true>(bn, ta, tb, p, splits, s) : dispatch_bn_tf32<false, false>(bn, ta, tb, p, splits, s);
}

} // extern "C"
