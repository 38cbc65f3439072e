// Fused gather + gradient-aggregation-rule + optimizer update + parameter broadcast (sm_90a).
//
// This is the H100 replacement of the reference's whole PS data path
// (SURVEY §3.2: worker->PS gradient transfer, `native/op_krum/cpu.cpp`, `native/op_bulyan/cpu.cpp`,
// `deprecated_native/native.cpp` median/averaged-median/average-nan, `opt.apply_gradients`,
// PS->worker variable transfer). Per rank and step:
//
//   phase A kernels  (Krum/Bulyan/MDA, optional, one per gradient *bucket*, launched on a side stream while the backward pass is still
//                    producing the earlier layers' gradients) entry flag of the bucket, then stream this rank's share of the bucket of
//                    all n gradients straight from the peers' buffers (P2P loads over NVLink), accumulate the partial squared
//                    distances with direct differences, stage the tile locally
//   finish kernel    (cooperative) phase A of whatever was not pre-accumulated; partial matrices go to every peer's mailbox together
//                    with the rank's loss sum; summed in rank order => bit-identical distance matrix (and total loss) on every rank;
//                    one warp: Krum scores / Bulyan iterative selection, or the whole grid: MDA's minimum-diameter search
//                    (replicated on all ranks); phase D: aggregate the owned coordinates (mean of selected / coordinate-wise
//                    trimmed mean / median / NaN-aware mean), apply the optimizer,
//                    store the new parameters into every rank's buffer (P2P stores or one NVLS multimem.st); exit barrier
//                    geometric median / centered clipping instead: T + 1 passes over the owned coordinates, with one exchange of
//                    the n row distances per iteration (see `iterative_rule`)
//
// Attacked steps with an omniscient attack (ALIE / IPM) run `gar_byzantine_kernel` first: each rank crafts its owned coordinates of
// every Byzantine row from the honest values.
// With R = 1 the finish kernel alone is the stand-alone `[n, d] -> [d]` aggregation op. n <= 32 workers: up to 8 rows are held in
// registers at a time; more rows are processed in 8-row blocks (diagonal + cross passes over the staged copy).
// Step-varying scalars (flag epoch, learning rate, optimizer hyper-parameters) may be read from device memory so that the
// launches can be captured once in a CUDA graph.
// Ordering convention: finite ascending, non-finite last, ties -> lower worker index.

#include <cmath>

#include <cooperative_groups.h>
#include <cuda_bf16.h>

#include <agb_device.cuh>

namespace cg = cooperative_groups;
using namespace agb;

namespace {

constexpr int kMaxWorkers = 32;
constexpr int kMaxRanks = 16;
constexpr int kMaxPairs = kMaxWorkers * (kMaxWorkers - 1) / 2;   // 496
constexpr int kMaxSeg = 8;                // owned coordinate segments (one per gradient bucket)
constexpr int kSlotExchange = kMaxSeg;    // flag slots: [0, kMaxSeg) bucket entry, then exchange, then exit
constexpr int kSlotExit = kMaxSeg + 1;
constexpr int kSlotCraft = kMaxSeg + 2;   // entry barrier of the Byzantine crafting kernel
constexpr int kMaxIterations = 16;        // geometric median, centered clipping: iterations
constexpr int kSlotGeoMedian = kMaxSeg + 3;   // geometric median, centered clipping: one exchange slot per iteration
constexpr int kFlagSlots = kSlotGeoMedian + kMaxIterations;
constexpr int kBlockRows = 8;             // rows held in registers at a time

constexpr long long kMdaMaxSets = 1 << 20; // MDA enumerates the C(n, f) removal sets
enum Rule { kAverage = 0, kAverageNan = 1, kMedian = 2, kAveragedMedian = 3, kKrum = 4, kBulyan = 5, kTrimmedMean = 6, kMda = 7, kGeoMedian = 8,
           kCenteredClipping = 9 };
enum Opt { kNone = 0, kSgd = 1, kAdam = 2, kRmsprop = 3, kAdagrad = 4, kAdadelta = 5 };

struct GarArgs {
    int n, f, m, beta, rule;
    int R, rank;
    int nseg, first_seg;               // owned segments; segments [0, first_seg) were pre-accumulated by phase A kernels
    long long seg_lo[kMaxSeg], seg_hi[kMaxSeg];   // multiples of 4
    int seg_ctas[kMaxSeg];             // grid of the phase A kernel that handled segment s
    int seg_max_ctas;                  // stride (in CTAs) of `seg_partials`
    float const* grad[kMaxWorkers];    // row base pointers (local or peer-mapped)
    float const* grad_mc;              // multicast address of the [w, d] gradient matrix (NVLS in-switch reduction), or null
    int workers_per_rank;
    long long row_stride;              // elements between two rows of a rank's gradient matrix
    float* agg_out;                    // optional [d] (local): aggregated gradient of the owned coordinates
    int opt;
    float lr, h0, h1, h2;              // adam: b1,b2,eps | rmsprop: decay,momentum,eps | adadelta: rho,eps
    float const* hyper_ptr;            // device [lr, h0, h1, h2] overriding the immediates (graph replay), or null
    float* param;                      // local fp32 parameters [d]
    float* slot0;
    float* slot1;
    float* param_dst[kMaxRanks];       // every rank's parameter buffer (peer-mapped), incl. own
    float* param_mc;                   // multicast address of the parameter buffers, or null
    __nv_bfloat16* param_bf16_dst[kMaxRanks]; // optional bf16 compute copy of the parameters
    uint32_t* signal[kMaxRanks];       // [kFlagSlots][R] flags of every rank
    float* mailbox[kMaxRanks];         // [R][kMaxPairs + 1] partial distances (+ loss sum) of every rank
    uint32_t epoch;                    // immediate epoch, used when epoch_ptr is null
    uint32_t* epoch_ptr;               // device counter of completed steps: flags use *epoch_ptr + 1; the finish kernel increments it
    float* cta_partials;               // [grid][kMaxPairs]
    float* seg_partials;               // [kMaxSeg][seg_max_ctas][kMaxPairs]
    float* staging;                    // [n][owned length] or null
    float* dist_out;                   // optional [n * n] (geometric median, centered clipping: [iterations][n])
    int* info;                         // optional [64]: selection masks for tests/diagnostics
    float const* loss_in;              // optional [nloss] local per-worker losses
    int nloss;
    float* loss_out;                   // [1]: total loss over all ranks (summed in rank order)
    int iterations;                    // geometric median, centered clipping: iterations T in [1, kMaxIterations]
    float nu;                          // geometric median: smoothing, finite and > 0
    float tau;                         // centered clipping: clipping radius, finite and > 0
    float* center;                     // centered clipping: [d] (local) center v, read and updated on the owned coordinates
};

struct Shared {
    float dist[kMaxWorkers][kMaxWorkers + 1];
    union {
        float pruned[kMaxWorkers][kMaxWorkers + 1];      // Bulyan
        struct {                                          // MDA
            unsigned short order[kMaxPairs];              // pairs (i | j << 8) by descending distance
            unsigned binom[kMaxWorkers + 1][kMaxWorkers / 2 + 1];
            unsigned long long best[16];                  // per-warp minimum keys
        } mda;
        struct {                                          // geometric median, centered clipping: weights of the current iterate
            float beta[kMaxWorkers];                      // 1 / max(nu, sqrt(D_i)) (CC: the clipping factors c_i) of the kept rows
            float sum;                                    // geometric median: their sum, in ascending worker order
            unsigned mask;                                // kept rows; 0: no weights, the iterate is the median (CC: z_t is unchanged)
        } geo;
    };
    float scores[kMaxWorkers];
    float warp_partials[16][kBlockRows * kBlockRows];
    unsigned selmask[kMaxWorkers];   // Krum, MDA: [0]; Bulyan: one per round
    int selcount[kMaxWorkers];
    int theta;
    float hyper[4];
    uint32_t epoch;
};

// ---- VEC-wide (4 or 1) coordinate accesses ----------------------------------- //
template<int VEC> struct V;
template<> struct V<4> {
    static __device__ __forceinline__ void load_stream(float const* p, float (&v)[4]) {
        float4 t = ld_stream_f4(p);
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    static __device__ __forceinline__ void load(float const* p, float (&v)[4]) {
        float4 t = *reinterpret_cast<float4 const*>(p);
        v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    static __device__ __forceinline__ void store(float* p, float const (&v)[4]) {
        *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    }
    static __device__ __forceinline__ void store_stream(float* p, float const (&v)[4]) {
        st_stream_f4(p, make_float4(v[0], v[1], v[2], v[3]));
    }
    static __device__ __forceinline__ void store_mc(float* p, float const (&v)[4]) {
        multimem_st_f4(p, make_float4(v[0], v[1], v[2], v[3]));
    }
    static __device__ __forceinline__ void store_bf16(__nv_bfloat16* p, float const (&v)[4]) {
        __nv_bfloat162 lo = __floats2bfloat162_rn(v[0], v[1]), hi = __floats2bfloat162_rn(v[2], v[3]);
        *reinterpret_cast<uint2*>(p) = make_uint2(*reinterpret_cast<unsigned*>(&lo), *reinterpret_cast<unsigned*>(&hi));
    }
};
template<> struct V<1> {
    static __device__ __forceinline__ void load_stream(float const* p, float (&v)[1]) {
        asm volatile("ld.global.L1::no_allocate.f32 %0, [%1];" : "=f"(v[0]) : "l"(p));
    }
    static __device__ __forceinline__ void load(float const* p, float (&v)[1]) { v[0] = *p; }
    static __device__ __forceinline__ void store(float* p, float const (&v)[1]) { *p = v[0]; }
    static __device__ __forceinline__ void store_stream(float* p, float const (&v)[1]) {
        asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" :: "l"(p), "f"(v[0]) : "memory");
    }
    static __device__ __forceinline__ void store_mc(float* p, float const (&v)[1]) {
        asm volatile("multimem.st.relaxed.sys.global.f32 [%0], %1;" :: "l"(p), "f"(v[0]) : "memory");
    }
    static __device__ __forceinline__ void store_bf16(__nv_bfloat16* p, float const (&v)[1]) { *p = __float2bfloat16(v[0]); }
};

// ---- optimizer update of VEC consecutive coordinates + broadcast ------------- //
template<int VEC>
__device__ __forceinline__ void apply_update(GarArgs const& a, float const (&hyper)[4], long long x, float const (&g)[VEC]) {
    if (a.agg_out)
        V<VEC>::store(a.agg_out + x, g);
    if (a.opt == kNone)
        return;
    float const lr = hyper[0], h0 = hyper[1], h1 = hyper[2], h2 = hyper[3];
    float p[VEC];
    V<VEC>::load(a.param + x, p);
    if (a.opt == kSgd) {
#pragma unroll
        for (int c = 0; c < VEC; ++c)
            p[c] -= lr * g[c];
    } else {
        float s0[VEC], s1[VEC];
        V<VEC>::load(a.slot0 + x, s0);
        if (a.slot1) {
            V<VEC>::load(a.slot1 + x, s1);
        } else {
#pragma unroll
            for (int c = 0; c < VEC; ++c)
                s1[c] = 0.f;
        }
#pragma unroll
        for (int c = 0; c < VEC; ++c) {
            float const gc = g[c];
            float &pc = p[c], &u = s0[c], &v = s1[c];
            if (a.opt == kAdam) {            // lr already carries the bias correction sqrt(1-b2^t)/(1-b1^t)
                u = h0 * u + (1.f - h0) * gc;
                v = h1 * v + (1.f - h1) * gc * gc;
                pc -= lr * u / (sqrtf(v) + h2);
            } else if (a.opt == kRmsprop) {  // u: mean square, v: momentum
                u = h0 * u + (1.f - h0) * gc * gc;
                v = h1 * v + lr * gc * rsqrtf(u + h2);
                pc -= v;
            } else if (a.opt == kAdagrad) {  // u: accumulator
                u += gc * gc;
                pc -= lr * gc * rsqrtf(u);
            } else {                         // adadelta; u: accum, v: accum_update
                u = h0 * u + (1.f - h0) * gc * gc;
                float upd = sqrtf(v + h1) * rsqrtf(u + h1) * gc;
                v = h0 * v + (1.f - h0) * upd * upd;
                pc -= lr * upd;
            }
        }
        V<VEC>::store(a.slot0 + x, s0);
        if (a.slot1)
            V<VEC>::store(a.slot1 + x, s1);
    }
    if (a.param_mc) {
        V<VEC>::store_mc(a.param_mc + x, p);
    } else {
        for (int q = 0; q < a.R; ++q)
            V<VEC>::store_stream(a.param_dst[q] + x, p);
    }
    if (a.param_bf16_dst[0]) {
        for (int q = 0; q < a.R; ++q)
            V<VEC>::store_bf16(a.param_bf16_dst[q] + x, p);
    }
}

// ---- coordinate-wise rules on N register-resident values -------------------- //
// rank-counting selection: branch free, NaN-correct, index-stable; O(n^2) compares per coordinate.
template<int N> __device__ __forceinline__ float coord_median(float const (&v)[N], int n) {
    float out = 0.f;
    int const target = n / 2;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        if (i < n) {
            int rank = 0;
#pragma unroll
            for (int j = 0; j < N; ++j)
                if (j < n && j != i)
                    rank += before(v[j], j, v[i], i) ? 1 : 0;
            if (rank == target)
                out = v[i];
        }
    }
    return out;
}

// mean of the `beta` values closest to the (upper) median, summed in index order
template<int N> __device__ __forceinline__ float coord_averaged_median(float const (&v)[N], int n, int beta) {
    float const zero = coord_median<N>(v, n);
    float dev[N];
#pragma unroll
    for (int i = 0; i < N; ++i)
        dev[i] = fabsf(v[i] - zero);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        if (i < n) {
            int rank = 0;
#pragma unroll
            for (int j = 0; j < N; ++j)
                if (j < n && j != i)
                    rank += before(dev[j], j, dev[i], i) ? 1 : 0;
            if (rank < beta)
                sum += v[i];
        }
    }
    return sum / static_cast<float>(beta);
}

// mean of the values ranked [f, n - f), summed in index order (the f smallest and the f largest or non-finite values are dropped)
template<int N> __device__ __forceinline__ float coord_trimmed_mean(float const (&v)[N], int n, int f) {
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < N; ++i) {
        if (i < n) {
            int rank = 0;
#pragma unroll
            for (int j = 0; j < N; ++j)
                if (j < n && j != i)
                    rank += before(v[j], j, v[i], i) ? 1 : 0;
            if (rank >= f && rank < n - f)
                sum += v[i];
        }
    }
    return sum / static_cast<float>(n - 2 * f);
}

template<int N> __device__ __forceinline__ float coord_average_nan(float const (&v)[N], int n) {
    float sum = 0.f;
    int count = 0;
#pragma unroll
    for (int i = 0; i < N; ++i)
        if (i < n && is_finite(v[i])) {
            sum += v[i];
            ++count;
        }
    return sum / static_cast<float>(count);
}

// ---- cross-rank flag barrier ---------------------------------------------------- //
// `Args`: any kernel argument block with R, rank, signal[], epoch and epoch_ptr (GarArgs, ByzArgs)
template<class Args> __device__ __forceinline__ void signal_all(Args const& a, int slot, uint32_t epoch) {
    if (threadIdx.x < a.R)
        st_release_sys(a.signal[threadIdx.x] + slot * a.R + a.rank, epoch);
}
template<class Args> __device__ __forceinline__ void wait_all(Args const& a, int slot, uint32_t epoch) {
    if (threadIdx.x < a.R)
        wait_flag_sys(a.signal[a.rank] + slot * a.R + threadIdx.x, epoch);
}
template<class Args> __device__ __forceinline__ uint32_t current_epoch(Args const& a) {
    return a.epoch_ptr ? ld_acquire_sys(a.epoch_ptr) + 1u : a.epoch;
}

// index of the pair (i < j) in the row-major upper triangle of an n x n matrix
__device__ __forceinline__ int pair_index(int i, int j, int n) {
    return i * n - (i * (i + 1)) / 2 + (j - i - 1);
}

// offset of segment `seg` inside the staged copy (segments are stored back to back)
__device__ __forceinline__ long long staged_offset(GarArgs const& a, int seg) {
    long long off = 0;
    for (int s = 0; s < seg; ++s)
        off += a.seg_hi[s] - a.seg_lo[s];
    return off;
}
__device__ __forceinline__ long long owned_length(GarArgs const& a) {
    return staged_offset(a, a.nseg);
}

// ---- selection stages (warp 0) -------------------------------------------------- //
__device__ void select_krum(GarArgs const& a, Shared& sh) {
    int const lane = threadIdx.x, n = a.n, count = a.n - a.f - 2;
    float score = 0.f;
    if (lane < n) {
        for (int r = 0; r < count; ++r) {  // add the distances in ascending order (matches the host oracle)
            for (int j = 0; j < n; ++j) {
                if (j == lane)
                    continue;
                int rank = 0;
                for (int k = 0; k < n; ++k)
                    if (k != lane && k != j)
                        rank += before(sh.dist[lane][k], k, sh.dist[lane][j], j) ? 1 : 0;
                if (rank == r)
                    score += sh.dist[lane][j];
            }
        }
        sh.scores[lane] = score;
    }
    __syncwarp();
    bool selected = false;
    if (lane < n) {
        int rank = 0;
        for (int j = 0; j < n; ++j)
            if (j != lane)
                rank += before(sh.scores[j], j, score, lane) ? 1 : 0;
        selected = rank < a.m;
    }
    unsigned mask = __ballot_sync(0xffffffffu, selected);
    if (lane == 0) {
        sh.selmask[0] = mask;
        sh.selcount[0] = a.m;
        sh.theta = 1;
    }
}

__device__ void select_bulyan(GarArgs const& a, Shared& sh) {
    int const lane = threadIdx.x, n = a.n, inscore = a.n - a.f - 2, theta = a.n - 2 * a.f - 2;
    float score = 0.f;
    if (lane < n) {
        for (int j = 0; j < n; ++j) {
            if (j == lane) {
                sh.pruned[lane][j] = 0.f;
                continue;
            }
            int rank = 0;
            for (int k = 0; k < n; ++k)
                if (k != lane && k != j)
                    rank += before(sh.dist[lane][k], k, sh.dist[lane][j], j) ? 1 : 0;
            sh.pruned[lane][j] = rank < inscore ? sh.dist[lane][j] : 0.f; // farthest f+1 never counted => never subtracted
        }
        for (int r = 0; r < inscore; ++r)
            for (int j = 0; j < n; ++j) {
                if (j == lane)
                    continue;
                int rank = 0;
                for (int k = 0; k < n; ++k)
                    if (k != lane && k != j)
                        rank += before(sh.dist[lane][k], k, sh.dist[lane][j], j) ? 1 : 0;
                if (rank == r)
                    score += sh.dist[lane][j];
            }
    }
    bool removed = false;
    for (int k = 0; k < theta; ++k) {
        if (lane < n)
            sh.scores[lane] = score;
        unsigned removed_mask = __ballot_sync(0xffffffffu, removed);
        __syncwarp();
        int rank = 0;
        if (lane < n) {
            for (int j = 0; j < n; ++j) {
                if (j == lane)
                    continue;
                bool rj = (removed_mask >> j) & 1u;
                bool j_first = rj != removed ? !rj : before(sh.scores[j], j, score, lane);
                rank += j_first ? 1 : 0;
            }
        }
        int const count = a.m - k;
        unsigned mask = __ballot_sync(0xffffffffu, lane < n && rank < count);
        unsigned best_mask = __ballot_sync(0xffffffffu, lane < n && rank == 0);
        int const best = __ffs(best_mask) - 1;
        if (lane == 0) {
            sh.selmask[k] = mask;
            sh.selcount[k] = count;
        }
        if (lane == best)
            removed = true;
        else if (lane < n && !removed)
            score -= sh.pruned[lane][best];
        __syncwarp();
    }
    if (lane == 0)
        sh.theta = theta;
}

// MDA (every thread of the grid): the kept set S, |S| = n - f, of smallest diameter (largest distance between two members); ties -> the
// lexicographically smallest sorted index list, i.e. the largest __brev(mask). The C(n, f) removal sets are split over all threads: a
// thread unranks the first set of its range (colexicographic order = ascending masks) and steps with Gosper's hack. A set's diameter
// is the distance of the first pair, in descending distance order, whose ends are both kept: at most f (n - 1) + 1 steps. Keys
// (diameter bits, ~__brev(mask)) are exact, so their minimum does not depend on the reduction order: every CTA and every rank (same
// distance matrix) selects the same set. The per-CTA minima go through `cta_partials`, free again once the distances are exchanged.
__device__ void select_mda(GarArgs const& a, Shared& sh, cg::grid_group& grid) {
    constexpr int K = kMaxWorkers / 2 + 1;
    int const n = a.n, f = a.f, npairs = n * (n - 1) / 2;
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    for (int p = threadIdx.x; p < (kMaxWorkers + 1) * K; p += blockDim.x) {
        int const m = p / K, k = p % K;
        unsigned long long c = 1;   // C(m, k) < 2^32 for m <= 32; every partial product is an exact binomial times (m - t)
        for (int t = 0; t < k && t < m; ++t)
            c = c * (m - t) / (t + 1);
        sh.mda.binom[m][k] = k > m ? 0u : static_cast<unsigned>(c);
    }
    for (int p = threadIdx.x; p < npairs; p += blockDim.x) {   // rank of pair p by (distance descending, pair index ascending)
        int i = 0, rest = p;
        while (rest >= n - 1 - i) {
            rest -= n - 1 - i;
            ++i;
        }
        int const j = i + 1 + rest;
        float const dp = sh.dist[i][j];
        int rank = 0, q = 0;
        for (int qi = 0; qi < n - 1; ++qi)
            for (int qj = qi + 1; qj < n; ++qj, ++q) {
                float const dq = sh.dist[qi][qj];
                rank += (dq > dp || (dq == dp && q < p)) ? 1 : 0;
            }
        sh.mda.order[rank] = static_cast<unsigned short>(i | (j << 8));
    }
    __syncthreads();
    long long const total = sh.mda.binom[n][f];
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const per = (total + nthreads - 1) / nthreads;
    long long r = tid * per;
    long long const end = r + per < total ? r + per : total;
    unsigned const full = n == 32 ? 0xffffffffu : (1u << n) - 1u;
    unsigned long long best = ~0ull;
    if (r < end) {
        unsigned removed = 0;   // combinatorial number system: r = sum_k C(c_k, k), c_f > ... > c_1
        long long rest = r;
        for (int k = f; k >= 1; --k) {
            int c = n - 1;
            while (sh.mda.binom[c][k] > rest)
                --c;
            removed |= 1u << c;
            rest -= sh.mda.binom[c][k];
        }
        for (;;) {
            unsigned const keep = full & ~removed;
            float diam = 0.f;
            for (int q = 0; q < npairs; ++q) {
                unsigned const pr = sh.mda.order[q], i = pr & 0xffu, j = pr >> 8;
                if ((keep >> i) & (keep >> j) & 1u) {
                    diam = sh.dist[i][j];
                    break;
                }
            }
            unsigned long long const key = static_cast<unsigned long long>(__float_as_uint(diam)) << 32 | ~__brev(keep);
            best = key < best ? key : best;
            if (++r >= end)
                break;
            unsigned const low = removed & (0u - removed), up = removed + low;   // Gosper's hack: next mask with f bits
            removed = (((up ^ removed) >> 2) >> (__ffs(low) - 1)) | up;
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        unsigned long long const other = __shfl_xor_sync(0xffffffffu, best, o);
        best = other < best ? other : best;
    }
    if (lane == 0)
        sh.mda.best[warp] = best;
    __syncthreads();
    unsigned long long* const slots = reinterpret_cast<unsigned long long*>(a.cta_partials);
    if (threadIdx.x == 0) {
        for (int w = 0; w < nwarps; ++w)
            best = sh.mda.best[w] < best ? sh.mda.best[w] : best;
        slots[static_cast<long long>(blockIdx.x) * (kMaxPairs / 2)] = best;
    }
    __threadfence();
    grid.sync();
    if (threadIdx.x == 0) {
        unsigned long long key = ~0ull;
        for (unsigned b = 0; b < gridDim.x; ++b) {
            unsigned long long const other = *reinterpret_cast<unsigned long long volatile*>(slots + static_cast<long long>(b) * (kMaxPairs / 2));
            key = other < key ? other : key;
        }
        sh.selmask[0] = __brev(~static_cast<unsigned>(key));
        sh.selcount[0] = n - f;
        sh.theta = 1;
    }
}

// ---- phase A: partial pairwise squared distances over one owned segment --------------------------------------------- //
// Rows are handled in blocks of 8. Block 0's *diagonal* pass streams its rows from their owners (P2P loads), stages them locally and
// accumulates the pairs inside the block; the *cross* passes (0, b) do the same for the rows of block b while pairing them with the
// staged block 0; every later pass (diagonal b >= 1, cross (b, c > b)) reads the staged copy only (local HBM / L2), so each gradient
// crosses NVLink exactly once. n <= 8 is a single diagonal pass. Every pass folds its accumulators lanes -> warps -> CTA in a fixed
// order and adds the CTA's partial to `out[pair]` (slots only this CTA, and for a given pair only one of its threads, touches).
template<int COUNT>
__device__ __forceinline__ void fold_pass(Shared& sh, float const (&acc)[COUNT], float* out, int const* pair_of) {
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
#pragma unroll
    for (int p = 0; p < COUNT; ++p) {
        float s = warp_sum(acc[p]);
        if (lane == 0)
            sh.warp_partials[warp][p] = s;
    }
    __syncthreads();
    if (threadIdx.x < COUNT && pair_of[threadIdx.x] >= 0) {
        float s = 0.f;
        for (int w = 0; w < nwarps; ++w)
            s += sh.warp_partials[w][threadIdx.x];
        out[pair_of[threadIdx.x]] += s;
    }
    __syncthreads();
}

__device__ __forceinline__ float sq_dist(float4 const& u, float4 const& v) {
    float dx = u.x - v.x, dy = u.y - v.y, dz = u.z - v.z, dw = u.w - v.w;
    return (dx * dx + dy * dy) + (dz * dz + dw * dw);
}

template<bool CROSS>
__device__ void phase_a_segment(GarArgs const& a, Shared& sh, int* pair_of, int seg, float* out, long long tid, long long nthreads) {
    constexpr int B = kBlockRows, NPB = B * (B - 1) / 2;
    int const n = a.n, nb = CROSS ? (n + B - 1) / B : 1;
    long long const lo = a.seg_lo[seg], len4 = (a.seg_hi[seg] - lo) >> 2;
    long long const owned = owned_length(a), soff = staged_offset(a, seg);
    auto staged = [&](int row, long long v) { return a.staging + row * owned + soff + (v << 2); };
    for (int bi = 0; bi < nb; ++bi) {
        int const i0 = bi * B;
        bool const from_copy = a.staging != nullptr && bi > 0;   // blocks >= 1 were staged by the cross passes (0, b)
        if (threadIdx.x < NPB) {   // local pair index -> (i, j) -> global pair index
            int i = 0, rest = threadIdx.x;
            while (rest >= B - 1 - i) {
                rest -= B - 1 - i;
                ++i;
            }
            int const j = i + 1 + rest;
            pair_of[threadIdx.x] = i0 + j < n ? pair_index(i0 + i, i0 + j, n) : -1;
        }
        __syncthreads();
        {
            float acc[NPB];
#pragma unroll
            for (int p = 0; p < NPB; ++p)
                acc[p] = 0.f;
            for (long long v = tid; v < len4; v += nthreads) {
                long long const x = lo + (v << 2);
                float4 g[B];
#pragma unroll
                for (int i = 0; i < B; ++i) {
                    if (i0 + i < n)
                        g[i] = from_copy ? *reinterpret_cast<float4 const*>(staged(i0 + i, v)) : ld_stream_f4(a.grad[i0 + i] + x);
                    else
                        g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
                if (a.staging && !from_copy) {
#pragma unroll
                    for (int i = 0; i < B; ++i)
                        if (i0 + i < n)
                            *reinterpret_cast<float4*>(staged(i0 + i, v)) = g[i];
                }
                int p = 0;
#pragma unroll
                for (int i = 0; i < B - 1; ++i) {
#pragma unroll
                    for (int j = i + 1; j < B; ++j, ++p)
                        if (i0 + j < n)
                            acc[p] += sq_dist(g[i], g[j]);
                }
            }
            fold_pass<NPB>(sh, acc, out, pair_of);
        }
        if (CROSS) {
            for (int bj = bi + 1; bj < nb; ++bj) {
                int const j0 = bj * B;
                bool const j_from_copy = a.staging != nullptr && bi > 0;   // first touch of block bj is the pass (0, bj)
                if (threadIdx.x < B * B) {
                    int const i = threadIdx.x / B, j = threadIdx.x % B;
                    pair_of[threadIdx.x] = (i0 + i < n && j0 + j < n) ? pair_index(i0 + i, j0 + j, n) : -1;
                }
                __syncthreads();
                float acc[B * B];
#pragma unroll
                for (int p = 0; p < B * B; ++p)
                    acc[p] = 0.f;
                for (long long v = tid; v < len4; v += nthreads) {
                    long long const x = lo + (v << 2);
                    float4 gi[B], gj[B];
#pragma unroll
                    for (int i = 0; i < B; ++i) {
                        if (i0 + i < n)
                            gi[i] = a.staging ? *reinterpret_cast<float4 const*>(staged(i0 + i, v)) : ld_stream_f4(a.grad[i0 + i] + x);
                        else
                            gi[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
#pragma unroll
                    for (int j = 0; j < B; ++j) {
                        if (j0 + j < n) {
                            if (j_from_copy) {
                                gj[j] = *reinterpret_cast<float4 const*>(staged(j0 + j, v));
                            } else {
                                gj[j] = ld_stream_f4(a.grad[j0 + j] + x);
                                if (a.staging)
                                    *reinterpret_cast<float4*>(staged(j0 + j, v)) = gj[j];
                            }
                        } else {
                            gj[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                        }
                    }
#pragma unroll
                    for (int i = 0; i < B; ++i) {
#pragma unroll
                        for (int j = 0; j < B; ++j)
                            acc[i * B + j] += sq_dist(gi[i], gj[j]);
                    }
                }
                fold_pass<B * B>(sh, acc, out, pair_of);
            }
        }
    }
}

// Stand-alone phase A of one segment (bucket), launched while the backward pass is still running: non-cooperative, few CTAs.
template<bool CROSS>
__global__ void __launch_bounds__(256, 1) gar_phase_a_kernel(GarArgs const a, int seg) {
    __shared__ Shared sh;
    __shared__ int pair_of[kBlockRows * kBlockRows];
    int const npairs = a.n * (a.n - 1) / 2;
    uint32_t const epoch = current_epoch(a);
    if (a.R > 1) {   // bucket entry barrier: every rank's workers have produced this bucket's gradients
        if (blockIdx.x == 0)
            signal_all(a, seg, epoch);
        wait_all(a, seg, epoch);
    }
    float* out = a.seg_partials + (static_cast<long long>(seg) * a.seg_max_ctas + blockIdx.x) * kMaxPairs;
    for (int p = threadIdx.x; p < npairs; p += blockDim.x)
        out[p] = 0.f;
    __syncthreads();
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    phase_a_segment<CROSS>(a, sh, pair_of, seg, out, tid, nthreads);
}

// ---- iterative rules: geometric median (smoothed Weiszfeld, RFA) and centered clipping ---------- //
// Geometric median: z_0 = coordinate-wise median; for t < T: D_i = ||z_t - x_i||^2, rows with a non-finite D_i are skipped,
// beta_i = 1 / max(nu, sqrt(D_i)), S = sum beta_i and z_{t+1} = (sum beta_i x_i) / S, both sums over the kept rows in ascending worker
// order from +0; no kept row: z_{t+1} = z_t.
// Centered clipping (Karimireddy et al.): z_0 = the center v; for t < T: the same D_i and skipped rows, s_i = sqrt(D_i),
// c_i = 1 if s_i <= tau else tau / s_i, u = sum c_i (x_i - z_t) over the kept rows in ascending worker order from +0,
// z_{t+1} = z_t + u / n (all n rows); no kept row: z_{t+1} = z_t. v <- z_T.
// Every operation rounded once (explicit _rn intrinsics: no FMA contraction). Output z_T.
// T + 1 passes over the owned coordinates. Pass 0 loads the n values of each coordinate (P2P from the peers) and stages them when
// R > 1; later passes read the staged tile, or the local rows when R = 1. The geometric median's pass t recomputes z_t from the rows
// and the weights every CTA keeps in shared memory (z_t is never stored). Centered clipping keeps z_t in the center buffer: pass 0
// reads z_0, pass t >= 1 reads z_{t-1}, applies the weights of iteration t - 1 and stores z_t; every element is read and written by
// the same thread, between grid barriers. Each pass but the last accumulates the partial D_i in registers; the last pass goes
// through the optimizer and the broadcast instead.
// Exchange of iteration t: lanes -> warps -> CTA -> `cta_partials` -> grid barrier; block 0 folds the CTAs in order and stores the
// rank's partials into every rank's mailbox (floats [(t & 1) * 32, + n) of its [kMaxPairs + 1] region), then signals slot
// kSlotGeoMedian + t; every rank sums the R partials in rank order, so all ranks (and all CTAs) get the same D and the same weights.
// Double buffering makes the mailbox safe to reuse: the half written at iteration t + 1 was last read at iteration t - 1; a rank
// reads it before its block 0 reaches the grid barrier of iteration t, hence before it signals iteration t, and a writer stores
// iteration t + 1 only after it has passed the barrier of iteration t, i.e. after every rank's iteration-t signal. With R = 1 a
// second grid barrier takes the place of the flags. The loss travels through the exit barrier, as for the coordinate-wise rules.
template<int N, int VEC>
__device__ __forceinline__ void iterative_rule(GarArgs const& a, Shared& sh, cg::grid_group& grid, float const (&hyper)[4], uint32_t epoch,
                                               long long tid, long long nthreads) {
    int const n = a.n, T = a.iterations, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    bool const multi = a.R > 1;
    long long const owned = owned_length(a);
    if (threadIdx.x == 0)
        sh.geo.mask = 0u;
    __syncthreads();
    for (int t = 0; t <= T; ++t) {
        unsigned const mask = sh.geo.mask;
        float const S = sh.geo.sum;
        float acc[N];
#pragma unroll
        for (int i = 0; i < N; ++i)
            acc[i] = 0.f;
        for (int seg = 0; seg < a.nseg; ++seg) {
            long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC, soff = staged_offset(a, seg);
            for (long long v = tid; v < lenv; v += nthreads) {
                long long const x = lo + v * VEC;
                float g[N][VEC];
#pragma unroll
                for (int i = 0; i < N; ++i) {
                    if (i < n) {
                        float* const staged = a.staging ? a.staging + i * owned + soff + v * VEC : nullptr;
                        if (t == 0 || !staged) {
                            V<VEC>::load_stream(a.grad[i] + x, g[i]);
                            if (staged)
                                V<VEC>::store(staged, g[i]);
                        } else {
                            V<VEC>::load(staged, g[i]);
                        }
                    } else {
#pragma unroll
                        for (int c = 0; c < VEC; ++c)
                            g[i][c] = 0.f;
                    }
                }
                // z_t coordinate by coordinate, each followed by its share of the partial D_i: a coordinate's n values are dead
                // once it is done, which keeps the pass within the register budget of the 8-worker instance
                float z[VEC];
                if (a.rule == kCenteredClipping)
                    V<VEC>::load(a.center + x, z);   // z_0, or z_{t-1}
#pragma unroll
                for (int c = 0; c < VEC; ++c) {
                    if (a.rule == kCenteredClipping) {
                        if (mask != 0u) {
                            float u = 0.f;
#pragma unroll
                            for (int i = 0; i < N; ++i)
                                if ((mask >> i) & 1u)
                                    u = __fadd_rn(u, __fmul_rn(sh.geo.beta[i], __fsub_rn(g[i][c], z[c])));
                            z[c] = __fadd_rn(z[c], __fdiv_rn(u, static_cast<float>(n)));
                        }
                    } else if (mask == 0u) {
                        float vals[N];
#pragma unroll
                        for (int i = 0; i < N; ++i)
                            vals[i] = g[i][c];
                        z[c] = coord_median<N>(vals, n);
                    } else {
                        float num = 0.f;
#pragma unroll
                        for (int i = 0; i < N; ++i)
                            if ((mask >> i) & 1u)
                                num = __fadd_rn(num, __fmul_rn(sh.geo.beta[i], g[i][c]));
                        z[c] = __fdiv_rn(num, S);
                    }
                    if (t < T) {
#pragma unroll
                        for (int i = 0; i < N; ++i)
                            if (i < n) {
                                float const e = __fsub_rn(z[c], g[i][c]);
                                acc[i] = __fmaf_rn(e, e, acc[i]);
                            }
                    }
                }
                if (a.rule == kCenteredClipping && mask != 0u)
                    V<VEC>::store(a.center + x, z);   // z_t
                if (t == T)
                    apply_update<VEC>(a, hyper, x, z);
            }
        }
        if (t == T)
            break;
        // -------- exchange of the n squared distances of iteration t -------- //
#pragma unroll
        for (int i = 0; i < N; ++i) {
            if (i < n) {
                float const s = warp_sum(acc[i]);
                if (lane == 0)
                    sh.warp_partials[warp][i] = s;
            }
        }
        __syncthreads();
        if (threadIdx.x < n) {
            float s = 0.f;
            for (int w = 0; w < nwarps; ++w)
                s += sh.warp_partials[w][threadIdx.x];
            a.cta_partials[static_cast<long long>(blockIdx.x) * kMaxPairs + threadIdx.x] = s;
        }
        __threadfence();
        grid.sync();
        int const half = (t & 1) * kMaxWorkers;
        if (blockIdx.x == 0) {
            if (threadIdx.x < n) {
                float s = 0.f;
                for (unsigned b = 0; b < gridDim.x; ++b)
                    s += ld_volatile_f(a.cta_partials + static_cast<long long>(b) * kMaxPairs + threadIdx.x);
                for (int q = 0; q < a.R; ++q)
                    a.mailbox[q][a.rank * (kMaxPairs + 1) + half + threadIdx.x] = s;
            }
            fence_sys();
            __syncthreads();
            if (multi)
                signal_all(a, kSlotGeoMedian + t, epoch);
        }
        if (multi) {
            wait_all(a, kSlotGeoMedian + t, epoch);
            __syncthreads();
        } else {
            grid.sync();
        }
        // -------- weights of z_{t+1} (warp 0 of every CTA, identical everywhere) -------- //
        if (warp == 0) {
            float D = 0.f;
            if (lane < n) {
                for (int q = 0; q < a.R; ++q)
                    D += ld_volatile_f(a.mailbox[a.rank] + q * (kMaxPairs + 1) + half + lane);
                if (a.dist_out && blockIdx.x == 0)
                    a.dist_out[t * n + lane] = D;
            }
            bool const keep = lane < n && is_finite(D);
            unsigned const kept = __ballot_sync(0xffffffffu, keep);
            if (a.rule == kCenteredClipping) {   // no kept row: mask 0, the next pass keeps z_t
                float const s = __fsqrt_rn(D);
                sh.geo.beta[lane] = keep ? (s <= a.tau ? 1.f : __fdiv_rn(a.tau, s)) : 0.f;
                if (lane == 0)
                    sh.geo.mask = kept;
            } else if (kept != 0u) {   // no kept row: z_{t+1} = z_t, the weights stay
                float const beta = keep ? __fdiv_rn(1.f, fmaxf(a.nu, __fsqrt_rn(D))) : 0.f;
                float sum = 0.f;
                for (int j = 0; j < n; ++j) {
                    float const bj = __shfl_sync(0xffffffffu, beta, j);
                    if ((kept >> j) & 1u)
                        sum = __fadd_rn(sum, bj);
                }
                sh.geo.beta[lane] = beta;
                if (lane == 0) {
                    sh.geo.mask = kept;
                    sh.geo.sum = sum;
                }
            }
        }
        __syncthreads();
    }
}

// ---- the finish kernel -------------------------------------------------------------- //
template<int N, int VEC>
__global__ void __launch_bounds__(N <= 8 ? 512 : 256, 1) gar_fused_kernel(GarArgs const a) {
    __shared__ Shared sh;
    __shared__ int pair_of[kBlockRows * kBlockRows];
    cg::grid_group grid = cg::this_grid();
    int const n = a.n, npairs = n * (n - 1) / 2;
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    bool const multi = a.R > 1;
    bool const distance_rule = a.rule == kKrum || a.rule == kBulyan || a.rule == kMda;
    if (threadIdx.x == 0) {
        sh.epoch = current_epoch(a);
        for (int i = 0; i < 4; ++i)
            sh.hyper[i] = a.hyper_ptr ? a.hyper_ptr[i] : (i == 0 ? a.lr : i == 1 ? a.h0 : i == 2 ? a.h1 : a.h2);
    }
    __syncthreads();
    uint32_t const epoch = sh.epoch;
    float const hyper[4] = {sh.hyper[0], sh.hyper[1], sh.hyper[2], sh.hyper[3]};
    long long const owned = owned_length(a);

    if (multi && a.first_seg < a.nseg) { // entry barrier of the segments aggregated here: every rank's gradients are published
        if (blockIdx.x == 0)
            signal_all(a, a.first_seg, epoch);
        wait_all(a, a.first_seg, epoch);
        __syncthreads();
    }
    float local_loss = 0.f;
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss_in)
        for (int j = 0; j < a.nloss; ++j)
            local_loss += a.loss_in[j];

    if (distance_rule) {
        // -------- phase A of the segments that were not pre-accumulated -------- //
        float* mine = a.cta_partials + static_cast<long long>(blockIdx.x) * kMaxPairs;
        for (int p = threadIdx.x; p < npairs; p += blockDim.x)
            mine[p] = 0.f;
        __syncthreads();
        for (int seg = a.first_seg; seg < a.nseg; ++seg)
            phase_a_segment<(N > kBlockRows)>(a, sh, pair_of, seg, mine, tid, nthreads);
        __threadfence();
        grid.sync();
        // fixed order: pre-accumulated segments (ascending, their CTAs ascending), then this kernel's CTAs, then ranks (ascending)
        if (blockIdx.x == 0) {
            for (int p = threadIdx.x; p < npairs; p += blockDim.x) {
                float s = 0.f;
                for (int seg = 0; seg < a.first_seg; ++seg)
                    for (int b = 0; b < a.seg_ctas[seg]; ++b)
                        s += ld_volatile_f(a.seg_partials + (static_cast<long long>(seg) * a.seg_max_ctas + b) * kMaxPairs + p);
                for (unsigned b = 0; b < gridDim.x; ++b)
                    s += ld_volatile_f(a.cta_partials + static_cast<long long>(b) * kMaxPairs + p);
                for (int q = 0; q < a.R; ++q)
                    a.mailbox[q][a.rank * (kMaxPairs + 1) + p] = s;
            }
            if (threadIdx.x == 0)
                for (int q = 0; q < a.R; ++q)
                    a.mailbox[q][a.rank * (kMaxPairs + 1) + kMaxPairs] = local_loss;
            fence_sys();
            __syncthreads();
            if (multi)
                signal_all(a, kSlotExchange, epoch);
        }
        if (multi) {
            wait_all(a, kSlotExchange, epoch);
            __syncthreads();
        } else {
            grid.sync();
        }
        // -------- full distance matrix (rank order => identical everywhere) + selection -------- //
        for (int p = threadIdx.x; p < kMaxWorkers * (kMaxWorkers + 1); p += blockDim.x)
            (&sh.dist[0][0])[p] = 0.f;
        __syncthreads();
        for (int p = threadIdx.x; p < npairs; p += blockDim.x) {
            int i = 0, rest = p;
            while (rest >= n - 1 - i) { // pair index -> (i, j) of the upper triangle
                rest -= n - 1 - i;
                ++i;
            }
            int const j = i + 1 + rest;
            float s = 0.f;
            for (int q = 0; q < a.R; ++q)
                s += ld_volatile_f(a.mailbox[a.rank] + q * (kMaxPairs + 1) + p);
            if (!is_finite(s))
                s = __int_as_float(0x7f800000);
            sh.dist[i][j] = s;
            sh.dist[j][i] = s;
            if (a.dist_out && blockIdx.x == 0) {
                a.dist_out[i * n + j] = s;
                a.dist_out[j * n + i] = s;
            }
        }
        if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss_out) {
            float total = 0.f;
            for (int q = 0; q < a.R; ++q)
                total += ld_volatile_f(a.mailbox[a.rank] + q * (kMaxPairs + 1) + kMaxPairs);
            *a.loss_out = total;
        }
        __syncthreads();
        if (a.rule == kMda) {
            select_mda(a, sh, grid);
        } else if (threadIdx.x < 32) {
            if (a.rule == kKrum)
                select_krum(a, sh);
            else
                select_bulyan(a, sh);
        }
        __syncthreads();
        if (a.info && blockIdx.x == 0 && threadIdx.x < sh.theta) {
            a.info[0] = sh.theta;
            a.info[1 + threadIdx.x] = static_cast<int>(sh.selmask[threadIdx.x]);
        }
        // -------- phase D: aggregate the owned coordinates from the staged copy, update, broadcast -------- //
        int const theta = sh.theta;
        for (int seg = 0; seg < a.nseg; ++seg) {
            long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC, soff = staged_offset(a, seg);
            for (long long v = tid; v < lenv; v += nthreads) {
                long long const x = lo + v * VEC;
                auto load_row = [&](int i, float (&dst)[VEC]) {
                    if (a.staging)
                        V<VEC>::load(a.staging + i * owned + soff + v * VEC, dst);
                    else
                        V<VEC>::load_stream(a.grad[i] + x, dst);
                };
                float out[VEC];
                if (a.rule != kBulyan) {   // Krum, MDA: mean of the selected rows
                    unsigned const mask = sh.selmask[0];
                    float sum[VEC];
#pragma unroll
                    for (int c = 0; c < VEC; ++c)
                        sum[c] = 0.f;
                    if (N <= 16) {   // all selected rows in flight at once, summed in ascending worker order
                        float g[N][VEC];
#pragma unroll
                        for (int i = 0; i < N; ++i)
                            if ((mask >> i) & 1u)
                                load_row(i, g[i]);
#pragma unroll
                        for (int i = 0; i < N; ++i)
                            if ((mask >> i) & 1u) {
#pragma unroll
                                for (int c = 0; c < VEC; ++c)
                                    sum[c] += g[i][c];
                            }
                    } else {
                        for (int i = 0; i < n; ++i) {
                            if ((mask >> i) & 1u) {
                                float g[VEC];
                                load_row(i, g);
#pragma unroll
                                for (int c = 0; c < VEC; ++c)
                                    sum[c] += g[c];
                            }
                        }
                    }
                    float const count = static_cast<float>(sh.selcount[0]);
#pragma unroll
                    for (int c = 0; c < VEC; ++c)
                        out[c] = sum[c] / count;
                } else {
                    unsigned needed = 0;
                    for (int k = 0; k < theta; ++k)
                        needed |= sh.selmask[k];
                    float g[N][VEC];
#pragma unroll
                    for (int i = 0; i < N; ++i) {
                        if (i < n && ((needed >> i) & 1u)) {
                            load_row(i, g[i]);
                        } else {
#pragma unroll
                            for (int c = 0; c < VEC; ++c)
                                g[i][c] = 0.f;
                        }
                    }
#pragma unroll
                    for (int c = 0; c < VEC; ++c) {
                        float vals[N];
#pragma unroll
                        for (int k = 0; k < N; ++k) {
                            vals[k] = 0.f;
                            if (k < theta) {
                                unsigned const mask = sh.selmask[k];
                                float sum = 0.f;
#pragma unroll
                                for (int i = 0; i < N; ++i)
                                    if ((mask >> i) & 1u)
                                        sum += g[i][c];
                                vals[k] = sum / static_cast<float>(sh.selcount[k]);
                            }
                        }
                        out[c] = coord_averaged_median<N>(vals, theta, a.beta);
                    }
                }
                apply_update<VEC>(a, hyper, x, out);
            }
        }
    } else if (a.rule == kGeoMedian || a.rule == kCenteredClipping) {
        iterative_rule<N, VEC>(a, sh, grid, hyper, epoch, tid, nthreads);
    } else {
        // -------- coordinate-wise rules: one streaming pass -------- //
        bool const in_switch = a.rule == kAverage && a.grad_mc != nullptr;
        for (int seg = 0; seg < a.nseg; ++seg) {
            long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC;
            for (long long v = tid; v < lenv; v += nthreads) {
                long long const x = lo + v * VEC;
                float out[VEC];
                if (a.rule == kAverage) {
                    float sum[VEC];
#pragma unroll
                    for (int c = 0; c < VEC; ++c)
                        sum[c] = 0.f;
                    if (VEC == 4 && in_switch) {   // NVLS: the switch adds the same row of every rank; rows of one rank are added here
                        for (int j = 0; j < a.workers_per_rank; ++j) {
                            float4 t = multimem_ld_reduce_add_f4(a.grad_mc + j * a.row_stride + x);
                            sum[0] += t.x; sum[1 % VEC] += t.y; sum[2 % VEC] += t.z; sum[3 % VEC] += t.w;
                        }
                    } else {
                        if (N <= 16) {
                            float g[N][VEC];
#pragma unroll
                            for (int i = 0; i < N; ++i)
                                if (i < n)
                                    V<VEC>::load_stream(a.grad[i] + x, g[i]);
#pragma unroll
                            for (int i = 0; i < N; ++i)
                                if (i < n) {
#pragma unroll
                                    for (int c = 0; c < VEC; ++c)
                                        sum[c] += g[i][c];
                                }
                        } else {
                            for (int i = 0; i < n; ++i) {
                                float g[VEC];
                                V<VEC>::load_stream(a.grad[i] + x, g);
#pragma unroll
                                for (int c = 0; c < VEC; ++c)
                                    sum[c] += g[c];
                            }
                        }
                    }
                    float const count = static_cast<float>(n);
#pragma unroll
                    for (int c = 0; c < VEC; ++c)
                        out[c] = sum[c] / count;
                } else {
                    float g[N][VEC];
#pragma unroll
                    for (int i = 0; i < N; ++i) {
                        if (i < n) {
                            V<VEC>::load_stream(a.grad[i] + x, g[i]);
                        } else {
#pragma unroll
                            for (int c = 0; c < VEC; ++c)
                                g[i][c] = 0.f;
                        }
                    }
#pragma unroll
                    for (int c = 0; c < VEC; ++c) {
                        float vals[N];
#pragma unroll
                        for (int i = 0; i < N; ++i)
                            vals[i] = g[i][c];
                        float r;
                        if (a.rule == kAverageNan)
                            r = coord_average_nan<N>(vals, n);
                        else if (a.rule == kMedian)
                            r = coord_median<N>(vals, n);
                        else if (a.rule == kTrimmedMean)
                            r = coord_trimmed_mean<N>(vals, n, a.f);
                        else
                            r = coord_averaged_median<N>(vals, n, a.beta);
                        out[c] = r;
                    }
                }
                apply_update<VEC>(a, hyper, x, out);
            }
        }
    }

    if (multi) { // exit barrier: all slices have landed on all ranks, gradient buffers are free again
        fence_sys();
        grid.sync();
        if (blockIdx.x == 0) {
            if (!distance_rule && threadIdx.x == 0) {   // rules without an exchange stage carry the loss through the exit barrier
                for (int q = 0; q < a.R; ++q)
                    a.mailbox[q][a.rank * (kMaxPairs + 1) + kMaxPairs] = local_loss;
                fence_sys();
            }
            __syncthreads();
            signal_all(a, kSlotExit, epoch);
            wait_all(a, kSlotExit, epoch);
            __syncthreads();
            if (!distance_rule && threadIdx.x == 0 && a.loss_out) {
                float total = 0.f;
                for (int q = 0; q < a.R; ++q)
                    total += ld_volatile_f(a.mailbox[a.rank] + q * (kMaxPairs + 1) + kMaxPairs);
                *a.loss_out = total;
            }
        }
    } else if (!distance_rule && blockIdx.x == 0 && threadIdx.x == 0 && a.loss_out) {
        *a.loss_out = local_loss;
    }
    if (a.epoch_ptr && blockIdx.x == 0 && threadIdx.x == 0)
        *a.epoch_ptr = epoch;   // this step is complete (every CTA read the counter before the barriers above)
}

// ---- omniscient Byzantine rows (ALIE / IPM) ------------------------------------------ //
// Every Byzantine row receives, at each owned coordinate, a value computed from the honest values of that coordinate only:
//   mu = ((h[Hs0] + h[Hs1]) + ...) / H           honest slots ascending, one division
//   v  = (sum_i (h_i - mu) * (h_i - mu)) / (H - 1)  ALIE only, same order
//   ALIE: b = mu + z * sqrt(v)          IPM: b = (-eps) * mu
// one IEEE-rounded operation at a time (explicit _rn intrinsics: no FMA contraction), so that every back-end gets the same bits.
//
// With R > 1 each rank crafts its owned segments of every Byzantine row, wherever that row lives (P2P stores into peers' gradient
// buffers). Entry barrier (slot kSlotCraft, the step's epoch): every rank's backward has written its rows before any honest value is
// read or any Byzantine row is overwritten. The kernel is not cooperative, so every CTA signals (idempotent) before it waits: no CTA
// waits on a CTA that may never be scheduled. No exit barrier: rank q writes only its own segments of each Byzantine row, and only
// rank q's finish kernel (next in the same stream) reads them; the closing system-scope fence orders these stores before that
// kernel's loads, including its NVLS multimem.ld_reduce of `average`. The rows are overwritten again only by the next step's
// backward, which every rank starts after the finish kernels' exit barrier.
//
// Up to N = 8 honest values are held in registers across both passes; with more, the variance pass re-reads them from memory.
struct ByzArgs {
    float* rows[kMaxWorkers];          // row base pointers (local or peer-mapped)
    int honest[kMaxWorkers];           // honest slots, ascending
    int byz[kMaxWorkers];              // Byzantine slots
    int H, K;
    int mode;                          // 0: ALIE, 1: IPM
    float coef;                        // ALIE: z; IPM: epsilon
    int nseg;
    long long seg_lo[kMaxSeg], seg_hi[kMaxSeg];
    int R, rank;
    uint32_t* signal[kMaxRanks];
    uint32_t epoch;
    uint32_t* epoch_ptr;
};
enum ByzMode { kAlie = 0, kIpm = 1 };

template<int N>
__global__ void __launch_bounds__(256) gar_byzantine_kernel(ByzArgs const a) {
    if (a.R > 1) {
        uint32_t const epoch = current_epoch(a);
        signal_all(a, kSlotCraft, epoch);
        wait_all(a, kSlotCraft, epoch);
        __syncthreads();
    }
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    int const H = a.H;
    float const count = static_cast<float>(H);
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4;
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            float g[N > 0 ? N : 1][4];
            float mu[4], out[4];
            if constexpr (N > 0) {   // registers: the H honest values are loaded once
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if (i < H)
                        V<4>::load_stream(a.rows[a.honest[i]] + x, g[i]);
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    mu[c] = g[0][c];
#pragma unroll
                for (int i = 1; i < N; ++i)
                    if (i < H) {
#pragma unroll
                        for (int c = 0; c < 4; ++c)
                            mu[c] = __fadd_rn(mu[c], g[i][c]);
                    }
            } else {
                V<4>::load(a.rows[a.honest[0]] + x, mu);
                for (int i = 1; i < H; ++i) {
                    float h[4];
                    V<4>::load(a.rows[a.honest[i]] + x, h);
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        mu[c] = __fadd_rn(mu[c], h[c]);
                }
            }
#pragma unroll
            for (int c = 0; c < 4; ++c)
                mu[c] = __fdiv_rn(mu[c], count);
            if (a.mode == kIpm) {
                float const neg = -a.coef;
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    out[c] = __fmul_rn(neg, mu[c]);
            } else {
                float var[4];
                auto add_square = [&](int i, float const (&h)[4]) {
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        float const dev = __fsub_rn(h[c], mu[c]);
                        float const sq = __fmul_rn(dev, dev);
                        var[c] = i == 0 ? sq : __fadd_rn(var[c], sq);
                    }
                };
                if constexpr (N > 0) {
#pragma unroll
                    for (int i = 0; i < N; ++i)
                        if (i < H)
                            add_square(i, g[i]);
                } else {
                    for (int i = 0; i < H; ++i) {
                        float h[4];
                        V<4>::load(a.rows[a.honest[i]] + x, h);
                        add_square(i, h);
                    }
                }
                float const dof = static_cast<float>(H - 1);
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    out[c] = __fadd_rn(mu[c], __fmul_rn(a.coef, __fsqrt_rn(__fdiv_rn(var[c], dof))));
            }
            for (int k = 0; k < a.K; ++k)
                V<4>::store_stream(a.rows[a.byz[k]] + x, out);
        }
    }
    fence_sys();
}

// ---- small stand-alone kernels (baseline path, attacks, diagnostics) ------------- //
__global__ void sgd_kernel(float* __restrict__ p, float const* __restrict__ g, float lr, long long d) {
    long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
    long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
    for (; i + 3 < d; i += stride) {
        float4 pv = *reinterpret_cast<float4 const*>(p + i), gv = *reinterpret_cast<float4 const*>(g + i);
        pv.x -= lr * gv.x; pv.y -= lr * gv.y; pv.z -= lr * gv.z; pv.w -= lr * gv.w;
        *reinterpret_cast<float4*>(p + i) = pv;
    }
}

// Worker momentum (El Mhamdi et al., "Distributed Momentum for Byzantine-resilient SGD"): every element of the w rows of a rank,
// M <- beta * M + c * G, then G <- M, each operation rounded once (explicit _rn intrinsics: no FMA contraction); c = 1 - dampening.
// One launch for the w rows (blockIdx.y = row), grid-stride along a row; streaming: G and M are read and written once, 16 bytes per
// coordinate. M is only read again at the next step, G right away by the aggregation.
template<int VEC>
__global__ void worker_momentum_kernel(float* __restrict__ g, long long g_stride, float* __restrict__ m, long long m_stride, long long d,
                                       float beta, float c) {
    float* const grow = g + static_cast<long long>(blockIdx.y) * g_stride;
    float* const mrow = m + static_cast<long long>(blockIdx.y) * m_stride;
    long long const stride = static_cast<long long>(gridDim.x) * blockDim.x * VEC;
    for (long long x = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * VEC; x < d; x += stride) {
        float gv[VEC], mv[VEC];
        V<VEC>::load(grow + x, gv);
        V<VEC>::load_stream(mrow + x, mv);
#pragma unroll
        for (int k = 0; k < VEC; ++k)
            mv[k] = __fadd_rn(__fmul_rn(beta, mv[k]), __fmul_rn(c, gv[k]));
        V<VEC>::store_stream(mrow + x, mv);
        V<VEC>::store(grow + x, mv);
    }
}

// Lossy-transport emulation (reference: tf_patches mpi_rendezvous_mgr.patch:814-843): every `chunk`-byte
// datagram of the serialized gradient is lost with probability `rate`; lost chunks become NaN (mode 0),
// zeros (mode 1) or the previous gradient's bytes (mode 2, "CLEVER").
__global__ void drop_chunks_kernel(float* g, float const* previous, long long d, long long chunk_elems, float rate, int mode, unsigned long long seed) {
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (; i < d; i += stride) {
        unsigned long long h = (static_cast<unsigned long long>(i / chunk_elems) + 1) * 0x9E3779B97F4A7C15ull ^ seed;
        h ^= h >> 33; h *= 0xff51afd7ed558ccdull; h ^= h >> 33; h *= 0xc4ceb9fe1a85ec53ull; h ^= h >> 33;
        float u = static_cast<float>(h >> 40) * (1.0f / 16777216.0f);
        if (u < rate)
            g[i] = mode == 0 ? __int_as_float(0x7fc00000) : mode == 1 ? 0.f : previous[i];
    }
}

// Order-independent 64-bit checksum of a float buffer (debug: cross-rank parameter equality).
__global__ void checksum_kernel(float const* p, long long d, unsigned long long* out) {
    unsigned long long local = 0;
    long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (; i < d; i += stride) {
        unsigned long long h = (static_cast<unsigned long long>(__float_as_uint(p[i])) << 20) ^ static_cast<unsigned long long>(i);
        h ^= h >> 29; h *= 0xbf58476d1ce4e5b9ull; h ^= h >> 32;
        local += h;
    }
    for (int offset = 16; offset > 0; offset >>= 1)
        local += __shfl_xor_sync(0xffffffffu, local, offset);
    if ((threadIdx.x & 31) == 0)
        atomicAdd(out, local);
}

__global__ void cast_bf16_kernel(float const* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long d) {
    long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
    long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
    for (; i + 3 < d; i += stride) {
        float4 v = *reinterpret_cast<float4 const*>(src + i);
        __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
        *reinterpret_cast<uint2*>(dst + i) = make_uint2(*reinterpret_cast<unsigned*>(&lo), *reinterpret_cast<unsigned*>(&hi));
    }
}

template<int N, int VEC> int launch(GarArgs& a, int max_ctas, cudaStream_t stream) {
    int const threads = N <= 8 ? 512 : 256;
    int device = 0, sms = 0, per_sm = 0;
    AGB_CUDA_OK(cudaGetDevice(&device));
    AGB_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    AGB_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gar_fused_kernel<N, VEC>, threads, 0));
    if (per_sm < 1)
        return 2;
    long long work = 0;
    for (int s = 0; s < a.nseg; ++s)
        work += (a.seg_hi[s] - a.seg_lo[s]) / VEC;
    long long want = (work + threads - 1) / threads;
    int grid = sms * per_sm;
    if (max_ctas > 0 && grid > max_ctas)
        grid = max_ctas;
    if (want < grid)
        grid = want < 1 ? 1 : static_cast<int>(want);
    void* params[] = {&a};
    AGB_CUDA_OK(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(gar_fused_kernel<N, VEC>), dim3(grid), dim3(threads), params, 0, stream));
    return 0;
}

// ptrs layout (all device addresses, 0 = absent):
//   [0..32) gradient rows | [32] agg_out | [33] param | [34] slot0 | [35] slot1 | [36] param_mc | [37] cta_partials | [38] staging
//   [39] dist_out | [40] info | [41] grad_mc | [42] epoch_ptr | [43] hyper_ptr | [44] seg_partials | [45] loss_in | [46] loss_out
//   [48..64) param_dst | [64..80) signal | [80..96) mailbox | [96..112) param_bf16_dst
// ints: n f m beta rule R rank opt epoch max_ctas workers_per_rank nseg first_seg nloss seg_max_ctas phase_a_ctas | [16..24) seg_ctas | [24] phase_a_threads
//   [47] center (centered clipping)
//       [25] iterations
// longs: row_stride | [1..9) seg_lo | [9..17) seg_hi ; floats: lr h0 h1 h2 nu tau
int fill_args(GarArgs& a, unsigned long long const* ptrs, int const* ints, long long const* longs, float const* floats) {
    a.n = ints[0]; a.f = ints[1]; a.m = ints[2]; a.beta = ints[3]; a.rule = ints[4];
    a.R = ints[5]; a.rank = ints[6]; a.opt = ints[7]; a.epoch = static_cast<uint32_t>(ints[8]);
    a.workers_per_rank = ints[10];
    a.nseg = ints[11]; a.first_seg = ints[12]; a.nloss = ints[13]; a.seg_max_ctas = ints[14];
    a.iterations = ints[25];
    a.row_stride = longs[0];
    a.lr = floats[0]; a.h0 = floats[1]; a.h1 = floats[2]; a.h2 = floats[3]; a.nu = floats[4]; a.tau = floats[5];
    a.center = reinterpret_cast<float*>(ptrs[47]);
    if (a.n < 1 || a.n > kMaxWorkers || a.R < 1 || a.R > kMaxRanks || a.rank < 0 || a.rank >= a.R)
        return 100;
    if (a.nseg < 1 || a.nseg > kMaxSeg || a.first_seg < 0 || a.first_seg > a.nseg)
        return 101;
    for (int s = 0; s < a.nseg; ++s) {
        a.seg_lo[s] = longs[1 + s];
        a.seg_hi[s] = longs[1 + kMaxSeg + s];
        a.seg_ctas[s] = ints[16 + s];
        if ((a.seg_lo[s] & 3) || (a.seg_hi[s] & 3) || a.seg_hi[s] < a.seg_lo[s])
            return 101;
    }
    if (a.rule < 0 || a.rule > kCenteredClipping)
        return 102;
    if (a.rule == kCenteredClipping && (a.f < 0 || 2 * a.f >= a.n || a.iterations < 1 || a.iterations > kMaxIterations || !(a.tau > 0.f) ||
                                        !std::isfinite(a.tau) || !a.center))
        return 116;
    if (a.rule == kGeoMedian && (a.f < 0 || 2 * a.f >= a.n || a.iterations < 1 || a.iterations > kMaxIterations || !(a.nu > 0.f) || !std::isfinite(a.nu)))
        return 115;
    if ((a.rule == kTrimmedMean || a.rule == kMda) && (a.f < 0 || 2 * a.f >= a.n))
        return a.rule == kTrimmedMean ? 112 : 113;
    if (a.rule == kMda) {
        long long sets = 1;   // C(n, f), exact while it stays below the bound
        for (int t = 0; t < a.f && sets <= kMdaMaxSets; ++t)
            sets = sets * (a.n - t) / (t + 1);
        if (sets > kMdaMaxSets)
            return 113;
    }
    if ((a.rule == kKrum || a.rule == kBulyan) && (a.n - a.f - 2 < 1 || a.m < 1 || a.m > a.n))
        return 103;
    if (a.rule == kBulyan && (a.n < 4 * a.f + 3 || a.beta != a.n - 4 * a.f - 2 || a.m < a.n - 2 * a.f - 2))
        return 104;
    if (a.rule == kAveragedMedian && (a.beta < 1 || a.beta > a.n))
        return 105;
    for (int i = 0; i < a.n; ++i)
        a.grad[i] = reinterpret_cast<float const*>(ptrs[i]);
    a.agg_out = reinterpret_cast<float*>(ptrs[32]);
    a.param = reinterpret_cast<float*>(ptrs[33]);
    a.slot0 = reinterpret_cast<float*>(ptrs[34]);
    a.slot1 = reinterpret_cast<float*>(ptrs[35]);
    a.param_mc = reinterpret_cast<float*>(ptrs[36]);
    a.cta_partials = reinterpret_cast<float*>(ptrs[37]);
    a.staging = reinterpret_cast<float*>(ptrs[38]);
    a.dist_out = reinterpret_cast<float*>(ptrs[39]);
    a.info = reinterpret_cast<int*>(ptrs[40]);
    a.grad_mc = reinterpret_cast<float const*>(ptrs[41]);
    a.epoch_ptr = reinterpret_cast<uint32_t*>(ptrs[42]);
    a.hyper_ptr = reinterpret_cast<float const*>(ptrs[43]);
    a.seg_partials = reinterpret_cast<float*>(ptrs[44]);
    a.loss_in = reinterpret_cast<float const*>(ptrs[45]);
    a.loss_out = reinterpret_cast<float*>(ptrs[46]);
    for (int q = 0; q < a.R; ++q) {
        a.param_dst[q] = reinterpret_cast<float*>(ptrs[48 + q]);
        a.signal[q] = reinterpret_cast<uint32_t*>(ptrs[64 + q]);
        a.mailbox[q] = reinterpret_cast<float*>(ptrs[80 + q]);
        a.param_bf16_dst[q] = reinterpret_cast<__nv_bfloat16*>(ptrs[96 + q]);
    }
    if (a.opt != kNone && (!a.param || (!a.param_mc && !a.param_dst[0])))
        return 106;
    if ((a.opt == kAdam || a.opt == kRmsprop || a.opt == kAdadelta) && (!a.slot0 || !a.slot1))
        return 107;
    if (a.opt == kAdagrad && !a.slot0)
        return 107;
    if ((a.rule == kKrum || a.rule == kBulyan || a.rule == kMda || a.rule == kGeoMedian || a.rule == kCenteredClipping) && (!a.cta_partials || !a.mailbox[0]))
        return 108;
    if ((a.rule == kGeoMedian || a.rule == kCenteredClipping) && a.R > 1 && !a.staging)
        return 108;   // the passes after the first re-read the staged copy instead of the peers' rows
    if (a.first_seg > 0 && !a.seg_partials)
        return 108;
    if (a.R > 1 && !a.signal[0])
        return 109;
    if (a.n > kBlockRows && a.R > 1 && (a.rule == kKrum || a.rule == kBulyan || a.rule == kMda) && !a.staging)
        return 110;   // blocked passes over remote rows need the staged copy
    return 0;
}

} // namespace

extern "C" {

char const* agb_op_list() {
    return "gar_fused,gar_phase_a,gar_max_ctas,gar_byzantine,sgd,worker_momentum,drop_chunks,checksum,cast_bf16";
}

// Wall-clock bound (seconds, 0 = none) of the cross-GPU flag waits of this library's kernels.
int agb_gar_set_flag_timeout(double seconds) {
    return set_flag_timeout(seconds);
}

// Upper bound of the grid the fused kernel may use (to size `cta_partials`: [ctas][496] floats).
int agb_gar_max_ctas() {
    int device = 0, sms = 0;
    if (cudaGetDevice(&device) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess)
        return 0;
    return sms * 4;
}

// Sizes of the per-rank communication regions (bytes): signal pad, mailbox.
int agb_gar_region_bytes(long long* out) {
    out[0] = static_cast<long long>(kFlagSlots) * kMaxRanks * 4;
    out[1] = static_cast<long long>(kMaxRanks) * (kMaxPairs + 1) * 4;
    return 0;
}

// The finish kernel (whole aggregation when nothing was pre-accumulated). See `fill_args` for the argument layout.
int agb_gar_fused(unsigned long long const* ptrs, int const* ints, long long const* longs, float const* floats, void* stream) {
    GarArgs a{};
    int const status = fill_args(a, ptrs, ints, longs, floats);
    if (status)
        return status;
    int const max_ctas = ints[9];
    long long total = 0;
    for (int s = 0; s < a.nseg; ++s)
        total += a.seg_hi[s] - a.seg_lo[s];
    if (total == 0 && a.R == 1)
        return 0;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (a.n <= 8)
        return launch<8, 4>(a, max_ctas, s);
    if (a.n <= 16)
        return launch<16, 4>(a, max_ctas, s);
    return launch<32, 1>(a, max_ctas, s);
}

// Phase A (partial pairwise distances + local staging) of owned segment `seg` alone, on `ctas` CTAs: launched on a side stream as soon as
// the backward pass has produced that bucket of gradients; the finish kernel is then called with first_seg > seg.
int agb_gar_phase_a(unsigned long long const* ptrs, int const* ints, long long const* longs, float const* floats, int seg, void* stream) {
    GarArgs a{};
    int const status = fill_args(a, ptrs, ints, longs, floats);
    if (status)
        return status;
    int const ctas = ints[15];
    if (seg < 0 || seg >= a.nseg || ctas < 1 || ctas > a.seg_max_ctas || !a.seg_partials || (a.rule != kKrum && a.rule != kBulyan && a.rule != kMda))
        return 111;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    // small CTAs: a 64-thread CTA (8 K registers, 13 KB of static shared memory) fits beside a persistent GEMM CTA of the backward pass
    // (320 threads x 168 registers, ~198 KB), so the distance pass shares SMs with it instead of taking them away
    int threads = ints[24] >= 32 && ints[24] <= 256 ? (ints[24] / 32) * 32 : 64;
    if (a.n <= kBlockRows)
        gar_phase_a_kernel<false><<<ctas, threads, 0, s>>>(a, seg);
    else
        gar_phase_a_kernel<true><<<ctas, threads < 64 ? 64 : threads, 0, s>>>(a, seg);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

// Omniscient Byzantine rows (ALIE: mode 0, coef = z; IPM: mode 1, coef = epsilon) over this rank's owned segments; see
// `gar_byzantine_kernel`. `rows`: n row addresses; `honest` / `byzantine`: disjoint slot masks; `signals`: R signal pads (R > 1);
// flags use *epoch_ptr + 1 when `epoch_ptr` is set, `epoch` otherwise. Collective when R > 1: every rank calls it.
int agb_gar_byzantine(unsigned long long const* rows, int n, long long const* seg_lo, long long const* seg_hi, int nseg, unsigned honest,
                      unsigned byzantine, int mode, float coef, int R, int rank, unsigned long long const* signals, unsigned epoch,
                      unsigned long long epoch_ptr, void* stream) {
    if (n < 1 || n > kMaxWorkers || R < 1 || R > kMaxRanks || rank < 0 || rank >= R)
        return 100;
    if (nseg < 1 || nseg > kMaxSeg)
        return 101;
    unsigned const all = n == 32 ? 0xffffffffu : (1u << n) - 1u;
    int const H = __builtin_popcount(honest), K = __builtin_popcount(byzantine);
    if ((honest & byzantine) || (honest & ~all) || (byzantine & ~all) || K < 1 || H < (mode == kAlie ? 2 : 1) || (mode != kAlie && mode != kIpm))
        return 114;
    ByzArgs a{};
    a.H = H;
    a.K = K;
    for (int i = 0, h = 0, b = 0; i < n; ++i) {
        a.rows[i] = reinterpret_cast<float*>(rows[i]);
        if ((honest >> i) & 1u)
            a.honest[h++] = i;
        if ((byzantine >> i) & 1u)
            a.byz[b++] = i;
    }
    a.mode = mode;
    a.coef = coef;
    a.nseg = nseg;
    long long work = 0;
    for (int s = 0; s < nseg; ++s) {
        a.seg_lo[s] = seg_lo[s];
        a.seg_hi[s] = seg_hi[s];
        if ((seg_lo[s] & 3) || (seg_hi[s] & 3) || seg_hi[s] < seg_lo[s])
            return 101;
        work += (seg_hi[s] - seg_lo[s]) / 4;
    }
    a.R = R;
    a.rank = rank;
    for (int q = 0; q < R; ++q) {
        a.signal[q] = reinterpret_cast<uint32_t*>(signals ? signals[q] : 0ull);
        if (R > 1 && !a.signal[q])
            return 109;
    }
    a.epoch = epoch;
    a.epoch_ptr = reinterpret_cast<uint32_t*>(epoch_ptr);
    if (work == 0 && R == 1)
        return 0;
    int const threads = 256;
    long long grid = (work + threads - 1) / threads;
    long long const cap = static_cast<long long>(agb::sm_count()) * 8;
    grid = grid < 1 ? 1 : grid > cap ? cap : grid;   // at least one CTA: a rank without owned coordinates still signals its peers
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (H <= kBlockRows)
        gar_byzantine_kernel<kBlockRows><<<static_cast<int>(grid), threads, 0, s>>>(a);
    else
        gar_byzantine_kernel<0><<<static_cast<int>(grid), threads, 0, s>>>(a);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

int agb_sgd(void* p, void const* g, float lr, long long d, void* stream) {
    if (d & 3)
        return 101;
    int blocks = static_cast<int>((d / 4 + 255) / 256);
    if (blocks > agb::sm_count() * 8)
        blocks = agb::sm_count() * 8;
    if (blocks > 0)
        sgd_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<float*>(p), static_cast<float const*>(g), lr, d);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

// Worker momentum over `w` rows of `d` fp32 elements: G rows `g_stride` elements apart, M rows `m_stride` apart (see
// `worker_momentum_kernel`). float4 accesses when d, both strides and both base addresses allow them, scalar ones otherwise.
int agb_worker_momentum(void* g, long long g_stride, void* m, long long m_stride, long long w, long long d, float beta, float c, void* stream) {
    if (w < 0 || w > 65535 || d < 0 || g_stride < d || m_stride < d || ((!g || !m) && w > 0 && d > 0))
        return 101;
    if (w == 0 || d == 0)
        return 0;
    bool const vec = (d % 4 == 0) && (g_stride % 4 == 0) && (m_stride % 4 == 0) && (reinterpret_cast<uintptr_t>(g) % 16 == 0) &&
                     (reinterpret_cast<uintptr_t>(m) % 16 == 0);
    long long const items = vec ? d / 4 : d;
    long long blocks = (items + 255) / 256;
    long long const cap = (static_cast<long long>(agb::sm_count()) * 8 + w - 1) / w;   // about 8 CTAs per SM over all the rows
    if (blocks > cap)
        blocks = cap;
    dim3 const grid(static_cast<unsigned>(blocks), static_cast<unsigned>(w));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (vec)
        worker_momentum_kernel<4><<<grid, 256, 0, s>>>(static_cast<float*>(g), g_stride, static_cast<float*>(m), m_stride, d, beta, c);
    else
        worker_momentum_kernel<1><<<grid, 256, 0, s>>>(static_cast<float*>(g), g_stride, static_cast<float*>(m), m_stride, d, beta, c);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

int agb_drop_chunks(void* g, void const* previous, long long d, long long chunk_bytes, float rate, int mode, unsigned long long seed, void* stream) {
    if (chunk_bytes < 4 || (mode == 2 && !previous))
        return 101;
    int blocks = static_cast<int>((d + 255) / 256);
    if (blocks > agb::sm_count() * 8)
        blocks = agb::sm_count() * 8;
    if (blocks > 0)
        drop_chunks_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<float*>(g), static_cast<float const*>(previous), d, chunk_bytes / 4, rate, mode, seed);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

int agb_checksum(void const* p, long long d, void* out, void* stream) {
    AGB_CUDA_OK(cudaMemsetAsync(out, 0, 8, static_cast<cudaStream_t>(stream)));
    int blocks = static_cast<int>((d + 255) / 256);
    if (blocks > agb::sm_count() * 4)
        blocks = agb::sm_count() * 4;
    if (blocks > 0)
        checksum_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<float const*>(p), d, static_cast<unsigned long long*>(out));
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

int agb_cast_bf16(void const* src, void* dst, long long d, void* stream) {
    if (d & 3)
        return 101;
    int blocks = static_cast<int>((d / 4 + 255) / 256);
    if (blocks > agb::sm_count() * 8)
        blocks = agb::sm_count() * 8;
    if (blocks > 0)
        cast_bf16_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<float const*>(src), static_cast<__nv_bfloat16*>(dst), d);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

} // extern "C"
