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
//                    one warp: Krum scores / Bulyan iterative selection, or the whole grid: MDA's minimum-diameter search or
//                    SMEA's smallest-largest-eigenvalue search (replicated on all ranks); phase D: aggregate the owned coordinates (mean of selected / coordinate-wise
//                    trimmed mean / median / NaN-aware mean), apply the optimizer,
//                    store the new parameters into every rank's buffer (P2P stores or one NVLS multimem.st); exit barrier
//                    geometric median / centered clipping instead: T + 1 passes over the owned coordinates, with one exchange of
//                    the n row distances per iteration (see `iterative_rule`)
//
// Nearest-neighbour mixing (NNM, `a.mix`) runs inside the finish kernel before any rule: raw distance pass (staging every row) and
// exchange, one selection warp, then every row of the staged tile is replaced by the mean of its n - f nearest rows; the rule then
// reads the mixed tile (see `nnm_pre_aggregation`). Adaptive robust clipping (ARC, bit kMixArc of `a.mix`) runs before NNM: a norm pass
// (staging every row), one exchange of the squared norms, one selection warp, then the clipped rows of the tile are rescaled in
// place (see `arc_pre_aggregation`). Bucketing (bit kMixBucketing, alone) runs first: the n_rows gathered rows are shuffled by a keyed
// permutation and replaced by the n = ceil(n_rows / s) means of buckets of s rows, staged as rows [0, n) of the tile; the rule then
// reads n rows (see `bucketing_pre_aggregation`). Its "buckets" are sets of rows, not the gradient buckets (coordinate segments) above.
// Attacked steps with an omniscient attack (ALIE / IPM) run `gar_byzantine_kernel` first: each rank crafts its owned coordinates of
// every Byzantine row from the honest values. Min-Max / Min-Sum run `gar_optimized_kernel` instead: a statistics pass, one exchange of
// whole-vector sums between the ranks, then the same per-coordinate write. Mimic runs `gar_mimic_warmup_kernel` (two exchanges) during
// its warm-up and `gar_mimic_copy_kernel` after it. Fang et al.'s Krum attack runs `gar_fang_krum_kernel` (Min-Max's passes and exchange,
// then a one-warp search over gamma), their trimmed-mean attack `gar_fang_trim_kernel` (one pass, a counter-based draw per row).
// DnC (rule kDnc) has a finish kernel of its own, `gar_dnc_kernel`: a sampled distance pass, one exchange, a float64 Jacobi per CTA,
// then Krum's phase D (see `dnc_selection`). FLTrust (rule kFltrust) too, `gar_fltrust_kernel`: a pass for the sums against the root
// gradient, one exchange, float64 coefficients, then the weighted sum. FoolsGold (rule kFoolsgold) too, `gar_foolsgold_kernel`: a pass
// that updates the per-worker histories and sums their products, one exchange, float64 coefficients, then FLTrust's weighted sum.
// With R = 1 the finish kernel alone is the stand-alone `[n, d] -> [d]` aggregation op. n <= 32 workers: up to 8 rows are held in
// registers at a time; more rows are processed in 8-row blocks (diagonal + cross passes over the staged copy).
// Step-varying scalars (flag epoch, learning rate, optimizer hyper-parameters) may be read from device memory so that the
// launches can be captured once in a CUDA graph.
// Ordering convention: finite ascending, non-finite last, ties -> lower worker index.

#include <cmath>
#include <cstring>

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
constexpr int kSlotMix = kSlotGeoMedian + kMaxIterations;   // NNM: exchange of the raw distances
constexpr int kSlotCraftStats = kSlotMix + 1;   // Min-Max / Min-Sum: exchange of the crafting statistics
constexpr int kSlotDnc = kSlotCraftStats + 1;   // DnC: exchange of the sampled distances
constexpr int kSlotArc = kSlotDnc + 1;   // ARC: exchange of the squared row norms
constexpr int kSlotMimic = kSlotArc + 1;   // mimic: second exchange of a warm-up step (the first one signals on kSlotCraftStats)
constexpr int kSlotFltrust = kSlotMimic + 1;   // FLTrust: exchange of the sums
constexpr int kSlotFoolsgold = kSlotFltrust + 1;   // FoolsGold: exchange of the sums and bad-row flags
constexpr int kFlagSlots = kSlotFoolsgold + 1;
constexpr int kMailboxRegion = kMaxRanks * (kMaxPairs + 1);  // floats of one mailbox region: [0] the rule's exchanges, [1] NNM's
// Min-Max / Min-Sum statistics of one rank: [0, kMaxPairs) honest pair distances D_jk | [kStatA, +32) A_i | [kStatB, +32) B_i | [kStatC] C.
// They travel through mailbox region 2 (float offset kCraftRegion, kMaxRanks x kCraftStats floats), after the two regions above.
constexpr int kStatA = kMaxPairs, kStatB = kStatA + kMaxWorkers, kStatC = kStatB + kMaxWorkers;
constexpr int kCraftStats = kStatC + 1;   // 561
constexpr int kCraftRegion = 2 * kMailboxRegion;
// mimic's posts in the same region 2 (one rank's kCraftStats floats): exchange 1 the s_i at [kMimicS, +32), exchange 2 the q_i at
// [kMimicQ, +32) and ||y||^2 at [kMimicY]; its `stats_out` (float64) adds 1 / ||y|| at [kMimicY + 1]
constexpr int kMimicS = 0, kMimicQ = kMaxWorkers, kMimicY = 2 * kMaxWorkers;
constexpr int kMimicStats = kMimicY + 2;
constexpr int kDncIterations = 8;         // DnC: iterations T in [1, kDncIterations]
constexpr int kDncStride = kDncIterations * kMaxPairs + 1;   // DnC post of one rank: T x [kMaxPairs] sampled distances, then the loss
constexpr int kDncRegion = kCraftRegion + kMaxRanks * kCraftStats;   // mailbox region 3: kMaxRanks x kDncStride floats
constexpr int kArcStride = kMaxWorkers + 1;   // ARC post of one rank: the n partial squared norms, then the loss
constexpr int kArcRegion = kDncRegion + kMaxRanks * kDncStride;   // mailbox region 4: kMaxRanks x kArcStride floats
constexpr int kFltrustStride = 2 * kMaxWorkers + 2;   // FLTrust post of one rank: P_i [0, 32), N_i [32, 64), N0 [64], then the loss
constexpr int kFltrustRegion = kArcRegion + kMaxRanks * kArcStride;   // mailbox region 5: kMaxRanks x kFltrustStride floats
constexpr int kFoolsgoldSums = kMaxWorkers * (kMaxWorkers + 1) / 2;   // 528: FoolsGold's P_ij, i <= j (`sum_index`)
// FoolsGold post of one rank (and CTA partials): the sums [0, n (n + 1) / 2), the bad-row flags [kFoolsgoldSums, +32), then the loss
constexpr int kFoolsgoldStride = kFoolsgoldSums + kMaxWorkers + 1;
constexpr int kFoolsgoldRegion = kFltrustRegion + kMaxRanks * kFltrustStride;   // mailbox region 6: kMaxRanks x kFoolsgoldStride floats
constexpr int kMailboxFloats = kFoolsgoldRegion + kMaxRanks * kFoolsgoldStride;
constexpr int kFltrustOut = 3 * kMaxWorkers + 1;   // FLTrust's `fltrust_out`: P [0, 32), N [32, 64), N0 [64], a [65, 97)
// FoolsGold's `foolsgold_out`: the sums [0, n (n + 1) / 2), the bad flags [kFoolsgoldSums, +32), c [kFoolsgoldSums + 32, +32)
constexpr int kFoolsgoldOut = kFoolsgoldSums + 2 * kMaxWorkers;
constexpr int kMixNnm = 1, kMixArc = 2, kMixBucketing = 4;   // GarArgs::mix bits (bucketing is never combined with the others)
constexpr unsigned long long kBucketingTag = 0x42554B54ull;   // "BUKT": third input of bucketing's key; >= 8, never a DnC iteration
constexpr int kJacobiSweeps = 32;         // DnC: sweep budget of the cyclic Jacobi
constexpr double kJacobiTol = 1e-26;      // DnC: stop once sum_{i != j} B_ij^2 <= kJacobiTol * sum_i B_ii^2
constexpr int kBlockRows = 8;             // rows held in registers at a time

constexpr long long kMdaMaxSets = 1 << 20; // MDA enumerates the C(n, f) removal sets
constexpr long long kSmeaMaxSets = 1 << 14;   // SMEA runs one float64 Jacobi per removal set (`_ops.SMEA_MAX_SETS`)
enum Rule { kAverage = 0, kAverageNan = 1, kMedian = 2, kAveragedMedian = 3, kKrum = 4, kBulyan = 5, kTrimmedMean = 6, kMda = 7, kGeoMedian = 8,
           kCenteredClipping = 9, kDnc = 10, kSmea = 11, kFltrust = 12, kFoolsgold = 13 };
enum Opt { kNone = 0, kSgd = 1, kAdam = 2, kRmsprop = 3, kAdagrad = 4, kAdadelta = 5 };

struct GarArgs {
    int n, f, m, beta, rule;           // n: the rows the rule sees (with bucketing: the n = ceil(n_rows / bkt_size) bucket means)
    int n_rows;                        // the gathered rows grad[0, n_rows): n, or the rows bucketing reduces to n
    int bkt_size;                      // bucketing: rows per bucket s in [1, n_rows]
    unsigned long long bkt_seed;       // bucketing: seed of the permutation (its step key is DnC's: dnc_step / dnc_step_ptr)
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
    float* mailbox[kMaxRanks];         // 2 x [kMaxRanks][kMaxPairs + 1] partial distances (+ loss sum) of every rank; region 1: NNM
    uint32_t epoch;                    // immediate epoch, used when epoch_ptr is null
    uint32_t* epoch_ptr;               // device counter of completed steps: flags use *epoch_ptr + 1; the finish kernel increments it
    float* cta_partials;               // [grid][kMaxPairs]
    float* seg_partials;               // [kMaxSeg][seg_max_ctas][kMaxPairs]
    float* staging;                    // [n][owned length] or null
    float* dist_out;                   // optional [n * n] (geometric median, centered clipping: [iterations][n]); with NNM: of the mixed rows
    float* raw_dist_out;               // optional [n * n]: NNM's distances of the raw rows
    int* info;                         // optional [192]: selection masks for tests/diagnostics; [64, 64 + n): NNM masks;
                                       // bucketing: [128, 128 + n_rows) the permutation, [160, 160 + n) the bucket masks
    float const* loss_in;              // optional [nloss] local per-worker losses
    int nloss;
    float* loss_out;                   // [1]: total loss over all ranks (summed in rank order)
    int iterations;                    // geometric median, centered clipping: iterations T in [1, kMaxIterations]
    float nu;                          // geometric median: smoothing, finite and > 0
    float tau;                         // centered clipping: clipping radius, finite and > 0
    float* center;                     // centered clipping: [d] (local) center v, read and updated on the owned coordinates
    int mix;                           // pre-aggregation bits (need the staging buffer): kMixNnm nearest-neighbour mixing, kMixArc adaptive
                                       // robust clipping; both: ARC, then NNM
    float* arc_out;                    // optional [2n]: ARC's squared norms N, then its factors c
    // DnC (T = iterations)
    int dnc_r;                         // rows removed per iteration, r = floor(c f)
    long long dnc_b, dnc_domain;       // subsample b and sample domain D: b' = min(b, D) coordinates of [0, D) per iteration
    unsigned long long dnc_seed;
    long long dnc_step;                // step key (DnC, bucketing), used when dnc_step_ptr is null
    long long const* dnc_step_ptr;     // device step key (graph replay), or null
    float* dnc_scratch;                // [grid][kDncIterations][kMaxPairs] CTA partials, then the samples [T][n][b'4]
    double* smea_scratch;              // SMEA: one [m][m] slab per warp of the grid (m = n - f), the double-centred matrix of its set
    float const* root;                 // FLTrust: the root gradient r [d] (rank 0's, peer-mapped), read on the owned coordinates
    float* fltrust_out;                // FLTrust: optional [kFltrustOut] sums and coefficients, for tests
    float* history;                    // FoolsGold: the histories H [n][owned] (local, the staged tile's layout), updated in place
    float* foolsgold_out;              // FoolsGold: optional [kFoolsgoldOut] sums, flags and coefficients, for tests
    double confidence;                 // FoolsGold: kappa, finite and > 0
};

// the rows `phase_a_segment` reads in DnC's sampled pass: one segment [0, b'4) of the gathered samples of one iteration, no staging
struct SampleRows {
    int n, nseg;
    long long seg_lo[1], seg_hi[1];
    float const* grad[kMaxWorkers];
    float* staging;
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
        struct {                                          // SMEA
            unsigned binom[kMaxWorkers + 1][kMaxWorkers / 2 + 1];
            unsigned long long best[16][2];               // per-warp minimum keys (score key, set key)
        } smea;
        struct {                                          // geometric median, centered clipping: weights of the current iterate
            float beta[kMaxWorkers];                      // 1 / max(nu, sqrt(D_i)) (CC: the clipping factors c_i) of the kept rows
            float sum;                                    // geometric median: their sum, in ascending worker order
            unsigned mask;                                // kept rows; 0: no weights, the iterate is the median (CC: z_t is unchanged)
        } geo;
    };
    float scores[kMaxWorkers];
    float warp_partials[16][kBlockRows * kBlockRows];
    unsigned selmask[kMaxWorkers];   // Krum, MDA: [0]; Bulyan: one per round
    unsigned nnm_mask[kMaxWorkers];  // NNM: neighbourhood of every row (itself included); outlives the rule's phases
    float arc_c[kMaxWorkers];        // ARC: clipping factor of every row
    unsigned arc_clipped;            // ARC: the rows the clip pass rescales
    unsigned bkt_mask[kMaxWorkers];  // bucketing: members of every bucket
    unsigned char bkt_perm[kMaxWorkers];    // bucketing: the permutation pi
    unsigned char bkt_order[kMaxWorkers];   // bucketing: the rows bucket by bucket, ascending inside a bucket
    signed char bkt_last[kMaxWorkers];      // bucketing: at the last position of a bucket, its index; -1 elsewhere
    int selcount[kMaxWorkers];
    int theta;
    float hyper[4];
    uint32_t epoch;
};

// DnC's selection state, declared by `gar_dnc_kernel` alone (the other kernels' shared memory does not grow)
struct DncShared {
    double B[kMaxWorkers][kMaxWorkers + 1];       // double-centred Gram matrix of the m remaining rows
    double V[kMaxWorkers][kMaxWorkers + 1];       // Jacobi eigenvectors
    double rot[kMaxWorkers / 2][2];               // (c, s) of every pair of the current round
    double rmean[kMaxWorkers];
    double score[kMaxWorkers];                    // by worker; +inf for the rows dropped for non-finite distances
    double grand;
    int idx[kMaxWorkers];                         // the remaining rows, ascending
    unsigned remaining, keep;
    int converged;
    SampleRows rows;
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
template<class Args> __device__ __forceinline__ long long staged_offset(Args const& a, int seg) {
    long long off = 0;
    for (int s = 0; s < seg; ++s)
        off += a.seg_hi[s] - a.seg_lo[s];
    return off;
}
template<class Args> __device__ __forceinline__ long long owned_length(Args const& a) {
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
// binom[m][k] = C(m, k) for m <= 32, k <= 16 (whole CTA; the caller synchronises)
__device__ __forceinline__ void fill_binomials(unsigned (&binom)[kMaxWorkers + 1][kMaxWorkers / 2 + 1]) {
    constexpr int K = kMaxWorkers / 2 + 1;
    for (int p = threadIdx.x; p < (kMaxWorkers + 1) * K; p += blockDim.x) {
        int const m = p / K, k = p % K;
        unsigned long long c = 1;   // C(m, k) < 2^32 for m <= 32; every partial product is an exact binomial times (m - t)
        for (int t = 0; t < k && t < m; ++t)
            c = c * (m - t) / (t + 1);
        binom[m][k] = k > m ? 0u : static_cast<unsigned>(c);
    }
}

// the removal set of rank r among the f-subsets of [0, n) in colexicographic order (= ascending masks): the combinatorial number
// system, r = sum_k C(c_k, k), c_f > ... > c_1
__device__ __forceinline__ unsigned unrank_removal(unsigned const (&binom)[kMaxWorkers + 1][kMaxWorkers / 2 + 1], int n, int f, long long r) {
    unsigned removed = 0;
    long long rest = r;
    for (int k = f; k >= 1; --k) {
        int c = n - 1;
        while (binom[c][k] > rest)
            --c;
        removed |= 1u << c;
        rest -= binom[c][k];
    }
    return removed;
}

// Gosper's hack: the next mask with as many bits as `removed` (removed != 0)
__device__ __forceinline__ unsigned next_removal(unsigned removed) {
    unsigned const low = removed & (0u - removed), up = removed + low;
    return (((up ^ removed) >> 2) >> (__ffs(low) - 1)) | up;
}

__device__ void select_mda(GarArgs const& a, Shared& sh, cg::grid_group& grid) {
    int const n = a.n, f = a.f, npairs = n * (n - 1) / 2;
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    fill_binomials(sh.mda.binom);
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
        unsigned removed = unrank_removal(sh.mda.binom, n, f, r);
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
            removed = next_removal(removed);
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

__device__ __forceinline__ float dot4(float4 const& u, float4 const& v) {
    return (u.x * v.x + u.y * v.y) + (u.z * v.z + u.w * v.w);
}

// FoolsGold's history row `row` at owned float4 `v` of a segment at staged offset `soff` (the history has the staged tile's layout)
template<class Args> __device__ __forceinline__ float4* history_at(Args const& a, int row, long long owned, long long soff, long long v) {
    return reinterpret_cast<float4*>(a.history + row * owned + soff + (v << 2));
}

// FoolsGold's first touch of row `row` at coordinate x: load g (P2P), stage it when a tile is given, add its finite values to the
// history (one fp32 add each), store the history back and return it; a non-finite value sets bit `row` of `bad`
template<class Args>
__device__ __forceinline__ float4 update_history(Args const& a, int row, long long x, long long owned, long long soff, long long v, unsigned& bad) {
    float4 const g = ld_stream_f4(a.grad[row] + x);
    if (a.staging)
        *reinterpret_cast<float4*>(a.staging + row * owned + soff + (v << 2)) = g;
    float4* const hp = history_at(a, row, owned, soff, v);
    float4 h = *hp;
    bool const fx = is_finite(g.x), fy = is_finite(g.y), fz = is_finite(g.z), fw = is_finite(g.w);
    h.x = fx ? __fadd_rn(h.x, g.x) : h.x;
    h.y = fy ? __fadd_rn(h.y, g.y) : h.y;
    h.z = fz ? __fadd_rn(h.z, g.z) : h.z;
    h.w = fw ? __fadd_rn(h.w, g.w) : h.w;
    *hp = h;
    if (!(fx && fy && fz && fw))
        bad |= 1u << row;
    return h;
}

// index of the sum (i <= j) in the row-major upper triangle of an n x n matrix, diagonal included
__device__ __forceinline__ int sum_index(int i, int j, int n) {
    return i * n - (i * (i - 1)) / 2 + (j - i);
}

// STAGED_ONLY (NNM's distances of the mixed rows): every pass, block 0's diagonal included, reads the staged tile and stores nothing.
// PRODUCTS (FoolsGold's sums, `gar_foolsgold_kernel`): the same blocks and folds over the histories H_i (`a.history`, [n][owned] in the
// staged tile's layout), with the products <H_i, H_j> for i <= j in place of the squared differences: a diagonal pass also has the
// pairs i == j, indexed by `sum_index`. The first touch of a row (block 0's diagonal pass, the cross passes (0, b)) is
// `update_history`; every later pass re-reads the updated history, which the same thread wrote (every pass maps (tid, 4) alike).
// `Args`: GarArgs, or ByzArgs for the honest distances of Min-Max (n, grad, staging and the segments, as GarArgs names them).
template<bool CROSS, bool STAGED_ONLY = false, bool PRODUCTS = false, class Args>
__device__ void phase_a_segment(Args const& a, Shared& sh, int* pair_of, int seg, float* out, long long tid, long long nthreads,
                                unsigned* bad = nullptr) {
    constexpr int B = kBlockRows, NPB = PRODUCTS ? B * (B + 1) / 2 : B * (B - 1) / 2;
    int const n = a.n, nb = CROSS ? (n + B - 1) / B : 1;
    long long const lo = a.seg_lo[seg], len4 = (a.seg_hi[seg] - lo) >> 2;
    long long const owned = owned_length(a), soff = staged_offset(a, seg);
    auto staged = [&](int row, long long v) { return a.staging + row * owned + soff + (v << 2); };
    for (int bi = 0; bi < nb; ++bi) {
        int const i0 = bi * B;
        bool const from_copy = STAGED_ONLY || (a.staging != nullptr && bi > 0);   // blocks >= 1 were staged by the cross passes (0, b)
        if (threadIdx.x < NPB) {   // local pair index -> (i, j) -> global pair index
            int i = 0, rest = threadIdx.x;
            while (rest >= B - (PRODUCTS ? 0 : 1) - i) {
                rest -= B - (PRODUCTS ? 0 : 1) - i;
                ++i;
            }
            int const j = i + (PRODUCTS ? 0 : 1) + rest;
            pair_of[threadIdx.x] = i0 + j < n ? (PRODUCTS ? sum_index(i0 + i, i0 + j, n) : pair_index(i0 + i, i0 + j, n)) : -1;
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
                    if (i0 + i < n) {
                        if constexpr (PRODUCTS)
                            g[i] = bi > 0 ? *history_at(a, i0 + i, owned, soff, v) : update_history(a, i0 + i, x, owned, soff, v, *bad);
                        else
                            g[i] = from_copy ? *reinterpret_cast<float4 const*>(staged(i0 + i, v)) : ld_stream_f4(a.grad[i0 + i] + x);
                    } else {
                        g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                }
                if (!PRODUCTS && a.staging && !from_copy) {
#pragma unroll
                    for (int i = 0; i < B; ++i)
                        if (i0 + i < n)
                            *reinterpret_cast<float4*>(staged(i0 + i, v)) = g[i];
                }
                int p = 0;
#pragma unroll
                for (int i = 0; i < B - (PRODUCTS ? 0 : 1); ++i) {
#pragma unroll
                    for (int j = i + (PRODUCTS ? 0 : 1); j < B; ++j, ++p)
                        if (i0 + j < n)
                            acc[p] += PRODUCTS ? dot4(g[i], g[j]) : sq_dist(g[i], g[j]);
                }
            }
            fold_pass<NPB>(sh, acc, out, pair_of);
        }
        if (CROSS) {
            for (int bj = bi + 1; bj < nb; ++bj) {
                int const j0 = bj * B;
                bool const j_from_copy = STAGED_ONLY || (a.staging != nullptr && bi > 0);   // first touch of block bj is the pass (0, bj)
                if (threadIdx.x < B * B) {
                    int const i = threadIdx.x / B, j = threadIdx.x % B;
                    pair_of[threadIdx.x] = (i0 + i < n && j0 + j < n) ? (PRODUCTS ? sum_index(i0 + i, j0 + j, n) : pair_index(i0 + i, j0 + j, n)) : -1;
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
                        if (i0 + i < n) {
                            if constexpr (PRODUCTS)
                                gi[i] = *history_at(a, i0 + i, owned, soff, v);
                            else
                                gi[i] = a.staging ? *reinterpret_cast<float4 const*>(staged(i0 + i, v)) : ld_stream_f4(a.grad[i0 + i] + x);
                        } else {
                            gi[i] = make_float4(0.f, 0.f, 0.f, 0.f);
                        }
                    }
#pragma unroll
                    for (int j = 0; j < B; ++j) {
                        if (j0 + j < n) {
                            if constexpr (PRODUCTS) {
                                gj[j] = bi > 0 ? *history_at(a, j0 + j, owned, soff, v) : update_history(a, j0 + j, x, owned, soff, v, *bad);
                            } else if (j_from_copy) {
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
                            acc[i * B + j] += PRODUCTS ? dot4(gi[i], gj[j]) : sq_dist(gi[i], gj[j]);
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

// ---- exchange of the pair distances: `cta_partials` (+ the pre-accumulated segments) -> every rank -> `sh.dist` ------------- //
// Fixed order: pre-accumulated segments [0, first_seg) (ascending, their CTAs ascending), then this kernel's CTAs, then ranks
// (ascending) => bit-identical matrix (and total loss) on every rank and in every CTA. `region`: float offset of the mailbox region,
// `slot`: flag slot of this exchange; the rank's loss sum travels with the distances. Non-finite distances become +inf.
__device__ void exchange_distances(GarArgs const& a, Shared& sh, cg::grid_group& grid, uint32_t epoch, int first_seg, int region, int slot,
                                   float local_loss, float* dist_out) {
    int const n = a.n, npairs = n * (n - 1) / 2;
    bool const multi = a.R > 1;
    __threadfence();
    grid.sync();
    if (blockIdx.x == 0) {
        for (int p = threadIdx.x; p < npairs; p += blockDim.x) {
            float s = 0.f;
            for (int seg = 0; seg < first_seg; ++seg)
                for (int b = 0; b < a.seg_ctas[seg]; ++b)
                    s += ld_volatile_f(a.seg_partials + (static_cast<long long>(seg) * a.seg_max_ctas + b) * kMaxPairs + p);
            for (unsigned b = 0; b < gridDim.x; ++b)
                s += ld_volatile_f(a.cta_partials + static_cast<long long>(b) * kMaxPairs + p);
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][region + a.rank * (kMaxPairs + 1) + p] = s;
        }
        if (threadIdx.x == 0)
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][region + a.rank * (kMaxPairs + 1) + kMaxPairs] = local_loss;
        fence_sys();
        __syncthreads();
        if (multi)
            signal_all(a, slot, epoch);
    }
    if (multi) {
        wait_all(a, slot, epoch);
        __syncthreads();
    } else {
        grid.sync();
    }
    // -------- full distance matrix (rank order => identical everywhere) -------- //
    for (int p = threadIdx.x; p < kMaxWorkers * (kMaxWorkers + 1); p += blockDim.x)
        (&sh.dist[0][0])[p] = 0.f;
    __syncthreads();
    float const* const box = a.mailbox[a.rank] + region;
    for (int p = threadIdx.x; p < npairs; p += blockDim.x) {
        int i = 0, rest = p;
        while (rest >= n - 1 - i) { // pair index -> (i, j) of the upper triangle
            rest -= n - 1 - i;
            ++i;
        }
        int const j = i + 1 + rest;
        float s = 0.f;
        for (int q = 0; q < a.R; ++q)
            s += ld_volatile_f(box + q * (kMaxPairs + 1) + p);
        if (!is_finite(s))
            s = __int_as_float(0x7f800000);
        sh.dist[i][j] = s;
        sh.dist[j][i] = s;
        if (dist_out && blockIdx.x == 0) {
            dist_out[i * n + j] = s;
            dist_out[j * n + i] = s;
        }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss_out) {
        float total = 0.f;
        for (int q = 0; q < a.R; ++q)
            total += ld_volatile_f(box + q * (kMaxPairs + 1) + kMaxPairs);
        *a.loss_out = total;
    }
    __syncthreads();
}

// ---- nearest-neighbour mixing (Allouah et al., "Fixing by Mixing", AISTATS 2023) ------------------------------------------ //
// D_ij = ||x_i - x_j||^2 (non-finite -> +inf); N_i = {i} and the n - f - 1 rows j != i first under the ordering convention;
// y_i = (((x_a0 + x_a1) + x_a2) + ...) / (n - f), the members of N_i in ascending worker order from +0, every operation rounded once.
//   1. raw distance pass over all owned segments: the rows cross NVLink once and land in the staged tile (block 0's diagonal and the
//      cross passes (0, b) store every row they load; after ARC, which staged and clipped every row, a STAGED_ONLY pass over the
//      tile, behind a grid barrier); exchange through mailbox region 1 and flag slot kSlotMix, which no other
//      exchange of the step touches (every CTA of every rank reads them, so a later exchange could not safely reuse them); the loss
//      travels with it;
//   2. warp 0 of every CTA builds the n masks from sh.dist (identical everywhere, so are the masks);
//   3. mix pass, in place on the staged tile: a thread loads the n raw values of a coordinate, then stores its n mixed values over
//      them. It uses the rules' own mapping (tid, VEC): a coordinate-wise or iterative rule's thread reads back only what it wrote
//      itself, so no grid barrier follows; the distance rules add one before their own pass over the mixed tile.
template<int N, int VEC>
__device__ __forceinline__ void nnm_pre_aggregation(GarArgs const& a, Shared& sh, int* pair_of, cg::grid_group& grid, uint32_t epoch,
                                                    float local_loss, long long tid, long long nthreads) {
    int const n = a.n, npairs = n * (n - 1) / 2;
    float* mine = a.cta_partials + static_cast<long long>(blockIdx.x) * kMaxPairs;
    for (int p = threadIdx.x; p < npairs; p += blockDim.x)
        mine[p] = 0.f;
    __syncthreads();
    for (int seg = 0; seg < a.nseg; ++seg) {
        if (a.mix & kMixArc)   // after ARC the rows are staged (and clipped): the distances of the tile
            phase_a_segment<(N > kBlockRows), true>(a, sh, pair_of, seg, mine, tid, nthreads);
        else
            phase_a_segment<(N > kBlockRows)>(a, sh, pair_of, seg, mine, tid, nthreads);
    }
    exchange_distances(a, sh, grid, epoch, 0, kMailboxRegion, kSlotMix, local_loss, a.raw_dist_out);
    if (threadIdx.x < 32) {
        int const lane = threadIdx.x, keep = n - a.f - 1;
        if (lane < n) {
            unsigned mask = 1u << lane;
            for (int j = 0; j < n; ++j) {
                if (j == lane)
                    continue;
                int rank = 0;
                for (int k = 0; k < n; ++k)
                    if (k != lane && k != j)
                        rank += before(sh.dist[lane][k], k, sh.dist[lane][j], j) ? 1 : 0;
                if (rank < keep)
                    mask |= 1u << j;
            }
            sh.nnm_mask[lane] = mask;
            if (a.info && blockIdx.x == 0)
                a.info[64 + lane] = static_cast<int>(mask);
        }
    }
    __syncthreads();
    long long const owned = owned_length(a);
    float const count = static_cast<float>(n - a.f);
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC, soff = staged_offset(a, seg);
        for (long long v = tid; v < lenv; v += nthreads) {
            float* const tile = a.staging + soff + v * VEC;
            float g[N][VEC];
#pragma unroll
            for (int i = 0; i < N; ++i) {
                if (i < n) {
                    V<VEC>::load(tile + i * owned, g[i]);
                } else {
#pragma unroll
                    for (int c = 0; c < VEC; ++c)
                        g[i][c] = 0.f;
                }
            }
#pragma unroll
            for (int c = 0; c < VEC; ++c) {   // a component's n raw values are all read before any of them is replaced
                float y[N];
#pragma unroll
                for (int i = 0; i < N; ++i) {
                    unsigned const mask = i < n ? sh.nnm_mask[i] : 0u;
                    float s = 0.f;
#pragma unroll
                    for (int j = 0; j < N; ++j)
                        if ((mask >> j) & 1u)
                            s = __fadd_rn(s, g[j][c]);
                    y[i] = __fdiv_rn(s, count);
                }
#pragma unroll
                for (int i = 0; i < N; ++i)
                    g[i][c] = y[i];
            }
#pragma unroll
            for (int i = 0; i < N; ++i)
                if (i < n)
                    V<VEC>::store(tile + i * owned, g[i]);
        }
    }
}

// ---- adaptive robust clipping (ARC; Allouah et al., "Boosting Robustness by Clipping Gradients in Distributed Learning") ------- //
// k = floor(2 f (n - f) / n); N_i = ||x_i||^2 (fp32); the k rows last under the ordering convention (by N) are clipped to the norm of
// the row at position n - k - 1, C = sqrt_rn(N_thr): c_i = 1 if s_i <= C else C / s_i (s_i = sqrt_rn(N_i), centered clipping's
// factor with radius C), y_i = x_i * c_i, one rounding each. c_i = 1 for every row when k = 0 or C is not finite.
//   1. norm pass over all owned segments, with the rules' (tid, VEC) mapping: the rows cross NVLink once and land in the staged tile,
//      N_i accumulates in registers (one FMA per value, as centered clipping's D_i);
//   2. lanes -> warps -> CTA -> `cta_partials` -> grid barrier; block 0 folds the CTAs in order and posts the rank's partials and its
//      loss into mailbox region 4 of every rank, then signals slot kSlotArc. Every CTA of every rank reads region 4 after the wait, so
//      no later exchange of the step may reuse it; the next write into it comes from the next step's ARC exchange, which a rank
//      reaches only after every rank's exit barrier of this step, hence after every CTA has finished reading;
//   3. warp 0 of every CTA sums the R posts in rank order and selects (identical everywhere): sh.arc_c, sh.arc_clipped;
//   4. clip pass, in place on the staged tile over the clipped rows only, with the same (tid, VEC) mapping: a coordinate-wise or
//      iterative rule's thread reads back only values it staged and clipped itself, so no grid barrier follows; the distance rules,
//      DnC's gather and NNM add one.
template<int N, int VEC>
__device__ __forceinline__ void arc_pre_aggregation(GarArgs const& a, Shared& sh, cg::grid_group& grid, uint32_t epoch, float local_loss,
                                                    long long tid, long long nthreads) {
    int const n = a.n, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    bool const multi = a.R > 1;
    long long const owned = owned_length(a);
    float acc[N];
#pragma unroll
    for (int i = 0; i < N; ++i)
        acc[i] = 0.f;
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC, soff = staged_offset(a, seg);
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * VEC;
#pragma unroll
            for (int i0 = 0; i0 < N; i0 += kBlockRows) {   // 8 rows in flight at a time: the pass stays within the rules' register budget
                float g[kBlockRows][VEC];
#pragma unroll
                for (int i = 0; i < kBlockRows; ++i)
                    if (i0 + i < n)
                        V<VEC>::load_stream(a.grad[i0 + i] + x, g[i]);
#pragma unroll
                for (int i = 0; i < kBlockRows; ++i) {
                    if (i0 + i < n) {
                        V<VEC>::store(a.staging + (i0 + i) * owned + soff + v * VEC, g[i]);
#pragma unroll
                        for (int c = 0; c < VEC; ++c)
                            acc[i0 + i] = __fmaf_rn(g[i][c], g[i][c], acc[i0 + i]);
                    }
                }
            }
        }
    }
    // -------- exchange of the n partial squared norms (and the loss) -------- //
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
    if (blockIdx.x == 0) {
        if (threadIdx.x < n) {
            float s = 0.f;
            for (unsigned b = 0; b < gridDim.x; ++b)
                s += ld_volatile_f(a.cta_partials + static_cast<long long>(b) * kMaxPairs + threadIdx.x);
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kArcRegion + a.rank * kArcStride + threadIdx.x] = s;
        }
        if (threadIdx.x == 0)
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kArcRegion + a.rank * kArcStride + kMaxWorkers] = local_loss;
        fence_sys();
        __syncthreads();
        if (multi)
            signal_all(a, kSlotArc, epoch);
    }
    if (multi) {
        wait_all(a, kSlotArc, epoch);
        __syncthreads();
    } else {
        grid.sync();
    }
    // -------- selection: warp 0 of every CTA -------- //
    if (warp == 0) {
        float const* const box = a.mailbox[a.rank] + kArcRegion;
        float N2 = 0.f;
        if (lane < n)
            for (int q = 0; q < a.R; ++q)
                N2 += ld_volatile_f(box + q * kArcStride + lane);
        int const k = (2 * a.f * (n - a.f)) / n;
        int rank = 0;
        for (int j = 0; j < n; ++j) {
            float const Nj = __shfl_sync(0xffffffffu, N2, j);
            if (j != lane)
                rank += before(Nj, j, N2, lane) ? 1 : 0;
        }
        unsigned const thr = __ballot_sync(0xffffffffu, lane < n && rank == n - k - 1);
        float const C = __fsqrt_rn(__shfl_sync(0xffffffffu, N2, __ffs(thr) - 1));
        bool const clipped = lane < n && k > 0 && is_finite(C) && rank >= n - k;
        float const s = __fsqrt_rn(N2);
        float const c = clipped ? (s <= C ? 1.f : __fdiv_rn(C, s)) : 1.f;
        sh.arc_c[lane] = c;
        unsigned const mask = __ballot_sync(0xffffffffu, clipped);
        if (lane == 0)
            sh.arc_clipped = mask;
        if (blockIdx.x == 0) {
            if (a.arc_out && lane < n) {
                a.arc_out[lane] = N2;
                a.arc_out[n + lane] = c;
            }
            if (lane == 0 && a.loss_out) {
                float total = 0.f;
                for (int q = 0; q < a.R; ++q)
                    total += ld_volatile_f(box + q * kArcStride + kMaxWorkers);
                *a.loss_out = total;
            }
        }
    }
    __syncthreads();
    // -------- clip pass over the clipped rows of the staged tile -------- //
    unsigned const mask = sh.arc_clipped;
    if (mask == 0u)
        return;
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC, soff = staged_offset(a, seg);
        for (long long v = tid; v < lenv; v += nthreads) {
            float* const tile = a.staging + soff + v * VEC;
#pragma unroll
            for (int i = 0; i < N; ++i) {
                if ((mask >> i) & 1u) {
                    float const c = sh.arc_c[i];
                    float y[VEC];
                    V<VEC>::load(tile + i * owned, y);
#pragma unroll
                    for (int e = 0; e < VEC; ++e)
                        y[e] = __fmul_rn(y[e], c);
                    V<VEC>::store(tile + i * owned, y);
                }
            }
        }
    }
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
// second grid barrier takes the place of the flags. The loss travels through the exit barrier, as for the coordinate-wise rules
// (with a pre-aggregation: through its exchange). After a pre-aggregation, pass 0 reads the staged tile too (mixed or clipped), with
// the mix and clip passes' mapping (same thread).
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
        bool const from_rows = !a.staging || (t == 0 && !a.mix);   // NNM, ARC: every pass reads the pre-aggregated tile
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
                        if (from_rows) {
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

// ---- divide-and-conquer (DnC; Shejwalkar & Houmansadr, "Manipulating the Byzantine", NDSS 2021) ----------------------------- //
// Iteration t < T of step `step` samples b' = min(b, D) distinct coordinates s_k = P(k) of [0, D), P a keyed permutation: a 4-round
// Feistel network on w bits (w the smallest even number >= max(2, bit length of D - 1), halves of h = w / 2 bits), round function
// F_r(R) = splitmix64(K ^ (r << 48) ^ R) mod 2^h with K = splitmix64(splitmix64(splitmix64(seed) ^ step) ^ t), cycle-walked into
// [0, D). D^t_ij = sum_k (x_i[s_k] - x_j[s_k])^2 (fp32). The rows with the most non-finite distances to the other remaining rows are
// dropped one at a time (the highest index first) until every remaining distance is finite; they score +inf. The m remaining rows
// score u_i^2, u the top eigenvector of B = -1/2 (D_ij - r_i - r_j + g) (classical double centring, float64), which ranks them as the
// paper's <x_i - mu, v>^2 = lambda_1 u_i^2 does. Iteration t keeps the n - r rows first under the ordering convention; the output is
// the mean of the rows every iteration kept (Krum's phase D).
//   1. gather: every thread evaluates P for its share of the T b'4 sample slots and copies the n values of the slots this rank owns
//      (P2P from the rows, or the mixed tile under NNM) into the compact scratch [T][n][b'4]; other slots hold +0, which adds exactly +0
//      to every distance;
//   2. grid barrier, then `phase_a_segment` over the scratch of every iteration, folded into the CTA's [T][kMaxPairs] partials;
//   3. one exchange: block 0 adds the CTA partials in index order and posts them with the loss into mailbox region 3 of every rank
//      (flag slot kSlotDnc, touched by no other exchange of the step); every CTA adds the R posts in rank order;
//   4. every CTA runs the same selection (same bits everywhere): a float64 cyclic Jacobi with round-robin pair ordering, every operation
//      rounded once (explicit _rn intrinsics: no FMA), which `_ops.dnc_scores` transcribes bit for bit.
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__device__ __forceinline__ long long dnc_permute(unsigned long long key, int h, long long domain, long long x) {
    unsigned long long const mask = (1ull << h) - 1ull;
    unsigned long long y = static_cast<unsigned long long>(x);
    do {
        unsigned long long L = y >> h, R = y & mask;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            unsigned long long const F = splitmix64(key ^ (static_cast<unsigned long long>(r) << 48) ^ R) & mask;
            unsigned long long const next = L ^ F;
            L = R;
            R = next;
        }
        y = (L << h) | R;
    } while (y >= static_cast<unsigned long long>(domain));
    return static_cast<long long>(y);
}

// ---- bucketing (Karimireddy, He & Jaggi, "Byzantine-Robust Learning on Heterogeneous Datasets via Bucketing", ICLR 2022) -------- //
// K = splitmix64(splitmix64(splitmix64(seed) ^ step) ^ kBucketingTag); pi starts as the identity and, for i = n_rows - 1 down to 1,
// pi[i] and pi[j] swap with j = splitmix64(K ^ i) mod (i + 1). Bucket b < n = ceil(n_rows / s) holds pi[b s], ..., pi[min((b + 1) s,
// n_rows) - 1]; y_b = (((x_a0 + x_a1) + ...) / |M_b|, its members in ascending worker order from +0, every operation rounded once
// (NNM's mixing arithmetic).
//   1. warp 0 of every CTA builds pi, the masks and the order in which the mean pass visits the rows (identical everywhere: the key is
//      the same on every CTA and every rank). No exchange: a bucket mean is per coordinate, and the loss keeps its usual path;
//   2. mean pass over all owned segments, with the rules' (tid, VEC) mapping (the instance is the rule's, chosen from n): the rows
//      are visited bucket by bucket, 8 loads in flight, into one running sum that is divided and stored as staging row b at the last member of bucket b. Every raw row
//      crosses NVLink once; only the n means are staged. A coordinate-wise or iterative rule's thread reads back only what it stored
//      itself, so no grid barrier follows; the distance rules and DnC's gather add one.
template<int N, int VEC>
__device__ __forceinline__ void bucketing_pre_aggregation(GarArgs const& a, Shared& sh, long long tid, long long nthreads) {
    int const nr = a.n_rows, s = a.bkt_size;
    if (threadIdx.x < 32) {
        int const lane = threadIdx.x;
        unsigned long long const step = static_cast<unsigned long long>(a.dnc_step_ptr ? *a.dnc_step_ptr : a.dnc_step);
        unsigned long long const key = splitmix64(splitmix64(splitmix64(a.bkt_seed) ^ step) ^ kBucketingTag);
        // the swap partner of every i, computed in parallel; the swaps themselves are sequential
        unsigned long long const i = static_cast<unsigned long long>(lane);
        int const partner = lane >= 1 && lane < nr ? static_cast<int>(splitmix64(key ^ i) % (i + 1ull)) : 0;
        if (lane < nr)
            sh.bkt_perm[lane] = static_cast<unsigned char>(lane);
        __syncwarp();
        for (int k = nr - 1; k >= 1; --k) {
            int const j = __shfl_sync(0xffffffffu, partner, k);
            if (lane == 0) {
                unsigned char const t = sh.bkt_perm[k];
                sh.bkt_perm[k] = sh.bkt_perm[j];
                sh.bkt_perm[j] = t;
            }
            __syncwarp();
        }
        if (lane < nr)
            sh.bkt_last[lane] = -1;
        __syncwarp();
        int const nb = a.n;
        if (lane < nb) {
            int const lo = lane * s, hi = lo + s < nr ? lo + s : nr;
            unsigned mask = 0u;
            for (int p = lo; p < hi; ++p)
                mask |= 1u << sh.bkt_perm[p];
            sh.bkt_mask[lane] = mask;
            int p = lo;
            for (unsigned rest = mask; rest != 0u; rest &= rest - 1u)
                sh.bkt_order[p++] = static_cast<unsigned char>(__ffs(rest) - 1);
            sh.bkt_last[hi - 1] = static_cast<signed char>(lane);
            if (a.info && blockIdx.x == 0)
                a.info[160 + lane] = static_cast<int>(mask);
        }
        if (a.info && blockIdx.x == 0 && lane < nr)
            a.info[128 + lane] = sh.bkt_perm[lane];
    }
    __syncthreads();
    long long const owned = owned_length(a);
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC, soff = staged_offset(a, seg);
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * VEC;
            float* const tile = a.staging + soff + v * VEC;
            float acc[VEC];
#pragma unroll
            for (int c = 0; c < VEC; ++c)
                acc[c] = 0.f;
            // 8 rows in flight at a time, in a loop over the n_rows gathered rows: the instance N only bounds the rule's n rows
            for (int p0 = 0; p0 < nr; p0 += kBlockRows) {
                float g[kBlockRows][VEC];
#pragma unroll
                for (int p = 0; p < kBlockRows; ++p)
                    if (p0 + p < nr)
                        V<VEC>::load_stream(a.grad[sh.bkt_order[p0 + p]] + x, g[p]);
#pragma unroll
                for (int p = 0; p < kBlockRows; ++p) {
                    if (p0 + p < nr) {
#pragma unroll
                        for (int c = 0; c < VEC; ++c)
                            acc[c] = __fadd_rn(acc[c], g[p][c]);
                        int const b = sh.bkt_last[p0 + p];
                        if (b >= 0) {
                            float const count = static_cast<float>(p0 + p + 1 - b * s);
#pragma unroll
                            for (int c = 0; c < VEC; ++c)
                                acc[c] = __fdiv_rn(acc[c], count);
                            V<VEC>::store(tile + b * owned, acc);
#pragma unroll
                            for (int c = 0; c < VEC; ++c)
                                acc[c] = 0.f;
                        }
                    }
                }
            }
        }
    }
}

__device__ __forceinline__ bool before_d(double a, int ia, double b, int ib) {
    bool const fa = isfinite(a), fb = isfinite(b);
    if (fa != fb)
        return fa;
    if (fa && a != b)
        return a < b;
    return ia < ib;
}

// the rotation (c, s) that zeroes B_pq != 0: tau = (B_qq - B_pp) / (2 B_pq), t = sign(tau) / (|tau| + sqrt(1 + tau^2)), c = 1 / sqrt(1 + t^2),
// s = t c, every operation rounded once (DnC's and SMEA's Jacobi, and `_ops.dnc_eigh`)
__device__ __forceinline__ void jacobi_rotation(double bpp, double bqq, double apq, double& c, double& s) {
    double const tau = __ddiv_rn(__dsub_rn(bqq, bpp), __dmul_rn(2.0, apq));
    double const t = __ddiv_rn(tau >= 0.0 ? 1.0 : -1.0, __dadd_rn(fabs(tau), __dsqrt_rn(__dadd_rn(1.0, __dmul_rn(tau, tau)))));
    c = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(1.0, __dmul_rn(t, t))));
    s = __dmul_rn(t, c);
}

// eigenvectors of ds.B[0, m)^2 (m >= 2) into ds.V; B ends (nearly) diagonal. A sweep is m' - 1 rounds (m' = m rounded up to
// even) of m' / 2 disjoint pairs (circle method: position 0 fixed, the others rotated); a round computes every pair's rotation from
// B as it stands, then rotates the rows, then the columns of B and V, then zeroes B_pq and B_qp.
__device__ void dnc_jacobi(DncShared& ds, int m) {
    int const mm = m + (m & 1), half = mm / 2;
    auto player = [&](int pos, int round) { return pos == 0 ? 0 : 1 + (pos - 1 + round) % (mm - 1); };
    for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
        if (threadIdx.x == 0) {
            double off = 0.0, diag = 0.0;
            for (int i = 0; i < m; ++i)
                for (int j = 0; j < m; ++j) {
                    double const sq = __dmul_rn(ds.B[i][j], ds.B[i][j]);
                    if (i == j)
                        diag = __dadd_rn(diag, sq);
                    else
                        off = __dadd_rn(off, sq);
                }
            ds.converged = off <= __dmul_rn(kJacobiTol, diag);
        }
        __syncthreads();
        if (ds.converged)
            break;
        for (int round = 0; round < mm - 1; ++round) {
            if (threadIdx.x < half) {
                int const u = player(threadIdx.x, round), v = player(mm - 1 - threadIdx.x, round);
                int const p = u < v ? u : v, q = u < v ? v : u;
                double c = 1.0, s = 0.0;
                if (q < m && ds.B[p][q] != 0.0)
                    jacobi_rotation(ds.B[p][p], ds.B[q][q], ds.B[p][q], c, s);
                ds.rot[threadIdx.x][0] = c;
                ds.rot[threadIdx.x][1] = s;
            }
            __syncthreads();
            for (int task = threadIdx.x; task < half * m; task += blockDim.x) {   // rows p, q of B
                int const k = task / m, j = task % m;
                int const u = player(k, round), v = player(mm - 1 - k, round);
                int const p = u < v ? u : v, q = u < v ? v : u;
                if (q < m) {
                    double const c = ds.rot[k][0], s = ds.rot[k][1], bp = ds.B[p][j], bq = ds.B[q][j];
                    ds.B[p][j] = __dsub_rn(__dmul_rn(c, bp), __dmul_rn(s, bq));
                    ds.B[q][j] = __dadd_rn(__dmul_rn(s, bp), __dmul_rn(c, bq));
                }
            }
            __syncthreads();
            for (int task = threadIdx.x; task < half * m; task += blockDim.x) {   // columns p, q of B and V
                int const k = task / m, i = task % m;
                int const u = player(k, round), v = player(mm - 1 - k, round);
                int const p = u < v ? u : v, q = u < v ? v : u;
                if (q < m) {
                    double const c = ds.rot[k][0], s = ds.rot[k][1];
                    double const bp = ds.B[i][p], bq = ds.B[i][q], vp = ds.V[i][p], vq = ds.V[i][q];
                    ds.B[i][p] = __dsub_rn(__dmul_rn(c, bp), __dmul_rn(s, bq));
                    ds.B[i][q] = __dadd_rn(__dmul_rn(s, bp), __dmul_rn(c, bq));
                    ds.V[i][p] = __dsub_rn(__dmul_rn(c, vp), __dmul_rn(s, vq));
                    ds.V[i][q] = __dadd_rn(__dmul_rn(s, vp), __dmul_rn(c, vq));
                }
            }
            __syncthreads();
            if (threadIdx.x < half) {
                int const u = player(threadIdx.x, round), v = player(mm - 1 - threadIdx.x, round);
                int const p = u < v ? u : v, q = u < v ? v : u;
                if (q < m) {
                    ds.B[p][q] = 0.0;
                    ds.B[q][p] = 0.0;
                }
            }
            __syncthreads();
        }
    }
}

// SMEA (every thread of the grid): the kept set S, |S| = m = n - f, whose double-centred matrix B_S = -1/2 (D_ij - r_i - r_j + g) (r_i
// the row means over S, g their mean, both added in ascending index) has the smallest largest eigenvalue; the score is the largest
// diagonal entry after the Jacobi of `dnc_jacobi` (same rounds, rotations, stop test and sweep budget; no eigenvectors), +inf for a set
// with a non-finite distance between two members, 0 for m = 1; ties -> the lexicographically smallest sorted index list. The C(n, f)
// removal sets are split over the warps of the grid, unranked and stepped as in `select_mda`; a warp keeps B_S in its own [m][m] slab of
// `smea_scratch` and runs every round warp-synchronously. Keys (the score's ordered bits with -0 -> +0 and non-finite -> +inf, then
// ~__brev(keep)) are exact, so their minimum does not depend on the reduction order. The per-CTA minima go through `cta_partials`;
// block 0 writes the winning score's bits to info[32, 34).
__device__ void select_smea(GarArgs const& a, Shared& sh, cg::grid_group& grid) {
    int const n = a.n, f = a.f, m = n - f, mm = m + (m & 1), half = mm / 2;
    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    unsigned const all = 0xffffffffu, full = n == 32 ? 0xffffffffu : (1u << n) - 1u;
    double const inf = __longlong_as_double(0x7ff0000000000000ll);
    fill_binomials(sh.smea.binom);
    __syncthreads();
    unsigned bad = 0u;   // lane i < n: the workers j with a non-finite D_ij
    if (lane < n)
        for (int j = 0; j < n; ++j)
            bad |= is_finite(sh.dist[lane][j]) ? 0u : 1u << j;
    long long const total = sh.smea.binom[n][f];
    long long const gwarps = static_cast<long long>(gridDim.x) * nwarps, gw = static_cast<long long>(blockIdx.x) * nwarps + warp;
    long long const per = (total + gwarps - 1) / gwarps;
    long long r = gw * per;
    long long const end = r + per < total ? r + per : total;
    double* const B = a.smea_scratch + gw * m * m;
    auto player = [&](int pos, int round) { return pos == 0 ? 0 : 1 + (pos - 1 + round) % (mm - 1); };
    unsigned long long best_score = ~0ull, best_set = ~0ull;
    if (r < end) {
        unsigned removed = unrank_removal(sh.smea.binom, n, f, r);
        for (;;) {
            unsigned const keep = full & ~removed;
            double score = 0.0;
            if (__any_sync(all, lane < n && ((keep >> lane) & 1u) && (bad & keep))) {
                score = inf;
            } else if (m >= 2) {
                int const i = lane < m ? static_cast<int>(__fns(keep, 0, lane + 1)) : 0;   // lane k < m: row k, the k-th kept worker
                double rmean = 0.0;
                if (lane < m) {
                    double sum = 0.0;
                    for (unsigned rest = keep; rest; rest &= rest - 1)
                        sum = __dadd_rn(sum, static_cast<double>(sh.dist[i][__ffs(rest) - 1]));
                    rmean = __ddiv_rn(sum, static_cast<double>(m));
                }
                double grand = 0.0;
                for (int k = 0; k < m; ++k)
                    grand = __dadd_rn(grand, __shfl_sync(all, rmean, k));
                grand = __ddiv_rn(grand, static_cast<double>(m));
                unsigned rest = keep;
                for (int j = 0; j < m; ++j, rest &= rest - 1) {
                    double const rj = __shfl_sync(all, rmean, j);
                    if (lane < m) {
                        double const dij = static_cast<double>(sh.dist[i][__ffs(rest) - 1]);
                        B[lane * m + j] = __dmul_rn(-0.5, __dadd_rn(__dsub_rn(__dsub_rn(dij, rmean), rj), grand));
                    }
                }
                __syncwarp();
                for (int sweep = 0; sweep < kJacobiSweeps; ++sweep) {
                    int converged = 0;
                    if (lane == 0) {
                        double off = 0.0, diag = 0.0;
                        for (int p = 0; p < m; ++p)
                            for (int q = 0; q < m; ++q) {
                                double const sq = __dmul_rn(B[p * m + q], B[p * m + q]);
                                if (p == q)
                                    diag = __dadd_rn(diag, sq);
                                else
                                    off = __dadd_rn(off, sq);
                            }
                        converged = off <= __dmul_rn(kJacobiTol, diag);
                    }
                    if (__shfl_sync(all, converged, 0))
                        break;
                    for (int round = 0; round < mm - 1; ++round) {
                        double c = 1.0, s = 0.0;   // lane k < m' / 2: the rotation of pair k, from B as it stands
                        if (lane < half) {
                            int const u = player(lane, round), v = player(mm - 1 - lane, round);
                            int const p = u < v ? u : v, q = u < v ? v : u;
                            if (q < m && B[p * m + q] != 0.0)
                                jacobi_rotation(B[p * m + p], B[q * m + q], B[p * m + q], c, s);
                        }
                        __syncwarp();
                        for (int base = 0; base < half * m; base += 32) {   // rows p, q
                            int const task = base + lane, k = task / m, j = task % m;
                            double const ck = __shfl_sync(all, c, k & 31), sk = __shfl_sync(all, s, k & 31);
                            int const u = player(k, round), v = player(mm - 1 - k, round);
                            int const p = u < v ? u : v, q = u < v ? v : u;
                            if (task < half * m && q < m) {
                                double const bp = B[p * m + j], bq = B[q * m + j];
                                B[p * m + j] = __dsub_rn(__dmul_rn(ck, bp), __dmul_rn(sk, bq));
                                B[q * m + j] = __dadd_rn(__dmul_rn(sk, bp), __dmul_rn(ck, bq));
                            }
                        }
                        __syncwarp();
                        for (int base = 0; base < half * m; base += 32) {   // columns p, q
                            int const task = base + lane, k = task / m, i2 = task % m;
                            double const ck = __shfl_sync(all, c, k & 31), sk = __shfl_sync(all, s, k & 31);
                            int const u = player(k, round), v = player(mm - 1 - k, round);
                            int const p = u < v ? u : v, q = u < v ? v : u;
                            if (task < half * m && q < m) {
                                double const bp = B[i2 * m + p], bq = B[i2 * m + q];
                                B[i2 * m + p] = __dsub_rn(__dmul_rn(ck, bp), __dmul_rn(sk, bq));
                                B[i2 * m + q] = __dadd_rn(__dmul_rn(sk, bp), __dmul_rn(ck, bq));
                            }
                        }
                        __syncwarp();
                        if (lane < half) {
                            int const u = player(lane, round), v = player(mm - 1 - lane, round);
                            int const p = u < v ? u : v, q = u < v ? v : u;
                            if (q < m) {
                                B[p * m + q] = 0.0;
                                B[q * m + p] = 0.0;
                            }
                        }
                        __syncwarp();
                    }
                }
                score = lane < m ? B[lane * (m + 1)] : -inf;   // the largest diagonal entry; a NaN wins
                for (int o = 16; o > 0; o >>= 1) {
                    double const other = __shfl_xor_sync(all, score, o);
                    score = (other > score || other != other) ? other : score;
                }
            }
            unsigned long long bits = !isfinite(score) ? 0x7ff0000000000000ull : score == 0.0 ? 0ull : static_cast<unsigned long long>(__double_as_longlong(score));
            unsigned long long const skey = (bits >> 63) ? ~bits : bits | (1ull << 63), set = ~__brev(keep);
            if (skey < best_score || (skey == best_score && set < best_set)) {
                best_score = skey;
                best_set = set;
            }
            if (++r >= end)
                break;
            removed = next_removal(removed);
        }
    }
    if (lane == 0) {
        sh.smea.best[warp][0] = best_score;
        sh.smea.best[warp][1] = best_set;
    }
    __syncthreads();
    unsigned long long* const slots = reinterpret_cast<unsigned long long*>(a.cta_partials);
    if (threadIdx.x == 0) {
        for (int w = 0; w < nwarps; ++w)
            if (sh.smea.best[w][0] < best_score || (sh.smea.best[w][0] == best_score && sh.smea.best[w][1] < best_set)) {
                best_score = sh.smea.best[w][0];
                best_set = sh.smea.best[w][1];
            }
        slots[static_cast<long long>(blockIdx.x) * (kMaxPairs / 2)] = best_score;
        slots[static_cast<long long>(blockIdx.x) * (kMaxPairs / 2) + 1] = best_set;
    }
    __threadfence();
    grid.sync();
    if (threadIdx.x == 0) {
        for (unsigned b = 0; b < gridDim.x; ++b) {
            unsigned long long volatile const* const slot = slots + static_cast<long long>(b) * (kMaxPairs / 2);
            unsigned long long const score = slot[0], set = slot[1];
            if (score < best_score || (score == best_score && set < best_set)) {
                best_score = score;
                best_set = set;
            }
        }
        sh.selmask[0] = __brev(~static_cast<unsigned>(best_set));
        sh.selcount[0] = m;
        sh.theta = 1;
        if (a.info && blockIdx.x == 0) {
            unsigned long long const bits = (best_score >> 63) ? best_score & ~(1ull << 63) : ~best_score;
            a.info[32] = static_cast<int>(static_cast<unsigned>(bits));
            a.info[33] = static_cast<int>(static_cast<unsigned>(bits >> 32));
        }
    }
}

// the rows iteration t keeps, from its distances in sh.dist (whole CTA; every thread returns the same mask)
__device__ unsigned dnc_keep(GarArgs const& a, Shared& sh, DncShared& ds) {
    int const n = a.n, lane = threadIdx.x & 31;
    unsigned const full = n == 32 ? 0xffffffffu : (1u << n) - 1u;
    if (threadIdx.x < 32) {   // drop the rows with the most non-finite distances, the highest index first
        unsigned bad = 0u;
        if (lane < n)
            for (int j = 0; j < n; ++j)
                bad |= is_finite(sh.dist[lane][j]) ? 0u : 1u << j;
        unsigned remaining = full;
        for (;;) {
            int count = lane < n && ((remaining >> lane) & 1u) ? __popc(bad & remaining) : 0;
            int most = count;
            for (int o = 16; o > 0; o >>= 1)
                most = max(most, __shfl_xor_sync(0xffffffffu, most, o));
            if (most == 0)
                break;
            unsigned const candidates = __ballot_sync(0xffffffffu, count == most);
            remaining &= ~(1u << (31 - __clz(candidates)));
        }
        if (lane == 0)
            ds.remaining = remaining;
        if (lane < n && ((remaining >> lane) & 1u))
            ds.idx[__popc(remaining & ((1u << lane) - 1u))] = lane;
        if (lane < n)
            ds.score[lane] = ((remaining >> lane) & 1u) ? 0.0 : __longlong_as_double(0x7ff0000000000000ll);
    }
    __syncthreads();
    int const m = __popc(ds.remaining);
    if (m >= 2) {
        if (threadIdx.x < m) {   // row means, ascending index
            int const i = ds.idx[threadIdx.x];
            double sum = 0.0;
            for (int j = 0; j < m; ++j)
                sum = __dadd_rn(sum, static_cast<double>(sh.dist[i][ds.idx[j]]));
            ds.rmean[threadIdx.x] = __ddiv_rn(sum, static_cast<double>(m));
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            double sum = 0.0;
            for (int i = 0; i < m; ++i)
                sum = __dadd_rn(sum, ds.rmean[i]);
            ds.grand = __ddiv_rn(sum, static_cast<double>(m));
        }
        __syncthreads();
        for (int e = threadIdx.x; e < m * m; e += blockDim.x) {
            int const i = e / m, j = e % m;
            double const dij = static_cast<double>(sh.dist[ds.idx[i]][ds.idx[j]]);
            ds.B[i][j] = __dmul_rn(-0.5, __dadd_rn(__dsub_rn(__dsub_rn(dij, ds.rmean[i]), ds.rmean[j]), ds.grand));
            ds.V[i][j] = i == j ? 1.0 : 0.0;
        }
        __syncthreads();
        dnc_jacobi(ds, m);
        if (threadIdx.x < m) {   // top eigenpair: the largest diagonal entry, ties -> lower column
            int best = 0;
            for (int k = 1; k < m; ++k)
                if (ds.B[k][k] > ds.B[best][best])
                    best = k;
            double const u = ds.V[threadIdx.x][best];
            ds.score[ds.idx[threadIdx.x]] = __dmul_rn(u, u);
        }
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        bool keep = false;
        if (lane < n) {
            int rank = 0;
            for (int j = 0; j < n; ++j)
                if (j != lane)
                    rank += before_d(ds.score[j], j, ds.score[lane], lane) ? 1 : 0;
            keep = rank < n - a.dnc_r;
        }
        unsigned const mask = __ballot_sync(0xffffffffu, keep);
        if (lane == 0)
            ds.keep = mask;
    }
    __syncthreads();
    unsigned const keep = ds.keep;
    __syncthreads();
    return keep;
}

template<int N>
__device__ void dnc_selection(GarArgs const& a, Shared& sh, DncShared& ds, int* pair_of, cg::grid_group& grid, uint32_t epoch,
                              float local_loss, long long tid, long long nthreads) {
    int const n = a.n, T = a.iterations, npairs = n * (n - 1) / 2;
    bool const multi = a.R > 1;
    long long const domain = a.dnc_domain, b = a.dnc_b < domain ? a.dnc_b : domain, b4 = (b + 3) & ~3ll;
    float* const partials = a.dnc_scratch;
    float* const samples = a.dnc_scratch + static_cast<long long>(gridDim.x) * kDncIterations * kMaxPairs;
    long long const owned = owned_length(a);
    unsigned long long const step = static_cast<unsigned long long>(a.dnc_step_ptr ? *a.dnc_step_ptr : a.dnc_step);
    int const width = 64 - __clzll(static_cast<unsigned long long>(domain - 1));
    int const h = (width < 2 ? 2 : width + (width & 1)) / 2;
    unsigned long long const base_key = splitmix64(splitmix64(a.dnc_seed) ^ step);
    // -------- 1. gather the owned samples -------- //
    for (long long k = tid; k < T * b4; k += nthreads) {
        int const t = static_cast<int>(k / b4);
        long long const slot = k - t * b4;
        float* const dst = samples + static_cast<long long>(t) * n * b4 + slot;
        long long x = -1, soff = 0;
        int seg = -1;
        if (slot < b) {
            x = dnc_permute(splitmix64(base_key ^ static_cast<unsigned long long>(t)), h, domain, slot);
            for (int s = 0; s < a.nseg; ++s) {
                if (x >= a.seg_lo[s] && x < a.seg_hi[s]) {
                    seg = s;
                    break;
                }
                soff += a.seg_hi[s] - a.seg_lo[s];
            }
        }
        for (int i = 0; i < n; ++i) {
            float value = 0.f;
            if (seg >= 0)
                value = a.mix ? a.staging[i * owned + soff + (x - a.seg_lo[seg])] : a.grad[i][x];
            dst[i * b4] = value;
        }
    }
    __threadfence();
    grid.sync();
    // -------- 2. sampled distances of every iteration -------- //
    float* const mine = partials + static_cast<long long>(blockIdx.x) * kDncIterations * kMaxPairs;
    for (int p = threadIdx.x; p < T * kMaxPairs; p += blockDim.x)
        mine[p] = 0.f;
    for (int t = 0; t < T; ++t) {
        if (threadIdx.x == 0) {
            ds.rows.n = n;
            ds.rows.nseg = 1;
            ds.rows.seg_lo[0] = 0;
            ds.rows.seg_hi[0] = b4;
            ds.rows.staging = nullptr;
        }
        if (threadIdx.x < n)
            ds.rows.grad[threadIdx.x] = samples + (static_cast<long long>(t) * n + threadIdx.x) * b4;
        __syncthreads();
        phase_a_segment<(N > kBlockRows)>(ds.rows, sh, pair_of, 0, mine + t * kMaxPairs, tid, nthreads);
    }
    // -------- 3. one exchange: T x npairs partial distances and the loss -------- //
    __threadfence();
    grid.sync();
    if (blockIdx.x == 0) {
        for (int k = threadIdx.x; k < T * npairs; k += blockDim.x) {
            int const t = k / npairs, p = k - t * npairs;
            float s = 0.f;
            for (unsigned c = 0; c < gridDim.x; ++c)
                s += ld_volatile_f(partials + static_cast<long long>(c) * kDncIterations * kMaxPairs + t * kMaxPairs + p);
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kDncRegion + a.rank * kDncStride + t * kMaxPairs + p] = s;
        }
        if (threadIdx.x == 0)
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kDncRegion + a.rank * kDncStride + kDncIterations * kMaxPairs] = local_loss;
        fence_sys();
        __syncthreads();
        if (multi)
            signal_all(a, kSlotDnc, epoch);
    }
    if (multi) {
        wait_all(a, kSlotDnc, epoch);
        __syncthreads();
    } else {
        grid.sync();
    }
    float const* const box = a.mailbox[a.rank] + kDncRegion;
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss_out) {
        float total = 0.f;
        for (int q = 0; q < a.R; ++q)
            total += ld_volatile_f(box + q * kDncStride + kDncIterations * kMaxPairs);
        *a.loss_out = total;
    }
    // -------- 4. selection, identical in every CTA of every rank -------- //
    unsigned good = n == 32 ? 0xffffffffu : (1u << n) - 1u;
    for (int t = 0; t < T; ++t) {
        for (int p = threadIdx.x; p < kMaxWorkers * (kMaxWorkers + 1); p += blockDim.x)
            (&sh.dist[0][0])[p] = 0.f;
        __syncthreads();
        for (int p = threadIdx.x; p < npairs; p += blockDim.x) {
            int i = 0, rest = p;
            while (rest >= n - 1 - i) {
                rest -= n - 1 - i;
                ++i;
            }
            int const j = i + 1 + rest;
            float s = 0.f;
            for (int q = 0; q < a.R; ++q)
                s += ld_volatile_f(box + q * kDncStride + t * kMaxPairs + p);
            if (!is_finite(s))
                s = __int_as_float(0x7f800000);
            sh.dist[i][j] = s;
            sh.dist[j][i] = s;
            if (a.dist_out && blockIdx.x == 0) {
                a.dist_out[(t * n + i) * n + j] = s;
                a.dist_out[(t * n + j) * n + i] = s;
            }
        }
        __syncthreads();
        unsigned const keep = dnc_keep(a, sh, ds);
        good &= keep;
        if (a.info && blockIdx.x == 0 && threadIdx.x == 0)
            a.info[96 + t] = static_cast<int>(keep);
    }
    if (threadIdx.x == 0) {
        sh.selmask[0] = good;
        sh.selcount[0] = __popc(good);
        sh.theta = 1;
    }
}

// ---- coordinate-wise rules: one streaming pass over the rows, or (STAGED, NNM / ARC) over the pre-aggregated tile, each thread
// reading what it wrote in the mix or clip pass ------------------------------------------------------------------------------ //
template<int N, int VEC, bool STAGED>
__device__ __forceinline__ void coordinate_rules(GarArgs const& a, float const (&hyper)[4], long long tid, long long nthreads) {
    int const n = a.n;
    long long const owned = STAGED ? owned_length(a) : 0;
    bool const in_switch = a.rule == kAverage && a.grad_mc != nullptr && !STAGED;
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC, soff = STAGED ? staged_offset(a, seg) : 0;
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * VEC;
            auto row = [&](int i) -> float const* { return STAGED ? a.staging + i * owned + soff + v * VEC : a.grad[i] + x; };
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
                                V<VEC>::load_stream(row(i), g[i]);
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
                            V<VEC>::load_stream(row(i), g);
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
                        V<VEC>::load_stream(row(i), g[i]);
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
    bool const distance_rule = a.rule == kKrum || a.rule == kBulyan || a.rule == kMda || a.rule == kSmea;
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

    if (a.mix) {
        if (a.mix & kMixBucketing) {
            bucketing_pre_aggregation<N, VEC>(a, sh, tid, nthreads);
            if (distance_rule) {
                __threadfence();
                grid.sync();   // the mean pass wrote the tile with the rule's (tid, VEC) mapping; distance passes read it by float4 blocks
            }
        }
        if (a.mix & kMixArc) {
            arc_pre_aggregation<N, VEC>(a, sh, grid, epoch, local_loss, tid, nthreads);
            if (distance_rule || (a.mix & kMixNnm)) {
                __threadfence();
                grid.sync();   // the clip pass wrote the tile with the rule's (tid, VEC) mapping; distance passes read it by float4 blocks
            }
        }
        if (a.mix & kMixNnm) {
            nnm_pre_aggregation<N, VEC>(a, sh, pair_of, grid, epoch, local_loss, tid, nthreads);
            if (distance_rule) {
                __threadfence();
                grid.sync();   // the mix pass wrote the tile with the rule's (tid, VEC) mapping; the distance pass reads it by float4 blocks
            }
        }
    }

    if (distance_rule) {
        // -------- phase A of the segments that were not pre-accumulated (pre-aggregation: of the staged tile) -------- //
        float* mine = a.cta_partials + static_cast<long long>(blockIdx.x) * kMaxPairs;
        for (int p = threadIdx.x; p < npairs; p += blockDim.x)
            mine[p] = 0.f;
        __syncthreads();
        for (int seg = a.first_seg; seg < a.nseg; ++seg) {
            if (a.mix)
                phase_a_segment<(N > kBlockRows), true>(a, sh, pair_of, seg, mine, tid, nthreads);
            else
                phase_a_segment<(N > kBlockRows)>(a, sh, pair_of, seg, mine, tid, nthreads);
        }
        // -------- full distance matrix + selection -------- //
        exchange_distances(a, sh, grid, epoch, a.first_seg, 0, kSlotExchange, local_loss, a.dist_out);
        if (a.rule == kMda) {
            select_mda(a, sh, grid);
        } else if (a.rule == kSmea) {
            select_smea(a, sh, grid);
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
                if (a.rule != kBulyan) {   // Krum, MDA, SMEA: mean of the selected rows
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
        if (a.mix)
            coordinate_rules<N, VEC, true>(a, hyper, tid, nthreads);
        else
            coordinate_rules<N, VEC, false>(a, hyper, tid, nthreads);
    }

    // the loss went through an exchange (distance rules, NNM, ARC); bucketing exchanges nothing
    bool const exchanged_loss = distance_rule || (a.mix & (kMixNnm | kMixArc));
    if (multi) { // exit barrier: all slices have landed on all ranks, gradient buffers are free again
        fence_sys();
        grid.sync();
        if (blockIdx.x == 0) {
            if (!exchanged_loss && threadIdx.x == 0) {   // steps without an exchange stage carry the loss through the exit barrier
                for (int q = 0; q < a.R; ++q)
                    a.mailbox[q][a.rank * (kMaxPairs + 1) + kMaxPairs] = local_loss;
                fence_sys();
            }
            __syncthreads();
            signal_all(a, kSlotExit, epoch);
            wait_all(a, kSlotExit, epoch);
            __syncthreads();
            if (!exchanged_loss && threadIdx.x == 0 && a.loss_out) {
                float total = 0.f;
                for (int q = 0; q < a.R; ++q)
                    total += ld_volatile_f(a.mailbox[a.rank] + q * (kMaxPairs + 1) + kMaxPairs);
                *a.loss_out = total;
            }
        }
    } else if (!exchanged_loss && blockIdx.x == 0 && threadIdx.x == 0 && a.loss_out) {
        *a.loss_out = local_loss;
    }
    if (a.epoch_ptr && blockIdx.x == 0 && threadIdx.x == 0)
        *a.epoch_ptr = epoch;   // this step is complete (every CTA read the counter before the barriers above)
}

// ---- the DnC finish kernel ------------------------------------------------------------- //
// The finish kernel of rule kDnc: the same steps as `gar_fused_kernel` (entry barrier, NNM, selection, Krum's phase D, exit barrier),
// with `dnc_selection` in place of the distance rules' phase A and selection. A kernel of its own keeps the sampled pass and the
// Jacobi out of the register allocation of the other rules' coordinate loops, and DncShared out of their shared memory.
template<int N, int VEC>
__global__ void __launch_bounds__(N <= 8 ? 512 : 256, 1) gar_dnc_kernel(GarArgs const a) {
    __shared__ Shared sh;
    __shared__ DncShared ds;
    __shared__ int pair_of[kBlockRows * kBlockRows];
    cg::grid_group grid = cg::this_grid();
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    bool const multi = a.R > 1;
    if (threadIdx.x == 0) {
        sh.epoch = current_epoch(a);
        for (int i = 0; i < 4; ++i)
            sh.hyper[i] = a.hyper_ptr ? a.hyper_ptr[i] : (i == 0 ? a.lr : i == 1 ? a.h0 : i == 2 ? a.h1 : a.h2);
    }
    __syncthreads();
    uint32_t const epoch = sh.epoch;
    float const hyper[4] = {sh.hyper[0], sh.hyper[1], sh.hyper[2], sh.hyper[3]};
    long long const owned = owned_length(a);
    if (multi) {   // entry barrier: every rank's gradients are published (nothing is pre-accumulated for DnC)
        if (blockIdx.x == 0)
            signal_all(a, 0, epoch);
        wait_all(a, 0, epoch);
        __syncthreads();
    }
    float local_loss = 0.f;
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss_in)
        for (int j = 0; j < a.nloss; ++j)
            local_loss += a.loss_in[j];
    if (a.mix) {
        if (a.mix & kMixBucketing)
            bucketing_pre_aggregation<N, VEC>(a, sh, tid, nthreads);
        if (a.mix & kMixArc) {
            arc_pre_aggregation<N, VEC>(a, sh, grid, epoch, local_loss, tid, nthreads);
            if (a.mix & kMixNnm) {
                __threadfence();
                grid.sync();   // the clip pass wrote the tile with the rule's (tid, VEC) mapping; NNM's distance pass reads float4 blocks
            }
        }
        if (a.mix & kMixNnm)
            nnm_pre_aggregation<N, VEC>(a, sh, pair_of, grid, epoch, local_loss, tid, nthreads);
        __threadfence();
        grid.sync();   // the mean, clip or mix pass wrote the tile with the rule's (tid, VEC) mapping; the gather reads any coordinate of it
    }
    dnc_selection<N>(a, sh, ds, pair_of, grid, epoch, local_loss, tid, nthreads);   // carries the loss
    __syncthreads();
    if (a.info && blockIdx.x == 0 && threadIdx.x == 0) {
        a.info[0] = 1;
        a.info[1] = static_cast<int>(sh.selmask[0]);
    }
    // -------- phase D: mean of the kept rows, update, broadcast (Krum's) -------- //
    unsigned const mask = sh.selmask[0];
    float const count = static_cast<float>(sh.selcount[0]);
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC, soff = staged_offset(a, seg);
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * VEC;
            float sum[VEC];
#pragma unroll
            for (int c = 0; c < VEC; ++c)
                sum[c] = 0.f;
            auto load_row = [&](int i, float (&dst)[VEC]) {
                if (a.staging)
                    V<VEC>::load(a.staging + i * owned + soff + v * VEC, dst);
                else
                    V<VEC>::load_stream(a.grad[i] + x, dst);
            };
            if (N <= 16) {   // all kept rows in flight at once, added in ascending worker order
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
                for (int i = 0; i < a.n; ++i) {
                    if ((mask >> i) & 1u) {
                        float g[VEC];
                        load_row(i, g);
#pragma unroll
                        for (int c = 0; c < VEC; ++c)
                            sum[c] += g[c];
                    }
                }
            }
            float out[VEC];
#pragma unroll
            for (int c = 0; c < VEC; ++c)
                out[c] = sum[c] / count;
            apply_update<VEC>(a, hyper, x, out);
        }
    }
    if (multi) {   // exit barrier, as in `gar_fused_kernel` (the loss went through DnC's exchange)
        fence_sys();
        grid.sync();
        if (blockIdx.x == 0) {
            __syncthreads();
            signal_all(a, kSlotExit, epoch);
            wait_all(a, kSlotExit, epoch);
            __syncthreads();
        }
    }
    if (a.epoch_ptr && blockIdx.x == 0 && threadIdx.x == 0)
        *a.epoch_ptr = epoch;   // this step is complete (every CTA read the counter before the barriers above)
}

// Phase D of FLTrust and FoolsGold: y = sum coef_i x_i from +0 in worker order (__fmul_rn / __fadd_rn: no FMA), the rows outside
// `mask` (coef_i = 0) skipped, then the optimizer and the parameter broadcast; the rows come from the staged tile, or from the rows
// themselves when R = 1 and n <= 8. Exit barrier as for DnC (the loss went through the kernel's exchange). `coef`: shared memory.
template<int N, int VEC>
__device__ __forceinline__ void weighted_phase_d(GarArgs const& a, cg::grid_group& grid, float const (&hyper)[4], float const* coef,
                                                 unsigned const mask, uint32_t const epoch, long long const tid, long long const nthreads) {
    int const n = a.n;
    bool const multi = a.R > 1;
    long long const owned = owned_length(a);
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
            float y[VEC];
#pragma unroll
            for (int c = 0; c < VEC; ++c)
                y[c] = 0.f;
            if (N <= 16) {   // every weighted row in flight at once, added in ascending worker order
                float g[N][VEC];
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if ((mask >> i) & 1u)
                        load_row(i, g[i]);
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if ((mask >> i) & 1u) {
                        float const ai = coef[i];
#pragma unroll
                        for (int c = 0; c < VEC; ++c)
                            y[c] = __fadd_rn(y[c], __fmul_rn(ai, g[i][c]));
                    }
            } else {
                for (int i = 0; i < n; ++i) {
                    if ((mask >> i) & 1u) {
                        float g[VEC];
                        load_row(i, g);
                        float const ai = coef[i];
#pragma unroll
                        for (int c = 0; c < VEC; ++c)
                            y[c] = __fadd_rn(y[c], __fmul_rn(ai, g[c]));
                    }
                }
            }
            apply_update<VEC>(a, hyper, x, y);
        }
    }
    if (multi) {   // exit barrier, as in `gar_dnc_kernel` (the loss went through the exchange)
        fence_sys();
        grid.sync();
        if (blockIdx.x == 0) {
            __syncthreads();
            signal_all(a, kSlotExit, epoch);
            wait_all(a, kSlotExit, epoch);
            __syncthreads();
        }
    }
    if (a.epoch_ptr && blockIdx.x == 0 && threadIdx.x == 0)
        *a.epoch_ptr = epoch;   // this step is complete (every CTA read the counter before the barriers above)
}

// ---- the FLTrust finish kernel (Cao, Fang, Liu & Gong, NDSS 2021) ---------------------------------------------------- //
// Rows x_i, root gradient r (rank 0's row, read over P2P on the owned coordinates). The arithmetic is `_ops.fltrust_coefficients`:
//   1. sums pass over the owned segments, with the rules' (tid, VEC) mapping: the n rows and r are loaded (8 rows in flight at a time,
//      as ARC's norm pass), P_i = <x_i, r>, N_i = ||x_i||^2 and N0 = ||r||^2 accumulate with one FMA per value; the rows are staged
//      when the staging tile is given (R > 1 or n > 8), so that the second pass never crosses NVLink again;
//   2. one exchange of the 2n + 1 partial sums and the loss: lanes -> warps -> CTA -> `cta_partials` -> grid barrier; block 0 folds
//      the CTAs in order and posts the rank's sums into mailbox region 5 of every rank, then signals slot kSlotFltrust. Every CTA of
//      every rank adds the R posts in rank order, so the sums are bit-identical everywhere. Region 5 and slot kSlotFltrust belong to
//      this exchange alone (FLTrust runs no pre-aggregation and no other exchange); every CTA reads region 5 before the exit barrier,
//      and the next write into it comes from the next step's exchange, which a rank reaches only after every rank's exit barrier;
//   3. the coefficients on warp 0 of every CTA (one lane per row), in float64 with explicit _rn intrinsics:
//        t_i = P_i / (sqrt(N_i) sqrt(N0)); TS_i = t_i if finite and > 0, else 0; S = sum TS_i in worker order;
//        a_i = fp32(((TS_i sqrt(N0)) / sqrt(N_i)) / S), every a_i = 0 when S = 0;
//   4. phase D: y = sum a_i x_i from +0 in worker order (__fmul_rn / __fadd_rn: no FMA), the rows with a_i = 0 skipped, then the
//      optimizer and the parameter broadcast; from the staged tile, or the local rows when R = 1 and n <= 8. Exit barrier as for DnC.
// A kernel of its own keeps the 2n + 1 accumulators out of the register allocation of `gar_fused_kernel`.
struct FltrustShared {
    float partials[16][2 * kMaxWorkers + 1];   // per-warp sums: P_i [0, n), N_i [n, 2n), N0 [2n]
    float coef[kMaxWorkers];                    // a_i
    unsigned mask;                              // rows with a_i != 0
    float hyper[4];
    uint32_t epoch;
};

template<int N, int VEC>
__global__ void __launch_bounds__(N <= 8 ? 512 : 256, 1) gar_fltrust_kernel(GarArgs const a) {
    __shared__ FltrustShared sh;
    cg::grid_group grid = cg::this_grid();
    int const n = a.n, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    bool const multi = a.R > 1;
    if (threadIdx.x == 0) {
        sh.epoch = current_epoch(a);
        for (int i = 0; i < 4; ++i)
            sh.hyper[i] = a.hyper_ptr ? a.hyper_ptr[i] : (i == 0 ? a.lr : i == 1 ? a.h0 : i == 2 ? a.h1 : a.h2);
    }
    __syncthreads();
    uint32_t const epoch = sh.epoch;
    float const hyper[4] = {sh.hyper[0], sh.hyper[1], sh.hyper[2], sh.hyper[3]};
    long long const owned = owned_length(a);
    if (multi) {   // entry barrier: every rank's gradients, and rank 0's root, are published (nothing is pre-accumulated)
        if (blockIdx.x == 0)
            signal_all(a, 0, epoch);
        wait_all(a, 0, epoch);
        __syncthreads();
    }
    float local_loss = 0.f;
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss_in)
        for (int j = 0; j < a.nloss; ++j)
            local_loss += a.loss_in[j];
    // -------- 1. sums pass -------- //
    float P[N], Q[N], R0 = 0.f;   // P_i, N_i, N0
#pragma unroll
    for (int i = 0; i < N; ++i) {
        P[i] = 0.f;
        Q[i] = 0.f;
    }
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / VEC, soff = staged_offset(a, seg);
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * VEC;
            float r[VEC];
            V<VEC>::load_stream(a.root + x, r);
#pragma unroll
            for (int c = 0; c < VEC; ++c)
                R0 = __fmaf_rn(r[c], r[c], R0);
#pragma unroll
            for (int i0 = 0; i0 < N; i0 += kBlockRows) {
                float g[kBlockRows][VEC];
#pragma unroll
                for (int i = 0; i < kBlockRows; ++i)
                    if (i0 + i < n)
                        V<VEC>::load_stream(a.grad[i0 + i] + x, g[i]);
#pragma unroll
                for (int i = 0; i < kBlockRows; ++i) {
                    if (i0 + i < n) {
                        if (a.staging)
                            V<VEC>::store(a.staging + (i0 + i) * owned + soff + v * VEC, g[i]);
#pragma unroll
                        for (int c = 0; c < VEC; ++c) {
                            P[i0 + i] = __fmaf_rn(g[i][c], r[c], P[i0 + i]);
                            Q[i0 + i] = __fmaf_rn(g[i][c], g[i][c], Q[i0 + i]);
                        }
                    }
                }
            }
        }
    }
    // -------- 2. exchange of the 2n + 1 sums (and the loss) -------- //
#pragma unroll
    for (int i = 0; i < N; ++i) {
        if (i < n) {
            float const p = warp_sum(P[i]), q = warp_sum(Q[i]);
            if (lane == 0) {
                sh.partials[warp][i] = p;
                sh.partials[warp][n + i] = q;
            }
        }
    }
    {
        float const r0 = warp_sum(R0);
        if (lane == 0)
            sh.partials[warp][2 * n] = r0;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 2 * n + 1; k += blockDim.x) {
        float s = 0.f;
        for (int w = 0; w < nwarps; ++w)
            s += sh.partials[w][k];
        a.cta_partials[static_cast<long long>(blockIdx.x) * kMaxPairs + k] = s;
    }
    __threadfence();
    grid.sync();
    if (blockIdx.x == 0) {
        for (int k = threadIdx.x; k < 2 * n + 1; k += blockDim.x) {
            float s = 0.f;
            for (unsigned b = 0; b < gridDim.x; ++b)
                s += ld_volatile_f(a.cta_partials + static_cast<long long>(b) * kMaxPairs + k);
            int const at = k < n ? k : k < 2 * n ? kMaxWorkers + (k - n) : 2 * kMaxWorkers;
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kFltrustRegion + a.rank * kFltrustStride + at] = s;
        }
        if (threadIdx.x == 0)
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kFltrustRegion + a.rank * kFltrustStride + 2 * kMaxWorkers + 1] = local_loss;
        fence_sys();
        __syncthreads();
        if (multi)
            signal_all(a, kSlotFltrust, epoch);
    }
    if (multi) {
        wait_all(a, kSlotFltrust, epoch);
        __syncthreads();
    } else {
        grid.sync();
    }
    // -------- 3. coefficients: warp 0 of every CTA -------- //
    if (warp == 0) {
        float const* const box = a.mailbox[a.rank] + kFltrustRegion;
        float Pi = 0.f, Ni = 0.f, N0 = 0.f;
        for (int q = 0; q < a.R; ++q) {
            if (lane < n) {
                Pi += ld_volatile_f(box + q * kFltrustStride + lane);
                Ni += ld_volatile_f(box + q * kFltrustStride + kMaxWorkers + lane);
            }
            N0 += ld_volatile_f(box + q * kFltrustStride + 2 * kMaxWorkers);
        }
        double const s0 = __dsqrt_rn(static_cast<double>(N0)), si = __dsqrt_rn(static_cast<double>(Ni));
        double const t = __ddiv_rn(static_cast<double>(Pi), __dmul_rn(si, s0));
        double const ts = (lane < n && isfinite(t) && t > 0.0) ? t : 0.0;
        double S = 0.0;
        for (int j = 0; j < n; ++j)
            S = __dadd_rn(S, __shfl_sync(0xffffffffu, ts, j));
        float const c = (S != 0.0 && ts > 0.0) ? __double2float_rn(__ddiv_rn(__ddiv_rn(__dmul_rn(ts, s0), si), S)) : 0.f;
        sh.coef[lane] = c;
        unsigned const mask = __ballot_sync(0xffffffffu, c != 0.f);
        if (lane == 0)
            sh.mask = mask;
        if (blockIdx.x == 0) {
            if (a.fltrust_out) {
                if (lane < n) {
                    a.fltrust_out[lane] = Pi;
                    a.fltrust_out[kMaxWorkers + lane] = Ni;
                    a.fltrust_out[2 * kMaxWorkers + 1 + lane] = c;
                }
                if (lane == 0)
                    a.fltrust_out[2 * kMaxWorkers] = N0;
            }
            if (lane == 0 && a.loss_out) {
                float total = 0.f;
                for (int q = 0; q < a.R; ++q)
                    total += ld_volatile_f(box + q * kFltrustStride + 2 * kMaxWorkers + 1);
                *a.loss_out = total;
            }
        }
    }
    __syncthreads();
    // -------- 4. phase D: weighted sum, update, broadcast -------- //
    weighted_phase_d<N, VEC>(a, grid, hyper, sh.coef, sh.mask, epoch, tid, nthreads);
}

// ---- the FoolsGold finish kernel (Fung, Yoon & Beschastnikh, RAID 2020) ------------------------------------------------- //
// Rows g_i, histories H_i (`a.history`: [n][owned], local, the staged tile's layout; they persist across steps and graph replays).
// The arithmetic is `_ops.foolsgold_coefficients`:
//   1. history pass over the owned segments: `phase_a_segment<.., PRODUCTS>`, Krum's 8-row blocks and folds with products in place of
//      squared differences. The first touch of a row loads g_i (P2P), stages it when the tile is given (R > 1 or n > 8, so that phase D
//      never crosses NVLink again), adds its finite values to H_i and stores H_i back; the n (n + 1) / 2 sums P_ij = <H_i, H_j>, i <= j,
//      of the updated histories land in the CTA's slot of `cta_partials` (kFoolsgoldStride floats), then the CTA's bad-row flags;
//   2. one exchange of the sums, the flags and the loss: grid barrier; block 0 folds the CTAs in order and posts the rank's values into
//      mailbox region 6 of every rank, then signals slot kSlotFoolsgold. Every CTA of every rank adds the R posts in rank order, so the
//      sums are bit-identical everywhere. Region 6 and slot kSlotFoolsgold belong to this exchange alone (FoolsGold runs no
//      pre-aggregation and no other exchange); every CTA reads region 6 before the exit barrier, and the next write into it comes from
//      the next step's exchange, which a rank reaches only after every rank's exit barrier;
//   3. the coefficients on warp 0 of every CTA (one lane per row, cs_ij recomputed from the sums where needed), in float64 with
//      explicit _rn intrinsics (the logarithm is CUDA's `log`, within 1 ulp):
//        cs_ij = P_ij / (sqrt(N_i) sqrt(N_j)), 0 for i == j, N_i or N_j zero or non-finite, or a non-finite quotient; v_i = max_j cs_ij;
//        pardoned (cs_ij v_i) / v_j when v_j > v_i; alpha_i = clip(1 - max_j cs_ij, 0, 1); all zero when max alpha = 0, otherwise
//        alpha / max alpha, 1 -> 0.99, clip(kappa (ln(alpha / (1 - alpha)) + 0.5), 0, 1); 0 for bad rows and non-finite N_i;
//        S = sum alpha_i in worker order; c_i = fp32(alpha_i / S), every c_i = 0 when S = 0;
//   4. FLTrust's phase D (`weighted_phase_d`): y = sum c_i g_i, the optimizer, the parameter broadcast, the exit barrier.
struct FoolsgoldShared {
    float coef[kMaxWorkers];   // c_i
    unsigned mask;             // rows with c_i != 0
    unsigned bad;              // the CTA's bad rows, then the step's
};

// cs_ij from the exchanged sums (float64, one rounding per operation)
__device__ __forceinline__ double foolsgold_cos(float pij, float ni, float nj) {
    if (!(is_finite(ni) && ni != 0.f && is_finite(nj) && nj != 0.f))
        return 0.0;
    double const q = __ddiv_rn(static_cast<double>(pij), __dmul_rn(__dsqrt_rn(static_cast<double>(ni)), __dsqrt_rn(static_cast<double>(nj))));
    return isfinite(q) ? q : 0.0;
}

// clip(x, 0, 1), +0 below
__device__ __forceinline__ double unit_clip(double x) {
    return x > 0.0 ? (x < 1.0 ? x : 1.0) : 0.0;
}

template<int N, int VEC>
__global__ void __launch_bounds__(N <= 8 ? 512 : 256, 1) gar_foolsgold_kernel(GarArgs const a) {
    __shared__ Shared sh;
    __shared__ int pair_of[kBlockRows * kBlockRows];
    __shared__ FoolsgoldShared fs;
    cg::grid_group grid = cg::this_grid();
    int const n = a.n, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nsums = n * (n + 1) / 2;
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    bool const multi = a.R > 1;
    if (threadIdx.x == 0) {
        sh.epoch = current_epoch(a);
        for (int i = 0; i < 4; ++i)
            sh.hyper[i] = a.hyper_ptr ? a.hyper_ptr[i] : (i == 0 ? a.lr : i == 1 ? a.h0 : i == 2 ? a.h1 : a.h2);
        fs.bad = 0u;
    }
    float* const mine = a.cta_partials + static_cast<long long>(blockIdx.x) * kFoolsgoldStride;
    for (int p = threadIdx.x; p < nsums; p += blockDim.x)
        mine[p] = 0.f;
    __syncthreads();
    uint32_t const epoch = sh.epoch;
    float const hyper[4] = {sh.hyper[0], sh.hyper[1], sh.hyper[2], sh.hyper[3]};
    if (multi) {   // entry barrier: every rank's gradients are published (nothing is pre-accumulated)
        if (blockIdx.x == 0)
            signal_all(a, 0, epoch);
        wait_all(a, 0, epoch);
        __syncthreads();
    }
    float local_loss = 0.f;
    if (blockIdx.x == 0 && threadIdx.x == 0 && a.loss_in)
        for (int j = 0; j < a.nloss; ++j)
            local_loss += a.loss_in[j];
    // -------- 1. history pass: H_i += g_i, the sums of the updated histories, the bad rows -------- //
    unsigned bad = 0u;
    for (int seg = 0; seg < a.nseg; ++seg)
        phase_a_segment<(N > kBlockRows), false, true>(a, sh, pair_of, seg, mine, tid, nthreads, &bad);
    bad = __reduce_or_sync(0xffffffffu, bad);
    if (lane == 0 && bad)
        atomicOr(&fs.bad, bad);
    __syncthreads();
    if (threadIdx.x < n)
        mine[kFoolsgoldSums + threadIdx.x] = ((fs.bad >> threadIdx.x) & 1u) ? 1.f : 0.f;
    // -------- 2. exchange of the sums, the flags and the loss -------- //
    __threadfence();
    grid.sync();
    if (blockIdx.x == 0) {
        for (int k = threadIdx.x; k < nsums + n; k += blockDim.x) {
            int const at = k < nsums ? k : kFoolsgoldSums + (k - nsums);
            float s = 0.f;
            for (unsigned b = 0; b < gridDim.x; ++b)
                s += ld_volatile_f(a.cta_partials + static_cast<long long>(b) * kFoolsgoldStride + at);
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kFoolsgoldRegion + a.rank * kFoolsgoldStride + at] = s;
        }
        if (threadIdx.x == 0)
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kFoolsgoldRegion + a.rank * kFoolsgoldStride + kFoolsgoldStride - 1] = local_loss;
        fence_sys();
        __syncthreads();
        if (multi)
            signal_all(a, kSlotFoolsgold, epoch);
    }
    if (multi) {
        wait_all(a, kSlotFoolsgold, epoch);
        __syncthreads();
    } else {
        grid.sync();
    }
    // -------- 3. the sums of every rank in rank order -> sh.dist (P, symmetric); coefficients on warp 0 -------- //
    float const* const box = a.mailbox[a.rank] + kFoolsgoldRegion;
    for (int p = threadIdx.x; p < nsums; p += blockDim.x) {
        int i = 0, rest = p;
        while (rest >= n - i) {   // sum index -> (i, j), i <= j
            rest -= n - i;
            ++i;
        }
        int const j = i + rest;
        float s = 0.f;
        for (int q = 0; q < a.R; ++q)
            s += ld_volatile_f(box + q * kFoolsgoldStride + p);
        sh.dist[i][j] = s;
        sh.dist[j][i] = s;
    }
    __syncthreads();
    if (warp == 0) {
        bool const row = lane < n;
        float flags = 0.f;
        for (int q = 0; q < a.R; ++q)
            flags += row ? ld_volatile_f(box + q * kFoolsgoldStride + kFoolsgoldSums + lane) : 0.f;
        float const ni = row ? sh.dist[lane][lane] : 0.f;
        double v = 0.0;   // v_i = max_j cs_ij, the diagonal's 0 included
        for (int j = 0; j < n; ++j)
            if (row && j != lane)
                v = fmax(v, foolsgold_cos(sh.dist[lane][j], ni, sh.dist[j][j]));
        double top_cs = 0.0;   // max_j of the pardoned cs_ij
        for (int j = 0; j < n; ++j) {
            double const vj = __shfl_sync(0xffffffffu, v, j);
            if (row && j != lane) {
                double cs = foolsgold_cos(sh.dist[lane][j], ni, sh.dist[j][j]);
                if (vj > v)
                    cs = __ddiv_rn(__dmul_rn(cs, v), vj);
                top_cs = fmax(top_cs, cs);
            }
        }
        double alpha = row ? unit_clip(__dsub_rn(1.0, top_cs)) : 0.0;
        double top = alpha;
        for (int o = 16; o > 0; o >>= 1)
            top = fmax(top, __shfl_xor_sync(0xffffffffu, top, o));
        float c = 0.f;
        if (top != 0.0) {
            alpha = __ddiv_rn(alpha, top);
            if (alpha == 1.0)
                alpha = 0.99;
            alpha = unit_clip(__dmul_rn(a.confidence, __dadd_rn(log(__ddiv_rn(alpha, __dsub_rn(1.0, alpha))), 0.5)));
            if (!row || flags != 0.f || !is_finite(ni))
                alpha = 0.0;
            double S = 0.0;
            for (int j = 0; j < n; ++j)
                S = __dadd_rn(S, __shfl_sync(0xffffffffu, alpha, j));
            c = S != 0.0 ? __double2float_rn(__ddiv_rn(alpha, S)) : 0.f;
        }
        fs.coef[lane] = c;
        unsigned const mask = __ballot_sync(0xffffffffu, c != 0.f);
        if (lane == 0)
            fs.mask = mask;
        if (blockIdx.x == 0) {
            if (a.foolsgold_out) {
                for (int p = lane; p < nsums; p += 32) {
                    float s = 0.f;
                    for (int q = 0; q < a.R; ++q)
                        s += ld_volatile_f(box + q * kFoolsgoldStride + p);
                    a.foolsgold_out[p] = s;
                }
                if (row) {
                    a.foolsgold_out[kFoolsgoldSums + lane] = flags != 0.f ? 1.f : 0.f;
                    a.foolsgold_out[kFoolsgoldSums + kMaxWorkers + lane] = c;
                }
            }
            if (lane == 0 && a.loss_out) {
                float total = 0.f;
                for (int q = 0; q < a.R; ++q)
                    total += ld_volatile_f(box + q * kFoolsgoldStride + kFoolsgoldStride - 1);
                *a.loss_out = total;
            }
        }
    }
    __syncthreads();
    // -------- 4. phase D: weighted sum, update, broadcast -------- //
    weighted_phase_d<N, VEC>(a, grid, hyper, fs.coef, fs.mask, epoch, tid, nthreads);
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
    // Min-Max / Min-Sum only (`gar_optimized_kernel`)
    int deviation;                     // 0: unit-vec (p = mu), 1: sign (p = sign(mu)), 2: std (p = sigma)
    int n;                             // the honest rows as `phase_a_segment` reads them: n = H rows grad[0, H), ascending slots,
    float const* grad[kMaxWorkers];    // no staging
    float* staging;
    float* mailbox[kMaxRanks];         // every rank's mailbox; region 2 (float offset kCraftRegion) carries the statistics
    float* partials;                   // [grid][kCraftStats] CTA partials of this rank
    float* stats_out;                  // optional [1 + kCraftStats]: gamma, then the statistics summed over the ranks
    // mimic only (`gar_mimic_warmup_kernel`, `gar_mimic_copy_kernel`)
    unsigned honest_mask;
    int t;                             // warm-up updates done before this one
    float* z;                          // (local) direction estimate of the owned coordinates, segments back to back (as the staged tile)
    float* y;                          // (local) scratch, same layout: y, kept apart so that z survives a degenerate ||y||
    int* istar;                        // [1] (local) target slot i*; a value that is no honest slot (-1 before any update) means the first one
    double* mimic_stats;               // optional [kMimicStats]: s_i, q_i, ||y||^2, 1 / ||y|| of the last warm-up step
    // Fang et al. only (`gar_fang_krum_kernel`: coef is the threshold; `gar_fang_trim_kernel`: coef is the scale beta)
    int f;                             // fang-krum: the rule's declared f
    int search;                        // fang-krum: 0 skips the candidate search (gamma = gamma_max), to time the passes alone
    double* fang_out;                  // fang-krum, optional [kFangOut]: gamma_max, t, selected
    unsigned long long key;            // fang-trim: K = splitmix64(splitmix64(splitmix64(seed) ^ step) ^ TAG), from the host
};
enum ByzMode { kAlie = 0, kIpm = 1, kMinMax = 2, kMinSum = 3 };
constexpr int kFangCandidates = 64;   // fang-krum: candidates gamma_max 2^-t, t < 64
constexpr int kFangOut = 3;           // fang-krum's `fang_out`: gamma_max, t (-1: no candidate tested), selected (0 / 1)
enum Deviation { kUnitVec = 0, kSign = 1, kStd = 2 };

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

// ---- Min-Max / Min-Sum (Shejwalkar & Houmansadr, NDSS 2021) ------------------------------------ //
// Every Byzantine row is b = mu - gamma * p, one rounded operation at a time, with ALIE's mu and the deviation p: mu (unit-vec), sign(mu)
// (+1, -1, 0 for +-0, NaN for NaN) or ALIE's sigma (std). gamma is one fp32 scalar per step, solved in closed form from sums over all
// d coordinates: A_i = sum (mu - h_i)^2, B_i = sum (mu - h_i) p, C = sum p^2 and, for Min-Max, the honest distances
// D_jk = sum (h_j - h_k)^2, T = max D_jk:
//   Min-Max: gamma = min_i gamma_i, E_i = max(T - A_i, 0), S_i = sqrt(B_i^2 + C E_i), gamma_i = (B_i + S_i) / C if B_i >= 0, else
//            E_i / (S_i - B_i) (the largest gamma >= 0 with max_i ||b - h_i||^2 <= T);
//   Min-Sum: gamma = sqrt(max_i A_i / C) (the summed constraint, reduced with sum_i B_i = 0 and sum_j D_ij = H A_i + sum A);
// in float64 from the fp32 sums, rounded once; gamma = 0 when C == 0 or any of T, A_i, B_i, C is not finite.
//
// One cooperative launch per rank:
//   1. entry barrier (slot kSlotCraft), as for ALIE / IPM;
//   2. statistics pass over the owned segments: mu and p per coordinate, A_i / B_i / C accumulated per thread for 8 honest rows at a time
//      (H <= 8: the H values stay in registers; above, one pass per 8-row block, mu and p recomputed from memory); Min-Max adds the
//      honest distances with `phase_a_segment` on the honest rows. Every pass folds lanes -> warps -> CTA (`fold_pass`) into the CTA's
//      slot of `partials`;
//   3. grid barrier; block 0 adds the CTA slots in index order and posts the rank's sums into mailbox region 2 of every rank, then
//      signals slot kSlotCraftStats; every CTA of every rank adds the R posts in rank order: the same bits, hence the same gamma,
//      everywhere;
//   4. write pass: mu and p recomputed from the honest rows (read a second time: staging them would cost 4 or 8 bytes of local HBM per
//      owned coordinate for a pass that is bound by the honest reads either way), b stored into every Byzantine row (P2P stores).
// It ends with a system-scope fence and no exit barrier, as `gar_byzantine_kernel` (same argument). Region 2 and slot kSlotCraftStats
// are touched by no other kernel: a fast rank's finish kernel writes regions 0 / 1 of a slow rank's mailbox while the slow rank's
// crafting CTAs may still be reading region 2. The next step's crafting does not race with this one: a rank posts into region 2 only
// after the next entry barrier, i.e. after every rank has started its next crafting kernel, so after every rank's current crafting
// kernel (same stream) has finished reading.

// mu and p of the 4 coordinates at x. N > 0: the H <= N honest values are in g; N == 0: they are read from memory. mu and sigma are
// computed exactly as in `gar_byzantine_kernel`.
template<int N>
__device__ __forceinline__ void mean_and_deviation(ByzArgs const& a, long long x, float const (&g)[N > 0 ? N : 1][4], float (&mu)[4], float (&p)[4]) {
    int const H = a.H;
    if constexpr (N > 0) {
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
    float const count = static_cast<float>(H);
#pragma unroll
    for (int c = 0; c < 4; ++c)
        mu[c] = __fdiv_rn(mu[c], count);
    if (a.deviation == kStd) {
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
            p[c] = __fsqrt_rn(__fdiv_rn(var[c], dof));
    } else if (a.deviation == kSign) {
#pragma unroll
        for (int c = 0; c < 4; ++c)
            p[c] = mu[c] > 0.f ? 1.f : mu[c] < 0.f ? -1.f : mu[c] == 0.f ? 0.f : mu[c];
    } else {
#pragma unroll
        for (int c = 0; c < 4; ++c)
            p[c] = mu[c];
    }
}

// A_i and B_i of the honest rows [i0, i0 + 8) (and C with the first block) over every owned segment, folded into `out`
template<int N>
__device__ void optimized_stats_pass(ByzArgs const& a, Shared& sh, int* pair_of, int i0, float* out, long long tid, long long nthreads) {
    constexpr int B = kBlockRows, COUNT = 2 * B + 1;
    static_assert(N == 0 || N == B, "registers hold one block of honest rows");
    int const H = a.H;
    if (threadIdx.x < COUNT) {
        int const t = threadIdx.x, i = i0 + t % B;
        pair_of[t] = t == 2 * B ? (i0 == 0 ? kStatC : -1) : i < H ? (t < B ? kStatA : kStatB) + i : -1;
    }
    __syncthreads();
    float acc[COUNT];
#pragma unroll
    for (int k = 0; k < COUNT; ++k)
        acc[k] = 0.f;
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4;
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            float g[N > 0 ? N : 1][4];
            if constexpr (N > 0) {
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if (i < H)
                        V<4>::load_stream(a.rows[a.honest[i]] + x, g[i]);
            }
            float mu[4], p[4];
            mean_and_deviation<N>(a, x, g, mu, p);
#pragma unroll
            for (int i = 0; i < B; ++i) {
                if (i0 + i < H) {
                    float h[4];
                    if constexpr (N > 0) {
#pragma unroll
                        for (int c = 0; c < 4; ++c)
                            h[c] = g[i][c];
                    } else {
                        V<4>::load(a.rows[a.honest[i0 + i]] + x, h);
                    }
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        float const dev = __fsub_rn(mu[c], h[c]);
                        acc[i] = __fmaf_rn(dev, dev, acc[i]);
                        acc[B + i] = __fmaf_rn(dev, p[c], acc[B + i]);
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < 4; ++c)
                acc[2 * B] = __fmaf_rn(p[c], p[c], acc[2 * B]);
        }
    }
    fold_pass<COUNT>(sh, acc, out, pair_of);
}

// gamma from the statistics summed over the ranks (see above), float64 with explicit roundings (no FMA contraction), rounded once to fp32
__device__ float optimized_gamma(int mode, int H, float const* st) {
    bool ok = is_finite(st[kStatC]) && st[kStatC] != 0.f;
    double const C = st[kStatC];
    double amax = 0.0, T = 0.0;
    for (int i = 0; i < H; ++i) {
        ok = ok && is_finite(st[kStatA + i]) && is_finite(st[kStatB + i]);
        amax = fmax(amax, static_cast<double>(st[kStatA + i]));
    }
    if (mode == kMinMax) {
        for (int k = 0; k < H * (H - 1) / 2; ++k) {
            ok = ok && is_finite(st[k]);
            T = fmax(T, static_cast<double>(st[k]));
        }
    }
    if (!ok)
        return 0.f;
    if (mode == kMinSum)
        return __double2float_rn(__dsqrt_rn(__ddiv_rn(amax, C)));
    double gamma = 0.0;
    for (int i = 0; i < H; ++i) {
        double const A = st[kStatA + i], Bi = st[kStatB + i];
        double const E = fmax(__dsub_rn(T, A), 0.0);
        double const S = __dsqrt_rn(__dadd_rn(__dmul_rn(Bi, Bi), __dmul_rn(C, E)));
        double const gi = Bi >= 0.0 ? __ddiv_rn(__dadd_rn(Bi, S), C) : __ddiv_rn(E, __dsub_rn(S, Bi));
        gamma = i == 0 ? gi : fmin(gamma, gi);
    }
    return __double2float_rn(gamma);
}

template<int N>
__global__ void __launch_bounds__(256) gar_optimized_kernel(ByzArgs const a) {
    __shared__ Shared sh;
    __shared__ int pair_of[kBlockRows * kBlockRows];
    __shared__ float stats[kCraftStats];
    __shared__ float gamma_sh;
    cg::grid_group grid = cg::this_grid();
    bool const multi = a.R > 1;
    uint32_t const epoch = current_epoch(a);
    if (multi) {
        signal_all(a, kSlotCraft, epoch);
        wait_all(a, kSlotCraft, epoch);
        __syncthreads();
    }
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    int const H = a.H;
    float* const mine = a.partials + static_cast<long long>(blockIdx.x) * kCraftStats;
    for (int k = threadIdx.x; k < kCraftStats; k += blockDim.x)
        mine[k] = 0.f;
    __syncthreads();
    // -------- statistics of the owned coordinates -------- //
    for (int i0 = 0; i0 < H; i0 += kBlockRows)
        optimized_stats_pass<N>(a, sh, pair_of, i0, mine, tid, nthreads);
    if (a.mode == kMinMax) {
        for (int seg = 0; seg < a.nseg; ++seg)
            phase_a_segment<(N == 0)>(a, sh, pair_of, seg, mine, tid, nthreads);
    }
    // -------- exchange: CTAs in index order, then ranks in rank order -------- //
    __threadfence();
    grid.sync();
    if (blockIdx.x == 0) {
        for (int k = threadIdx.x; k < kCraftStats; k += blockDim.x) {
            float s = 0.f;
            for (unsigned b = 0; b < gridDim.x; ++b)
                s += ld_volatile_f(a.partials + static_cast<long long>(b) * kCraftStats + k);
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kCraftRegion + a.rank * kCraftStats + k] = s;
        }
        fence_sys();
        __syncthreads();
        if (multi)
            signal_all(a, kSlotCraftStats, epoch);
    }
    if (multi) {
        wait_all(a, kSlotCraftStats, epoch);
        __syncthreads();
    } else {
        grid.sync();
    }
    float const* const box = a.mailbox[a.rank] + kCraftRegion;
    for (int k = threadIdx.x; k < kCraftStats; k += blockDim.x) {
        float s = 0.f;
        for (int q = 0; q < a.R; ++q)
            s += ld_volatile_f(box + q * kCraftStats + k);
        stats[k] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0)
        gamma_sh = optimized_gamma(a.mode, H, stats);
    __syncthreads();
    float const gamma = gamma_sh;
    if (a.stats_out && blockIdx.x == 0) {
        for (int k = threadIdx.x; k < kCraftStats; k += blockDim.x)
            a.stats_out[1 + k] = stats[k];
        if (threadIdx.x == 0)
            a.stats_out[0] = gamma;
    }
    // -------- b = mu - gamma * p into every Byzantine row -------- //
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4;
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            float g[N > 0 ? N : 1][4];
            if constexpr (N > 0) {
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if (i < H)
                        V<4>::load_stream(a.rows[a.honest[i]] + x, g[i]);
            }
            float mu[4], p[4], out[4];
            mean_and_deviation<N>(a, x, g, mu, p);
#pragma unroll
            for (int c = 0; c < 4; ++c)
                out[c] = __fsub_rn(mu[c], __fmul_rn(gamma, p[c]));
            for (int k = 0; k < a.K; ++k)
                V<4>::store_stream(a.rows[a.byz[k]] + x, out);
        }
    }
    fence_sys();
}

// ---- mimic (Karimireddy, He & Jaggi, ICLR 2022) ------------------------------------------------ //
// Every Byzantine row is a bit-for-bit copy of one honest row h_{i*}. During the T0 warm-up steps, i* follows the honest row that reaches
// furthest along the top principal direction z of the honest rows, estimated by the online power iteration of the paper's appendix:
//   mu = ((h_0 + h_1) + ...) / H, s_i = sum_j (h_i - mu)_j z_j,
//   u = (s_0 (h_0 - mu) + s_1 (h_1 - mu) + ...) / H, y = (t z + u) / (t + 1)   (fp32, one rounded operation at a time),
//   z <- y * (1 / ||y||), i* = argmax_i q_i with q_i = sum_j h_i,j y_j (ties: lower slot; non-finite q never wins; none finite: the first
//   honest slot); when ||y||^2 is 0 or not finite, z and i* keep their values.
// The whole-vector sums are fp32 partials per thread (FMA), folded lanes -> warps -> CTA (`fold_pass`) -> CTAs in index order, posted
// per rank and added over the ranks in rank order in float64; s_i and 1 / ||y|| are rounded once to fp32, every rank gets the same bits.
//
// Warm-up: one cooperative launch per rank (`gar_mimic_warmup_kernel`):
//   1. entry barrier (slot kSlotCraft), as for ALIE / IPM;
//   2. pass 1 over the owned segments: the s_i partials (H <= 8: the honest values in registers; above, 8-row blocks, mu recomputed);
//   3. exchange 1: region 2 floats [kMimicS, +32), slot kSlotCraftStats;
//   4. pass 2: mu and u recomputed, y stored into the y scratch, ||y||^2 and q_i partials;
//   5. exchange 2: region 2 floats [kMimicQ, kMimicY], slot kSlotMimic;
//   6. pass 3: z <- y / ||y|| on the owned coordinates, h_{i*} copied into every Byzantine row (P2P stores); block 0 stores i* and the
//      statistics.
// After the warm-up, `gar_mimic_copy_kernel` copies h_{i*}, with i* read from device memory: no exchange, no host read-back.
// Both end with a system-scope fence and no exit barrier, as `gar_byzantine_kernel` (same argument). Within a step the two posts are
// disjoint floats of region 2, so a fast rank's second post never overwrites a first post a slow rank is still adding; a rank's next
// post comes after the next entry barrier, i.e. after every rank has finished this kernel (same stream). Region 2 is Min-Max's, and an
// engine runs one attack.

// the slot i* designates: itself when it is an honest slot, the first honest slot otherwise
__device__ __forceinline__ int mimic_target(ByzArgs const& a, int istar) {
    return istar >= 0 && istar < kMaxWorkers && ((a.honest_mask >> istar) & 1u) ? istar : a.honest[0];
}

// the 4 values of honest row i (ascending honest index) at x: from the registers (N > 0) or from memory
template<int N>
__device__ __forceinline__ void honest_value(ByzArgs const& a, long long x, float const (&g)[N > 0 ? N : 1][4], int i, float (&h)[4]) {
    if constexpr (N > 0) {
#pragma unroll
        for (int c = 0; c < 4; ++c)
            h[c] = g[i][c];
    } else {
        V<4>::load(a.rows[a.honest[i]] + x, h);
    }
}

// pass 1: the s_i partials of the honest rows [i0, i0 + 8) over every owned segment, folded into `out`
template<int N>
__device__ void mimic_s_pass(ByzArgs const& a, Shared& sh, int* pair_of, int i0, float* out, long long tid, long long nthreads) {
    constexpr int B = kBlockRows;
    static_assert(N == 0 || N == B, "registers hold one block of honest rows");
    int const H = a.H;
    if (threadIdx.x < B)
        pair_of[threadIdx.x] = i0 + static_cast<int>(threadIdx.x) < H ? kMimicS + i0 + static_cast<int>(threadIdx.x) : -1;
    __syncthreads();
    float acc[B];
#pragma unroll
    for (int k = 0; k < B; ++k)
        acc[k] = 0.f;
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4, soff = staged_offset(a, seg);   // z, y: owned order
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            float g[N > 0 ? N : 1][4];
            if constexpr (N > 0) {
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if (i < H)
                        V<4>::load_stream(a.rows[a.honest[i]] + x, g[i]);
            }
            float mu[4], p[4], z[4];
            mean_and_deviation<N>(a, x, g, mu, p);
            V<4>::load(a.z + soff + v * 4, z);
#pragma unroll
            for (int i = 0; i < B; ++i) {
                if (i0 + i < H) {
                    float h[4];
                    honest_value<N>(a, x, g, N > 0 ? i : i0 + i, h);   // N > 0: one block, i0 == 0, a static register index
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        acc[i] = __fmaf_rn(__fsub_rn(h[c], mu[c]), z[c], acc[i]);
                }
            }
        }
    }
    fold_pass<B>(sh, acc, out, pair_of);
}

// pass 2: y = (t z + u) / (t + 1) into the y scratch, and the partials of q_i and ||y||^2, folded into `out`
template<int N>
__device__ void mimic_y_pass(ByzArgs const& a, Shared& sh, int* pair_of, float const* s, float* out, long long tid, long long nthreads) {
    constexpr int M = N > 0 ? N : kMaxWorkers, COUNT = M + 1;
    int const H = a.H;
    if (threadIdx.x < COUNT) {
        int const k = threadIdx.x;
        pair_of[k] = k == M ? kMimicY : k < H ? kMimicQ + k : -1;
    }
    __syncthreads();
    float const tf = static_cast<float>(a.t), t1 = static_cast<float>(a.t + 1), count = static_cast<float>(H);
    float acc[COUNT];
#pragma unroll
    for (int k = 0; k < COUNT; ++k)
        acc[k] = 0.f;
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4, soff = staged_offset(a, seg);   // z, y: owned order
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            float g[N > 0 ? N : 1][4];
            if constexpr (N > 0) {
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if (i < H)
                        V<4>::load_stream(a.rows[a.honest[i]] + x, g[i]);
            }
            float mu[4], p[4], z[4], u[4], y[4];
            mean_and_deviation<N>(a, x, g, mu, p);
            V<4>::load(a.z + soff + v * 4, z);
#pragma unroll
            for (int i = 0; i < M; ++i) {
                if (i < H) {
                    float h[4];
                    honest_value<N>(a, x, g, i, h);
                    float const si = s[i];
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        float const term = __fmul_rn(si, __fsub_rn(h[c], mu[c]));
                        u[c] = i == 0 ? term : __fadd_rn(u[c], term);
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                y[c] = __fdiv_rn(__fadd_rn(__fmul_rn(tf, z[c]), __fdiv_rn(u[c], count)), t1);
                acc[M] = __fmaf_rn(y[c], y[c], acc[M]);
            }
            V<4>::store(a.y + soff + v * 4, y);
#pragma unroll
            for (int i = 0; i < M; ++i) {
                if (i < H) {
                    float h[4];
                    honest_value<N>(a, x, g, i, h);
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        acc[i] = __fmaf_rn(h[c], y[c], acc[i]);
                }
            }
        }
    }
    fold_pass<COUNT>(sh, acc, out, pair_of);
}

// block 0 adds the CTA partials [lo, hi) in index order and posts them into region 2 of every rank, then signals `slot`; returns once
// every rank's post is visible to every CTA (mimic's two exchanges, fang-krum's one)
__device__ void stats_exchange(ByzArgs const& a, cg::grid_group& grid, int lo, int hi, int slot, uint32_t epoch) {
    bool const multi = a.R > 1;
    __threadfence();
    grid.sync();
    if (blockIdx.x == 0) {
        for (int k = lo + threadIdx.x; k < hi; k += blockDim.x) {
            float s = 0.f;
            for (unsigned b = 0; b < gridDim.x; ++b)
                s += ld_volatile_f(a.partials + static_cast<long long>(b) * kCraftStats + k);
            for (int q = 0; q < a.R; ++q)
                a.mailbox[q][kCraftRegion + a.rank * kCraftStats + k] = s;
        }
        fence_sys();
        __syncthreads();
        if (multi)
            signal_all(a, slot, epoch);
    }
    if (multi) {
        wait_all(a, slot, epoch);
        __syncthreads();
    } else {
        grid.sync();
    }
}

// the posts of float k of every rank, added in rank order in float64
__device__ __forceinline__ double mimic_total(ByzArgs const& a, int k) {
    float const* const box = a.mailbox[a.rank] + kCraftRegion;
    double s = 0.0;
    for (int q = 0; q < a.R; ++q)
        s += static_cast<double>(ld_volatile_f(box + q * kCraftStats + k));
    return s;
}

template<int N>
__global__ void __launch_bounds__(256) gar_mimic_warmup_kernel(ByzArgs const a) {
    __shared__ Shared sh;
    __shared__ int pair_of[kBlockRows * kBlockRows];
    __shared__ float s_sh[kMaxWorkers];
    __shared__ double q_sh[kMaxWorkers];
    __shared__ float inv_sh;
    __shared__ int target_sh, ok_sh;
    __shared__ double norm_sh;
    cg::grid_group grid = cg::this_grid();
    uint32_t const epoch = current_epoch(a);
    if (a.R > 1) {
        signal_all(a, kSlotCraft, epoch);
        wait_all(a, kSlotCraft, epoch);
        __syncthreads();
    }
    int const previous = *a.istar;   // read before the first grid barrier; block 0 stores the new i* after the last one
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    int const H = a.H;
    float* const mine = a.partials + static_cast<long long>(blockIdx.x) * kCraftStats;
    for (int k = threadIdx.x; k <= kMimicY; k += blockDim.x)
        mine[k] = 0.f;
    __syncthreads();
    // -------- pass 1 and exchange 1: s_i -------- //
    for (int i0 = 0; i0 < H; i0 += kBlockRows)
        mimic_s_pass<N>(a, sh, pair_of, i0, mine, tid, nthreads);
    stats_exchange(a, grid, kMimicS, kMimicS + H, kSlotCraftStats, epoch);
    int const lane = threadIdx.x;
    if (lane < H)
        s_sh[lane] = __double2float_rn(mimic_total(a, kMimicS + lane));
    __syncthreads();
    // -------- pass 2 and exchange 2: y, q_i, ||y||^2 -------- //
    mimic_y_pass<N>(a, sh, pair_of, s_sh, mine, tid, nthreads);
    stats_exchange(a, grid, kMimicQ, kMimicY + 1, kSlotMimic, epoch);
    if (lane < H)
        q_sh[lane] = mimic_total(a, kMimicQ + lane);
    if (lane == kMaxWorkers)
        norm_sh = mimic_total(a, kMimicY);
    __syncthreads();
    if (threadIdx.x == 0) {
        double const norm2 = norm_sh;
        bool const ok = norm2 > 0.0 && isfinite(norm2);
        int best = -1;
        for (int i = 0; i < H; ++i)
            if (isfinite(q_sh[i]) && (best < 0 || q_sh[i] > q_sh[best]))
                best = i;
        ok_sh = ok;
        inv_sh = ok ? __double2float_rn(__ddiv_rn(1.0, __dsqrt_rn(norm2))) : 0.f;
        target_sh = ok ? a.honest[best < 0 ? 0 : best] : mimic_target(a, previous);
    }
    __syncthreads();
    float const inv = inv_sh;
    int const target = target_sh;
    bool const ok = ok_sh != 0;
    // -------- pass 3: z <- y / ||y||, h_{i*} into every Byzantine row -------- //
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4, soff = staged_offset(a, seg);   // z, y: owned order
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            if (ok) {
                float y[4];
                V<4>::load(a.y + soff + v * 4, y);
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    y[c] = __fmul_rn(y[c], inv);
                V<4>::store(a.z + soff + v * 4, y);
            }
            float h[4];
            V<4>::load_stream(a.rows[target] + x, h);
            for (int k = 0; k < a.K; ++k)
                V<4>::store_stream(a.rows[a.byz[k]] + x, h);
        }
    }
    if (blockIdx.x == 0) {
        if (threadIdx.x == 0)
            *a.istar = target;
        if (a.mimic_stats) {
            if (lane < H) {
                a.mimic_stats[kMimicS + lane] = s_sh[lane];
                a.mimic_stats[kMimicQ + lane] = q_sh[lane];
            }
            if (threadIdx.x == 0) {
                a.mimic_stats[kMimicY] = norm_sh;
                a.mimic_stats[kMimicY + 1] = inv;
            }
        }
    }
    fence_sys();
}

__global__ void __launch_bounds__(256) gar_mimic_copy_kernel(ByzArgs const a) {
    if (a.R > 1) {
        uint32_t const epoch = current_epoch(a);
        signal_all(a, kSlotCraft, epoch);
        wait_all(a, kSlotCraft, epoch);
        __syncthreads();
    }
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    float const* const src = a.rows[mimic_target(a, *a.istar)];
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4;
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            float h[4];
            V<4>::load_stream(src + x, h);
            for (int k = 0; k < a.K; ++k)
                V<4>::store_stream(a.rows[a.byz[k]] + x, h);
        }
    }
    fence_sys();
}

// ---- Fang, Cao, Jia & Gong (USENIX Security 2020): full-knowledge Krum and trimmed-mean attacks, on gradient rows ------------- //
// fang-krum: every Byzantine row is b = (-gamma) * p, p = sign(mu) (Min-Max's `sign` deviation), one fp32 multiply. gamma comes from the
// fp32 sums A_i = sum h_i^2, B_i = sum h_i p, C = sum p^2 and the honest distances T_jk = sum (h_j - h_k)^2, posted in Min-Max's layout
// (pairs, A[32], B[32], C). In float64 with explicit roundings, as `_ops.fang_krum_gamma`:
//   gamma_max = min_i R_i / ((n - 2K - 1) sqrt(C)) + max_i sqrt(A_i) / sqrt(C), R_i the ascending sum of the H - 2 smallest sqrt(T_il);
//   candidates gamma_max 2^-t, t = 0, 1, ... while t == 0 or gamma_t >= threshold (at most 64): the first one for which Krum with the
//   declared f ranks a Byzantine slot first (ascending score, ties to the lower slot) is kept, else the last one tested; rounded once.
//   Krum sees 0 between Byzantine rows, max(0, (A_i + (2 gamma) B_i) + (gamma gamma) C) between a Byzantine row and honest row i, T
//   between honest rows; a score is the ascending sum of the row's n - f - 2 smallest distances.
//   gamma = 0 (not selected, t = -1) when C == 0 or any sum is not finite.
// One cooperative launch per rank on `gar_optimized_kernel`'s scaffolding: entry barrier (slot kSlotCraft); statistics pass and honest
// distance pass (`phase_a_segment` on the honest rows); one exchange through region 2 and slot kSlotCraftStats; the search on warp 0 of
// every CTA (a lane per honest row, whose distances are sorted once; per candidate a lane merges them with its K copies of the
// Byzantine distance, O(n) additions, and one lane scores the Byzantine rows, which all have the same score); write pass. No exit
// barrier, system-scope fence at the end, as `gar_optimized_kernel` (same argument: region 2 and its slot belong to the crafting kernels
// and an engine runs one attack).
//
// fang-trim: per coordinate x (global index of the padded vector) and Byzantine slot k, b = lo + u (hi - lo) (fp32, one rounding per
// operation) with, from ALIE's mu and the honest rows h (ascending slots):
//   mu > 0: e = min_i h_i, [lo, hi] = [e beta, e] if e <= 0, else [e / beta, e];
//   mu < 0: e = max_i h_i, [lo, hi] = [e, e beta] if e >= 0, else [e, e / beta];
//   b = mu when mu is +-0 or NaN; u = (splitmix64(K ^ (x 32 + k)) >> 40) 2^-24.
// The draw depends on (seed, step, slot, x) only: the rows are the same bits on every engine and every rank count. One pass, no
// exchange, `gar_byzantine_kernel`'s entry barrier and closing fence.

// A_i and B_i of the honest rows [i0, i0 + 8) (and C with the first block) over every owned segment, folded into `out`
template<int N>
__device__ void fang_stats_pass(ByzArgs const& a, Shared& sh, int* pair_of, int i0, float* out, long long tid, long long nthreads) {
    constexpr int B = kBlockRows, COUNT = 2 * B + 1;
    static_assert(N == 0 || N == B, "registers hold one block of honest rows");
    int const H = a.H;
    if (threadIdx.x < COUNT) {
        int const t = threadIdx.x, i = i0 + t % B;
        pair_of[t] = t == 2 * B ? (i0 == 0 ? kStatC : -1) : i < H ? (t < B ? kStatA : kStatB) + i : -1;
    }
    __syncthreads();
    float acc[COUNT];
#pragma unroll
    for (int k = 0; k < COUNT; ++k)
        acc[k] = 0.f;
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4;
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            float g[N > 0 ? N : 1][4];
            if constexpr (N > 0) {
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if (i < H)
                        V<4>::load_stream(a.rows[a.honest[i]] + x, g[i]);
            }
            float mu[4], p[4];
            mean_and_deviation<N>(a, x, g, mu, p);   // a.deviation == kSign
#pragma unroll
            for (int i = 0; i < B; ++i) {
                if (i0 + i < H) {
                    float h[4];
                    honest_value<N>(a, x, g, N > 0 ? i : i0 + i, h);   // N > 0: one block, i0 == 0, a static register index
#pragma unroll
                    for (int c = 0; c < 4; ++c) {
                        acc[i] = __fmaf_rn(h[c], h[c], acc[i]);
                        acc[B + i] = __fmaf_rn(h[c], p[c], acc[B + i]);
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < 4; ++c)
                acc[2 * B] = __fmaf_rn(p[c], p[c], acc[2 * B]);
        }
    }
    fold_pass<COUNT>(sh, acc, out, pair_of);
}

// the search of fang-krum on warp 0 over the statistics `st` summed over the ranks: lane i < H is honest row i (slot honest[i]), lane H
// the Byzantine rows. `sorted`: [32][32] float64 scratch (row i: the H - 1 honest distances of row i, ascending), `dist` / `ranked`: [32].
// Lane 0 stores gamma_max, t, selected and the float64 gamma into `out`.
__device__ void fang_krum_search(ByzArgs const& a, float const* st, double (*sorted)[kMaxWorkers], double* dist, double* ranked, double* out) {
    unsigned const all = 0xffffffffu;
    int const lane = threadIdx.x & 31, H = a.H, K = a.K, n = H + K, m = n - a.f - 2, npairs = H * (H - 1) / 2;
    bool finite = lane != 0 || (is_finite(st[kStatC]) && st[kStatC] != 0.f);
    for (int k = lane; k < npairs; k += 32)
        finite = finite && is_finite(st[k]);
    if (lane < H)
        finite = finite && is_finite(st[kStatA + lane]) && is_finite(st[kStatB + lane]);
    if (!__all_sync(all, finite)) {
        if (lane == 0) {
            out[0] = 0.0;
            out[1] = -1.0;
            out[2] = 0.0;
            out[3] = 0.0;
        }
        return;
    }
    double const C = st[kStatC];
    double R = __longlong_as_double(0x7ff0000000000000ll), root_a = -R;   // +inf, -inf: neutral for the lanes >= H
    double A = 0.0, Bi = 0.0;
    if (lane < H) {
        A = st[kStatA + lane];
        Bi = st[kStatB + lane];
        int count = 0;
        for (int l = 0; l < H; ++l) {   // insertion sort of the row's honest distances
            if (l == lane)
                continue;
            double const v = st[l < lane ? pair_index(l, lane, H) : pair_index(lane, l, H)];
            int at = count++;
            for (; at > 0 && sorted[lane][at - 1] > v; --at)
                sorted[lane][at] = sorted[lane][at - 1];
            sorted[lane][at] = v;
        }
        R = 0.0;
        for (int k = 0; k < H - 2; ++k)
            R = __dadd_rn(R, __dsqrt_rn(sorted[lane][k]));
        root_a = __dsqrt_rn(A);
    }
    for (int off = 16; off > 0; off >>= 1) {
        R = fmin(R, __shfl_xor_sync(all, R, off));
        root_a = fmax(root_a, __shfl_xor_sync(all, root_a, off));
    }
    double const root = __dsqrt_rn(C);
    double const gamma_max = __dadd_rn(__ddiv_rn(R, __dmul_rn(static_cast<double>(n - 2 * K - 1), root)), __ddiv_rn(root_a, root));
    double const threshold = a.coef;
    double gamma = gamma_max;
    int t = 0, selected = 0;
    int const candidates = a.search ? kFangCandidates : 1;
    for (int c = 0; c < candidates; ++c) {
        double const g = __dmul_rn(gamma_max, ldexp(1.0, -c));
        if (c > 0 && !(g >= threshold))
            break;
        gamma = g;
        t = c;
        if (!a.search)
            break;
        double D = 0.0;
        if (lane < H) {
            D = __dadd_rn(__dadd_rn(A, __dmul_rn(__dmul_rn(2.0, g), Bi)), __dmul_rn(__dmul_rn(g, g), C));
            D = D > 0.0 ? D : 0.0;
            dist[lane] = D;
        }
        __syncwarp();
        double score = __longlong_as_double(0x7ff0000000000000ll);
        int slot = kMaxWorkers;
        if (lane < H) {   // merge the sorted honest distances with K copies of D, the m smallest added in ascending order
            int rank = 0;
            for (int l = 0; l < H; ++l)
                rank += dist[l] < D || (dist[l] == D && l < lane);
            ranked[rank] = D;
            score = 0.0;
            for (int q = 0, j = 0, copies = 0; q < m; ++q) {
                double v;
                if (j < H - 1 && (copies >= K || sorted[lane][j] <= D)) {
                    v = sorted[lane][j++];
                } else {
                    v = D;
                    ++copies;
                }
                score = __dadd_rn(score, v);
            }
            slot = a.honest[lane];
        }
        __syncwarp();
        if (lane == H) {   // K - 1 zeros, then the distances to the honest rows in ascending order
            score = 0.0;
            for (int q = 0; q < m; ++q)
                score = __dadd_rn(score, q < K - 1 ? 0.0 : ranked[q - (K - 1)]);
            slot = a.byz[0];
        }
        for (int off = 16; off > 0; off >>= 1) {
            double const other = __shfl_xor_sync(all, score, off);
            int const other_slot = __shfl_xor_sync(all, slot, off);
            if (other < score || (other == score && other_slot < slot)) {
                score = other;
                slot = other_slot;
            }
        }
        __syncwarp();
        if (slot == a.byz[0]) {
            selected = 1;
            break;
        }
    }
    if (lane == 0) {
        out[0] = gamma_max;
        out[1] = t;
        out[2] = selected;
        out[3] = gamma;
    }
}

template<int N>
__global__ void __launch_bounds__(256) gar_fang_krum_kernel(ByzArgs const a) {
    __shared__ Shared sh;
    __shared__ int pair_of[kBlockRows * kBlockRows];
    __shared__ float stats[kCraftStats];
    __shared__ double sorted[kMaxWorkers][kMaxWorkers];
    __shared__ double dist[kMaxWorkers], ranked[kMaxWorkers];
    __shared__ double result[kFangOut + 1];
    cg::grid_group grid = cg::this_grid();
    uint32_t const epoch = current_epoch(a);
    if (a.R > 1) {
        signal_all(a, kSlotCraft, epoch);
        wait_all(a, kSlotCraft, epoch);
        __syncthreads();
    }
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    int const H = a.H;
    float* const mine = a.partials + static_cast<long long>(blockIdx.x) * kCraftStats;
    for (int k = threadIdx.x; k < kCraftStats; k += blockDim.x)
        mine[k] = 0.f;
    __syncthreads();
    // -------- statistics of the owned coordinates, then the honest distances -------- //
    for (int i0 = 0; i0 < H; i0 += kBlockRows)
        fang_stats_pass<N>(a, sh, pair_of, i0, mine, tid, nthreads);
    for (int seg = 0; seg < a.nseg; ++seg)
        phase_a_segment<(N == 0)>(a, sh, pair_of, seg, mine, tid, nthreads);
    // -------- exchange: CTAs in index order, then ranks in rank order -------- //
    stats_exchange(a, grid, 0, kCraftStats, kSlotCraftStats, epoch);
    float const* const box = a.mailbox[a.rank] + kCraftRegion;
    for (int k = threadIdx.x; k < kCraftStats; k += blockDim.x) {
        float s = 0.f;
        for (int q = 0; q < a.R; ++q)
            s += ld_volatile_f(box + q * kCraftStats + k);
        stats[k] = s;
    }
    __syncthreads();
    if (threadIdx.x < 32)
        fang_krum_search(a, stats, sorted, dist, ranked, result);
    __syncthreads();
    float const gamma = __double2float_rn(result[kFangOut]);
    if (blockIdx.x == 0) {
        if (a.stats_out) {
            for (int k = threadIdx.x; k < kCraftStats; k += blockDim.x)
                a.stats_out[1 + k] = stats[k];
            if (threadIdx.x == 0)
                a.stats_out[0] = gamma;
        }
        if (a.fang_out && threadIdx.x < kFangOut)
            a.fang_out[threadIdx.x] = result[threadIdx.x];
    }
    // -------- b = (-gamma) * sign(mu) into every Byzantine row -------- //
    float const neg = -gamma;
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4;
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            float g[N > 0 ? N : 1][4];
            if constexpr (N > 0) {
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if (i < H)
                        V<4>::load_stream(a.rows[a.honest[i]] + x, g[i]);
            }
            float mu[4], p[4], out[4];
            mean_and_deviation<N>(a, x, g, mu, p);
#pragma unroll
            for (int c = 0; c < 4; ++c)
                out[c] = __fmul_rn(neg, p[c]);
            for (int k = 0; k < a.K; ++k)
                V<4>::store_stream(a.rows[a.byz[k]] + x, out);
        }
    }
    fence_sys();
}

template<int N>
__global__ void __launch_bounds__(256) gar_fang_trim_kernel(ByzArgs const a) {
    if (a.R > 1) {
        uint32_t const epoch = current_epoch(a);
        signal_all(a, kSlotCraft, epoch);
        wait_all(a, kSlotCraft, epoch);
        __syncthreads();
    }
    long long const tid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    long long const nthreads = static_cast<long long>(gridDim.x) * blockDim.x;
    int const H = a.H;
    float const count = static_cast<float>(H), beta = a.coef;
    for (int seg = 0; seg < a.nseg; ++seg) {
        long long const lo = a.seg_lo[seg], lenv = (a.seg_hi[seg] - lo) / 4;
        for (long long v = tid; v < lenv; v += nthreads) {
            long long const x = lo + v * 4;
            float mu[4], low[4], high[4];
            auto add = [&](int i, float const (&h)[4]) {   // the sum of ALIE's mean, and the running min / max (strict comparisons)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    mu[c] = i == 0 ? h[c] : __fadd_rn(mu[c], h[c]);
                    low[c] = i == 0 || h[c] < low[c] ? h[c] : low[c];
                    high[c] = i == 0 || h[c] > high[c] ? h[c] : high[c];
                }
            };
            if constexpr (N > 0) {   // registers: the H honest values are loaded together
                float g[N][4];
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if (i < H)
                        V<4>::load_stream(a.rows[a.honest[i]] + x, g[i]);
#pragma unroll
                for (int i = 0; i < N; ++i)
                    if (i < H)
                        add(i, g[i]);
            } else {
                for (int i = 0; i < H; ++i) {
                    float h[4];
                    V<4>::load_stream(a.rows[a.honest[i]] + x, h);
                    add(i, h);
                }
            }
            float base[4], span[4];
            bool push[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                mu[c] = __fdiv_rn(mu[c], count);
                bool const pos = mu[c] > 0.f;
                push[c] = pos || mu[c] < 0.f;
                float const e = pos ? low[c] : high[c];
                float const scaled = __fmul_rn(e, beta), shrunk = __fdiv_rn(e, beta);
                float const l = pos ? (e <= 0.f ? scaled : shrunk) : e;
                float const h = pos ? e : (e >= 0.f ? scaled : shrunk);
                base[c] = l;
                span[c] = __fsub_rn(h, l);
            }
            for (int k = 0; k < a.K; ++k) {
                unsigned long long const slot = static_cast<unsigned long long>(a.byz[k]);
                float out[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    unsigned long long const z = splitmix64(a.key ^ (static_cast<unsigned long long>(x + c) * 32ull + slot));
                    float const u = __fmul_rn(static_cast<float>(static_cast<unsigned>(z >> 40)), 5.9604644775390625e-08f);   // 2^-24, exact
                    out[c] = push[c] ? __fadd_rn(base[c], __fmul_rn(u, span[c])) : mu[c];
                }
                V<4>::store_stream(a.rows[a.byz[k]] + x, out);
            }
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

template<int N, int VEC> int launch(GarArgs& a, int max_ctas, long long scratch_floats, cudaStream_t stream) {
    int const threads = N <= 8 ? 512 : 256;
    int device = 0, sms = 0, per_sm = 0;
    auto const kernel = a.rule == kDnc ? gar_dnc_kernel<N, VEC> : a.rule == kFltrust ? gar_fltrust_kernel<N, VEC>
                      : a.rule == kFoolsgold ? gar_foolsgold_kernel<N, VEC> : gar_fused_kernel<N, VEC>;
    AGB_CUDA_OK(cudaGetDevice(&device));
    AGB_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    AGB_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0));
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
    if (a.rule == kFoolsgold) {   // CTA slots of kFoolsgoldStride floats in `cta_partials` ([agb_gar_max_ctas()][kMaxPairs] floats)
        int const slots = static_cast<int>(static_cast<long long>(sms) * 4 * kMaxPairs / kFoolsgoldStride);
        grid = grid < slots ? grid : slots;
    }
    if (a.rule == kDnc) {   // CTA partials of this grid, then the samples
        long long const b = a.dnc_b < a.dnc_domain ? a.dnc_b : a.dnc_domain;
        if (static_cast<long long>(grid) * kDncIterations * kMaxPairs + a.iterations * a.n * ((b + 3) & ~3ll) > scratch_floats)
            return 108;
    }
    if (a.rule == kSmea && static_cast<long long>(grid) * (threads / 32) * (a.n - a.f) * (a.n - a.f) > scratch_floats)
        return 108;   // one [m][m] slab of doubles per warp
    void* params[] = {&a};
    AGB_CUDA_OK(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(kernel), dim3(grid), dim3(threads), params, 0, stream));
    return 0;
}

// The host checks of the fused entry points' arguments; returns a status (0: valid).
int check_args(GarArgs const& a) {
    if (a.n < 1 || a.n > kMaxWorkers || a.n_rows < 1 || a.n_rows > kMaxWorkers || a.R < 1 || a.R > kMaxRanks || a.rank < 0 || a.rank >= a.R)
        return 100;
    if (!(a.mix & kMixBucketing) && a.n_rows != a.n)
        return 100;
    if (a.nseg < 1 || a.nseg > kMaxSeg || a.first_seg < 0 || a.first_seg > a.nseg)
        return 101;
    for (int s = 0; s < a.nseg; ++s)
        if ((a.seg_lo[s] & 3) || (a.seg_hi[s] & 3) || a.seg_hi[s] < a.seg_lo[s])
            return 101;
    if (a.rule < 0 || a.rule > kFoolsgold)
        return 102;
    // FLTrust: any 0 <= f < n, a root, no pre-aggregation (it would change the rows whose direction and norm FLTrust scores), nothing
    // pre-accumulated
    if (a.rule == kFltrust && (a.f < 0 || a.f >= a.n || !a.root || a.mix != 0 || a.first_seg != 0))
        return 126;
    // FoolsGold: any 0 <= f < n, a finite kappa > 0, a history (127); no pre-aggregation (128: NNM mixes, ARC rescales and bucketing
    // reshuffles the rows every step, so a row would no longer be one worker's); nothing pre-accumulated (129: the history pass runs
    // in the finish kernel)
    if (a.rule == kFoolsgold && (a.f < 0 || a.f >= a.n || !a.history || !std::isfinite(a.confidence) || !(a.confidence > 0.0)))
        return 127;
    if (a.rule == kFoolsgold && a.mix != 0)
        return 128;
    if (a.rule == kFoolsgold && a.first_seg != 0)
        return 129;
    if (a.mix < 0 || a.mix > (kMixNnm | kMixArc | kMixBucketing))
        return 117;
    if ((a.mix & kMixBucketing) && (a.mix != kMixBucketing || a.bkt_size < 1 || a.bkt_size > a.n_rows ||
                                    a.n != (a.n_rows + a.bkt_size - 1) / a.bkt_size || !a.staging))   // the means land in the staging tile
        return 123;
    if ((a.mix & kMixArc) && (a.f < 0 || 2 * a.f >= a.n))
        return 120;
    if ((a.mix & kMixNnm) && (a.f < 0 || 2 * a.f >= a.n))
        return 117;
    if (a.rule == kCenteredClipping && (a.f < 0 || 2 * a.f >= a.n || a.iterations < 1 || a.iterations > kMaxIterations || !(a.tau > 0.f) ||
                                        !std::isfinite(a.tau) || !a.center))
        return 116;
    if (a.rule == kGeoMedian && (a.f < 0 || 2 * a.f >= a.n || a.iterations < 1 || a.iterations > kMaxIterations || !(a.nu > 0.f) || !std::isfinite(a.nu)))
        return 115;
    if (a.rule == kDnc && (a.f < 0 || 2 * a.f >= a.n || a.iterations < 1 || a.iterations > kDncIterations || a.dnc_r < 0 ||
                           a.n - a.iterations * a.dnc_r < 1 || a.dnc_b < 1 || a.dnc_b > (1ll << 20) || a.dnc_domain < 1 ||
                           a.dnc_domain > (1ll << 48) || a.dnc_step < 0))
        return 119;
    if ((a.rule == kTrimmedMean || a.rule == kMda) && (a.f < 0 || 2 * a.f >= a.n))
        return a.rule == kTrimmedMean ? 112 : 113;
    if (a.rule == kMda) {
        long long sets = 1;   // C(n, f), exact while it stays below the bound
        for (int t = 0; t < a.f && sets <= kMdaMaxSets; ++t)
            sets = sets * (a.n - t) / (t + 1);
        if (sets > kMdaMaxSets)
            return 113;
    }
    if (a.rule == kSmea) {
        if (a.f < 0 || 2 * a.f >= a.n)
            return 122;
        long long sets = 1;   // C(n, f), exact while it stays below the bound
        for (int t = 0; t < a.f && sets <= kSmeaMaxSets; ++t)
            sets = sets * (a.n - t) / (t + 1);
        if (sets > kSmeaMaxSets)
            return 122;
    }
    if ((a.rule == kKrum || a.rule == kBulyan) && (a.n - a.f - 2 < 1 || a.m < 1 || a.m > a.n))
        return 103;
    if (a.rule == kBulyan && (a.n < 4 * a.f + 3 || a.beta != a.n - 4 * a.f - 2 || a.m < a.n - 2 * a.f - 2))
        return 104;
    if (a.rule == kAveragedMedian && (a.beta < 1 || a.beta > a.n))
        return 105;
    if (a.opt != kNone && (!a.param || (!a.param_mc && !a.param_dst[0])))
        return 106;
    if ((a.opt == kAdam || a.opt == kRmsprop || a.opt == kAdadelta) && (!a.slot0 || !a.slot1))
        return 107;
    if (a.opt == kAdagrad && !a.slot0)
        return 107;
    if ((a.rule == kKrum || a.rule == kBulyan || a.rule == kMda || a.rule == kSmea || a.rule == kGeoMedian || a.rule == kCenteredClipping) &&
        (!a.cta_partials || !a.mailbox[0]))
        return 108;
    if (a.rule == kSmea && !a.smea_scratch)
        return 108;
    if (a.rule == kFltrust && (!a.cta_partials || !a.mailbox[0] || ((a.R > 1 || a.n > kBlockRows) && !a.staging)))
        return 108;   // FLTrust's second pass reads the staged rows over several ranks or beyond the 8 rows of one block
    if (a.rule == kFoolsgold && (!a.cta_partials || !a.mailbox[0] || ((a.R > 1 || a.n > kBlockRows) && !a.staging)))
        return 108;   // as FLTrust's: phase D reads the staged rows
    if ((a.rule == kGeoMedian || a.rule == kCenteredClipping) && a.R > 1 && !a.staging)
        return 108;   // the passes after the first re-read the staged copy instead of the peers' rows
    if (a.first_seg > 0 && !a.seg_partials)
        return 108;
    if (a.rule == kDnc && (!a.mailbox[0] || !a.dnc_scratch))
        return 108;
    if (a.rule == kDnc && a.first_seg > 0)
        return 111;   // DnC's sampled pass runs in its finish kernel: nothing is pre-accumulated
    if (a.mix && (!a.cta_partials || !a.mailbox[0] || !a.staging))
        return 108;   // NNM mixes, ARC clips the staged tile in place
    if (a.mix && a.first_seg > 0)
        return 111;   // NNM's raw distance pass, ARC's norm pass and bucketing's mean pass cover every segment: nothing is pre-accumulated
    if (a.R > 1 && !a.signal[0])
        return 109;
    if (a.n > kBlockRows && a.R > 1 && (a.rule == kKrum || a.rule == kBulyan || a.rule == kMda || a.rule == kSmea) && !a.staging)
        return 110;   // blocked passes over remote rows need the staged copy
    return 0;
}

} // namespace

extern "C" {

char const* agb_op_list() {
    return "gar_fused,gar_phase_a,gar_max_ctas,gar_byzantine,gar_byzantine_optimized,gar_byzantine_mimic,sgd,worker_momentum,drop_chunks,checksum,cast_bf16";
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
    out[1] = static_cast<long long>(kMailboxFloats) * 4;
    return 0;
}

// The finish kernel (whole aggregation when nothing was pre-accumulated), on at most `max_ctas` CTAs (0: no bound); the DnC and SMEA
// scratch holds `scratch_elems` elements (DnC: floats, SMEA: doubles). `args` points to a `GarArgs` (typed `void const*` since a
// parameter of a type of this file's anonymous namespace would hide the export); its entries past the n_rows rows, the R ranks and the
// nseg segments are null or zero.
int agb_gar_fused(void const* args, int max_ctas, long long scratch_elems, void* stream) {
    GarArgs a = *static_cast<GarArgs const*>(args);
    int const status = check_args(a);
    if (status)
        return status;
    long long total = 0;
    for (int s = 0; s < a.nseg; ++s)
        total += a.seg_hi[s] - a.seg_lo[s];
    if (total == 0 && a.R == 1)
        return 0;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    // the instance follows the rule's n rows (with bucketing n <= n_rows; the mean pass loops over the gathered rows), so the rule adds
    // in the same order as on n plain rows
    if (a.n <= 8)
        return launch<8, 4>(a, max_ctas, scratch_elems, s);
    if (a.n <= 16)
        return launch<16, 4>(a, max_ctas, scratch_elems, s);
    return launch<32, 1>(a, max_ctas, scratch_elems, s);
}

// Phase A (partial pairwise distances + local staging) of owned segment `seg` alone, on `ctas` CTAs: launched on a side stream as soon as
// the backward pass has produced that bucket of gradients; the finish kernel is then called with first_seg > seg.
int agb_gar_phase_a(void const* args, int seg, int ctas, int threads, void* stream) {
    GarArgs const& a = *static_cast<GarArgs const*>(args);
    int const status = check_args(a);
    if (status)
        return status;
    if (a.rule == kFoolsgold)
        return 129;
    if (seg < 0 || seg >= a.nseg || ctas < 1 || ctas > a.seg_max_ctas || !a.seg_partials || (a.rule != kKrum && a.rule != kBulyan && a.rule != kMda && a.rule != kSmea) ||
        a.mix)
        return 111;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    // small CTAs: a 64-thread CTA (8 K registers, 13 KB of static shared memory) fits beside a persistent GEMM CTA of the backward pass
    // (320 threads x 168 registers, ~198 KB), so the distance pass shares SMs with it instead of taking them away
    threads = threads >= 32 && threads <= 256 ? (threads / 32) * 32 : 64;
    if (a.n <= kBlockRows)
        gar_phase_a_kernel<false><<<ctas, threads, 0, s>>>(a, seg);
    else
        gar_phase_a_kernel<true><<<ctas, threads < 64 ? 64 : threads, 0, s>>>(a, seg);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

// The host prologue of the five crafting entry points: checks the workers, ranks and rank (100), the segment count (101), then returns
// `before_masks` if nonzero (an export's own check of its mode), checks the slot masks (114: disjoint, inside [0, n), at least one
// Byzantine slot), returns `after_masks` if nonzero, checks the segment bounds (101) and, rank by rank, the signal pads (109, R > 1) and,
// with `need_mailboxes`, the mailboxes (108). It fills the rows (the honest ones also as `grad` [0, H) with n = H, for
// `phase_a_segment`), the slot masks, the owned segments (`work`: their float4 count), the ranks, their signal pads and mailboxes and the
// epoch. Returns a status.
static int craft_args(ByzArgs& a, unsigned long long const* rows, int n, long long const* seg_lo, long long const* seg_hi, int nseg,
                      unsigned honest, unsigned byzantine, int before_masks, int after_masks, int R, int rank,
                      unsigned long long const* signals, unsigned long long const* mailboxes, bool need_mailboxes, unsigned epoch,
                      unsigned long long epoch_ptr, long long& work) {
    if (n < 1 || n > kMaxWorkers || R < 1 || R > kMaxRanks || rank < 0 || rank >= R)
        return 100;
    if (nseg < 1 || nseg > kMaxSeg)
        return 101;
    if (before_masks)
        return before_masks;
    unsigned const all = n == 32 ? 0xffffffffu : (1u << n) - 1u;
    if ((honest & byzantine) || (honest & ~all) || (byzantine & ~all) || !byzantine)
        return 114;
    if (after_masks)
        return after_masks;
    a.H = __builtin_popcount(honest);
    a.K = __builtin_popcount(byzantine);
    a.n = a.H;
    a.honest_mask = honest;
    for (int i = 0, h = 0, b = 0; i < n; ++i) {
        a.rows[i] = reinterpret_cast<float*>(rows[i]);
        if ((honest >> i) & 1u) {
            a.grad[h] = a.rows[i];
            a.honest[h++] = i;
        }
        if ((byzantine >> i) & 1u)
            a.byz[b++] = i;
    }
    a.nseg = nseg;
    work = 0;
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
        a.mailbox[q] = reinterpret_cast<float*>(mailboxes ? mailboxes[q] : 0ull);
        if (R > 1 && !a.signal[q])
            return 109;
        if (need_mailboxes && !a.mailbox[q])
            return 108;
    }
    a.epoch = epoch;
    a.epoch_ptr = reinterpret_cast<uint32_t*>(epoch_ptr);
    return 0;
}

constexpr int kCraftThreads = 256;

// Grid of a plain crafting launch: one thread per float4 of the owned work, at most 8 CTAs per SM, and at least one CTA: a rank without
// owned coordinates still signals its peers.
static int plain_grid(long long work) {
    long long const grid = (work + kCraftThreads - 1) / kCraftThreads;
    long long const cap = static_cast<long long>(agb::sm_count()) * 8;
    return static_cast<int>(grid < 1 ? 1 : grid > cap ? cap : grid);
}

// Cooperative launch of a crafting kernel over `work` float4s: at most the CTAs that fit on the device at once and `partial_ctas` (the
// CTA slots of the scratch), and at least one CTA: a rank without owned coordinates still posts and signals. The grid depends only on the
// owned work (and the device): the fused engine at R = 1 and the stand-alone op on the same rows fold the same partials in the same order.
static int launch_cooperative(void const* kernel, ByzArgs& a, long long work, int partial_ctas, cudaStream_t stream) {
    int per_sm = 0;
    AGB_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kCraftThreads, 0));
    if (per_sm < 1)
        return 2;
    long long grid = (work + kCraftThreads - 1) / kCraftThreads;
    long long cap = static_cast<long long>(agb::sm_count()) * per_sm;
    cap = cap > partial_ctas ? partial_ctas : cap;
    grid = grid < 1 ? 1 : grid > cap ? cap : grid;
    void* params[] = {&a};
    AGB_CUDA_OK(cudaLaunchCooperativeKernel(kernel, dim3(static_cast<unsigned>(grid)), dim3(kCraftThreads), params, 0, stream));
    return 0;
}

// Omniscient Byzantine rows (ALIE: mode 0, coef = z; IPM: mode 1, coef = epsilon) over this rank's owned segments; see
// `gar_byzantine_kernel`. `rows`: n row addresses; `honest` / `byzantine`: disjoint slot masks; `signals`: R signal pads (R > 1);
// flags use *epoch_ptr + 1 when `epoch_ptr` is set, `epoch` otherwise. Collective when R > 1: every rank calls it.
int agb_gar_byzantine(unsigned long long const* rows, int n, long long const* seg_lo, long long const* seg_hi, int nseg, unsigned honest,
                      unsigned byzantine, int mode, float coef, int R, int rank, unsigned long long const* signals, unsigned epoch,
                      unsigned long long epoch_ptr, void* stream) {
    bool const bad_rows = __builtin_popcount(honest) < (mode == kAlie ? 2 : 1) || (mode != kAlie && mode != kIpm);
    ByzArgs a{};
    long long work = 0;
    int const status = craft_args(a, rows, n, seg_lo, seg_hi, nseg, honest, byzantine, 0, bad_rows ? 114 : 0, R, rank, signals, nullptr,
                                  false, epoch, epoch_ptr, work);
    if (status)
        return status;
    a.mode = mode;
    a.coef = coef;
    if (work == 0 && R == 1)
        return 0;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (a.H <= kBlockRows)
        gar_byzantine_kernel<kBlockRows><<<plain_grid(work), kCraftThreads, 0, s>>>(a);
    else
        gar_byzantine_kernel<0><<<plain_grid(work), kCraftThreads, 0, s>>>(a);
    AGB_CUDA_OK(cudaGetLastError());
    return 0;
}

// Min-Max (mode 2) / Min-Sum (mode 3) with deviation 0 unit-vec, 1 sign, 2 std, over this rank's owned segments; see
// `gar_optimized_kernel`. Arguments as `agb_gar_byzantine`, plus: `mailboxes`: R mailbox addresses (every rank's, its own at `rank`);
// `partials`: [partial_ctas][561] floats of scratch (the grid never exceeds partial_ctas CTAs); `stats_out`: optional [562] floats,
// gamma then the statistics summed over the ranks ([0, 496) honest pair distances, [496, 528) A_i, [528, 560) B_i, [560] C).
// Cooperative launch; collective when R > 1.
int agb_gar_byzantine_optimized(unsigned long long const* rows, int n, long long const* seg_lo, long long const* seg_hi, int nseg, unsigned honest,
                                unsigned byzantine, int mode, int deviation, int R, int rank, unsigned long long const* signals,
                                unsigned long long const* mailboxes, unsigned long long partials, int partial_ctas, unsigned long long stats_out,
                                unsigned epoch, unsigned long long epoch_ptr, void* stream) {
    bool const bad_mode = (mode != kMinMax && mode != kMinSum) || deviation < kUnitVec || deviation > kStd;
    ByzArgs a{};
    long long work = 0;
    int const status = craft_args(a, rows, n, seg_lo, seg_hi, nseg, honest, byzantine, bad_mode ? 118 : 0,
                                  __builtin_popcount(honest) < 2 ? 114 : 0, R, rank, signals, mailboxes, true, epoch, epoch_ptr, work);
    if (status)
        return status;
    a.mode = mode;
    a.deviation = deviation;
    a.partials = reinterpret_cast<float*>(partials);
    a.stats_out = reinterpret_cast<float*>(stats_out);
    if (!a.partials || partial_ctas < 1)
        return 108;
    return launch_cooperative(a.H <= kBlockRows ? reinterpret_cast<void const*>(gar_optimized_kernel<kBlockRows>)
                                                : reinterpret_cast<void const*>(gar_optimized_kernel<0>),
                              a, work, partial_ctas, static_cast<cudaStream_t>(stream));
}

// Mimic over this rank's owned segments; see `gar_mimic_warmup_kernel`. Arguments as `agb_gar_byzantine_optimized`, plus: `warmup`: 1 runs
// the warm-up update number t + 1 (`z`, `y`: local fp32 buffers of the owned coordinates, segments back to back: the direction estimate
// and its scratch), 0 the copy pass alone;
// `istar`: [1] local int32, the target slot, read and (warm-up) written; `stats_out`: optional [66] float64, s_i [0, 32), q_i [32, 64),
// ||y||^2 [64], 1 / ||y|| [65]. The warm-up is a cooperative launch. Collective when R > 1.
int agb_gar_byzantine_mimic(unsigned long long const* rows, int n, long long const* seg_lo, long long const* seg_hi, int nseg, unsigned honest,
                            unsigned byzantine, int warmup, int t, int R, int rank, unsigned long long const* signals,
                            unsigned long long const* mailboxes, unsigned long long partials, int partial_ctas, unsigned long long z,
                            unsigned long long y, unsigned long long istar, unsigned long long stats_out, unsigned epoch,
                            unsigned long long epoch_ptr, void* stream) {
    bool const bad_args = __builtin_popcount(honest) < 2 || (warmup != 0 && warmup != 1) || t < 0 || t >= (1 << 24) || !istar ||
                          (warmup && (!z || !y));
    ByzArgs a{};
    long long work = 0;
    int const status = craft_args(a, rows, n, seg_lo, seg_hi, nseg, honest, byzantine, 0, bad_args ? 124 : 0, R, rank, signals, mailboxes,
                                  warmup != 0, epoch, epoch_ptr, work);
    if (status)
        return status;
    a.t = t;
    a.z = reinterpret_cast<float*>(z);
    a.y = reinterpret_cast<float*>(y);
    a.istar = reinterpret_cast<int*>(istar);
    a.mimic_stats = reinterpret_cast<double*>(stats_out);
    a.partials = reinterpret_cast<float*>(partials);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (!warmup) {
        if (work == 0 && R == 1)
            return 0;
        gar_mimic_copy_kernel<<<plain_grid(work), kCraftThreads, 0, s>>>(a);
        AGB_CUDA_OK(cudaGetLastError());
        return 0;
    }
    if (!a.partials || partial_ctas < 1)
        return 108;
    return launch_cooperative(a.H <= kBlockRows ? reinterpret_cast<void const*>(gar_mimic_warmup_kernel<kBlockRows>)
                                                : reinterpret_cast<void const*>(gar_mimic_warmup_kernel<0>),
                              a, work, partial_ctas, s);
}

// fang-krum over this rank's owned segments; see `gar_fang_krum_kernel`. Arguments as `agb_gar_byzantine_optimized`, plus: `f`: the rule's
// declared f; `threshold`: finite, > 0; `search`: 0 skips the candidate search (gamma = gamma_max, for timing the passes alone);
// `fang_out`: optional [3] float64, gamma_max, t, selected. Every row must be honest or Byzantine, with n - f - 2 >= 1,
// n - 2K - 1 >= 1 and H >= 2 (status 125 otherwise). Cooperative launch; collective when R > 1.
int agb_gar_byzantine_fang_krum(unsigned long long const* rows, int n, long long const* seg_lo, long long const* seg_hi, int nseg, unsigned honest,
                                unsigned byzantine, int f, float threshold, int search, int R, int rank, unsigned long long const* signals,
                                unsigned long long const* mailboxes, unsigned long long partials, int partial_ctas, unsigned long long stats_out,
                                unsigned long long fang_out, unsigned epoch, unsigned long long epoch_ptr, void* stream) {
    ByzArgs a{};
    long long work = 0;
    int const status = craft_args(a, rows, n, seg_lo, seg_hi, nseg, honest, byzantine, 0, honest ? 0 : 114, R, rank, signals, mailboxes,
                                  false, epoch, epoch_ptr, work);
    if (status)
        return status;
    unsigned const all = n == 32 ? 0xffffffffu : (1u << n) - 1u;
    if ((honest | byzantine) != all || f < 0 || n - f - 2 < 1 || n - 2 * a.K - 1 < 1 || a.H < 2 || !(threshold > 0.f) || !std::isfinite(threshold))
        return 125;
    a.deviation = kSign;
    a.f = f;
    a.coef = threshold;
    a.search = search ? 1 : 0;
    for (int q = 0; q < R; ++q)
        if (!a.mailbox[q])
            return 108;
    a.partials = reinterpret_cast<float*>(partials);
    a.stats_out = reinterpret_cast<float*>(stats_out);
    a.fang_out = reinterpret_cast<double*>(fang_out);
    if (!a.partials || partial_ctas < 1)
        return 108;
    return launch_cooperative(a.H <= kBlockRows ? reinterpret_cast<void const*>(gar_fang_krum_kernel<kBlockRows>)
                                                : reinterpret_cast<void const*>(gar_fang_krum_kernel<0>),
                              a, work, partial_ctas, static_cast<cudaStream_t>(stream));
}

// fang-trim over this rank's owned segments; see `gar_fang_trim_kernel`. Arguments as `agb_gar_byzantine`, plus: `scale`: beta, finite and
// > 1 (status 125 otherwise); `key`: splitmix64(splitmix64(splitmix64(seed) ^ step) ^ TAG) (`_ops.fang_trim_key`). Collective when R > 1.
int agb_gar_byzantine_fang_trim(unsigned long long const* rows, int n, long long const* seg_lo, long long const* seg_hi, int nseg, unsigned honest,
                                unsigned byzantine, float scale, unsigned long long key, int R, int rank, unsigned long long const* signals,
                                unsigned epoch, unsigned long long epoch_ptr, void* stream) {
    ByzArgs a{};
    long long work = 0;
    int const status = craft_args(a, rows, n, seg_lo, seg_hi, nseg, honest, byzantine, 0, honest ? 0 : 114, R, rank, signals, nullptr,
                                  false, epoch, epoch_ptr, work);
    if (status)
        return status;
    if (!(scale > 1.f) || !std::isfinite(scale))
        return 125;
    a.coef = scale;
    a.key = key;
    if (work == 0 && R == 1)
        return 0;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (a.H <= kBlockRows)
        gar_fang_trim_kernel<kBlockRows><<<plain_grid(work), kCraftThreads, 0, s>>>(a);
    else
        gar_fang_trim_kernel<0><<<plain_grid(work), kCraftThreads, 0, s>>>(a);
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
