// Implicit-GEMM k x k convolution (stride 1 or 2, zero padding) on the Hopper tensor cores: no im2col buffer.
//
// Activations are NHWC, so the A operand of the forward GEMM for filter tap (kh, kw) and a 64-channel slice is simply the
// activation tensor shifted by (kh - pad, kw - pad). A 4-D TMA tensor map (C, W, H, N) lets one `cp.async.bulk.tensor.4d`
// fetch a *box of pixels* x 64 channels straight into the 128B-swizzled K-major layout the MMA wants; coordinates that
// fall outside the image are zero-filled by the TMA unit, which is exactly the convolution's padding. The M tile (128
// rows) is a pixel box bw x bh x bn chosen so that it tiles the feature map: 8x8x2 (56x56), 4x4x8 (28x28), 2x2x32 (14x14),
// 7x1x16 (7x7, 112 valid rows) ...
//
//   forward  y[p, co]      = sum_{kh,kw,ci} x[p + (kh-pad, kw-pad), ci] * W[co, kh, kw, ci]       A: 4-D box of x,  B: K-major W
//   dgrad    dx[p, ci]     = sum_{kh,kw,co} dy[p + (pad-kh, pad-kw), co] * W[co, kh, kw, ci]      A: 4-D box of dy, B: MN-major W tap
//   wgrad    dW[co,kh,kw,ci] = sum_p dy[p, co] * x[p + (kh-pad, kw-pad), ci]                       A, B: 4-D MN-major boxes (K = pixels)
//
// Stride 2 (ResNet's down-sampling 3x3 convolutions, `external/slim/nets/resnet_v1.py:123-128`): the forward and weight-gradient
// products read x through a tensor map whose TMA *element strides* are (1, 2, 2, 1) — the box of bw x bh output pixels fetches every
// second input pixel, still one bulk-tensor copy per tap. The data gradient splits dx into its four pixel parities: the pixels
// (2i + ph, 2j + pw) only receive the taps with kh = ph + pad_t (mod 2), kw = pw + pad_l (mod 2), each a stride-1 shifted box of dy,
// so every parity class is a small stride-1 problem (1, 2, 2 and 4 taps for a 3x3 filter) whose epilogue scatters its rows to the
// strided dx addresses.
//
// Pipeline, main loop (wgmma, or mma.sync for TF32) and epilogue are those of the persistent GEMM (gemm_kernels.cuh); only the producer's
// coordinates and the epilogue's row -> address mapping differ.

#include "gemm_kernels.cuh"

namespace {

struct ConvParams {
    int N, H, W;            // input (x / dx) pixel grid
    int OH, OW;             // output (y / dy) pixel grid (= H, W for stride 1 "same" convolutions)
    int Cin, Cout, k, stride, pad_t, pad_l;
    int GH, GW;             // grid the M tiles (fwd, dgrad) or K blocks (wgrad) walk over: fwd/wgrad OH x OW; dgrad H/stride x W/stride per parity
    int bw, bh, bn;         // pixel box of one M tile (fwd/dgrad: product <= 128) or one K block (wgrad: product <= 64)
    int tiles_w, tiles_h, tiles_n;
    int groups, images_per_group;   // wgrad of several logical workers: K ranges = image ranges, one output per group
    int sbw, sbh, sbn;      // staged epilogue of fwd / dgrad: one warp's 16 rows as a sub-box of the pixel box
};

// The 16 consecutive rows (w fastest, then h, then n) of a warp's slab form a sub-box sbw x sbh x sbn of every bw x bh x bn pixel
// box when the widths nest: 8x8x2 -> 8x2x1, 4x4x8 -> 4x4x1, 2x2x32 -> 2x2x4. The 7x1x16 box of the 7x7 maps does not nest.
bool slab_box(int bw, int bh, int bn, int& sbw, int& sbh, int& sbn) {
    if ((bw * bh * bn) % 16)
        return false;
    if (bw >= 16) {
        sbw = 16; sbh = 1; sbn = 1;
        return bw % 16 == 0;
    }
    if (16 % bw)
        return false;
    sbw = bw;
    int const lines = 16 / bw;
    if (bh >= lines) {
        sbh = lines; sbn = 1;
        return bh % lines == 0;
    }
    if (lines % bh)
        return false;
    sbh = bh; sbn = lines / bh;
    return bn % sbn == 0;
}

enum ConvMode { kFwd = 0, kDgrad = 1, kWgrad = 2 };

// `estride` > 1: the box covers bw * estride x bh * estride source pixels and TMA keeps every estride-th one (bw x bh land in smem).
template<typename E>
inline int make_tmap_4d(CUtensorMap* map, void const* base, int C, int W, int H, int N, int bw, int bh, int bn, int estride = 1) {
    constexpr cuuint64_t kB = E::kBytes;
    cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(N)};
    cuuint64_t strides[3] = {static_cast<cuuint64_t>(C) * kB, static_cast<cuuint64_t>(W) * C * kB, static_cast<cuuint64_t>(H) * W * C * kB};
    cuuint32_t box[4] = {static_cast<cuuint32_t>(E::kChunk), static_cast<cuuint32_t>(bw * estride), static_cast<cuuint32_t>(bh * estride), static_cast<cuuint32_t>(bn)};
    cuuint32_t elem[4] = {1, static_cast<cuuint32_t>(estride), static_cast<cuuint32_t>(estride), 1};
    return encode_cached(map, E::kTf32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, dims, strides, box, elem);
}

// One persistent kernel for the three products. `tmap_a`: 4-D map of the activation that plays A (x for fwd, dy for dgrad and
// wgrad); `tmap_b`: 2-D weight map (fwd: K-major rows [Cout][k*k*Cin]; dgrad: the same matrix read as MN-major boxes) or
// the 4-D map of x (wgrad).
template<int BN, int MODE, typename E = ElemBF16>
__global__ void __launch_bounds__(kThreads, 1) conv_sm90_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                                                                    const __grid_constant__ CUtensorMap tmap_c, GemmParams const p, ConvParams const cp, int items_mn, int splits) {
    constexpr bool A_MN = MODE == kWgrad, B_MN = MODE != kFwd;
    using Cfg = Config<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::kRingBytes + kStagingBytes);
    uint64_t* empty = full + Cfg::kStages;

    int const warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int const taps = cp.k * cp.k;
    int const pixel_tiles = cp.tiles_w * cp.tiles_h * cp.tiles_n;
    int const box_rows = cp.bw * cp.bh * cp.bn;
    // number of K blocks of one work item before splitting
    int const cchunks = (MODE == kFwd ? cp.Cin : cp.Cout) / E::kChunk;
    constexpr int kChunkBytes = E::kBK * 128;   // one MN-major chunk of a stage
    int const groups = (MODE == kWgrad && cp.groups > 1) ? cp.groups : 1;
    int const parities = (MODE == kDgrad && cp.stride > 1) ? cp.stride * cp.stride : 1;   // dgrad of a strided convolution: one sub-problem per pixel parity
    int const total_kblocks = MODE == kWgrad ? pixel_tiles / groups : taps * cchunks;     // upper bound per item for dgrad parities (their tap subsets are smaller)
    int const total_items = items_mn * splits * groups;

    // Pixel boxes smaller than the MMA tile (7x7 maps) leave rows that TMA never writes: zero the ring once.
    if (box_rows < (MODE == kWgrad ? E::kBK : 128)) {
        uint4* ring = reinterpret_cast<uint4*>(smem);
        for (uint32_t i = threadIdx.x; i < Cfg::kStages * Cfg::kStageBytes / 16; i += blockDim.x)
            ring[i] = make_uint4(0, 0, 0, 0);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy zeros visible to the async (TMA/MMA) proxy
    }
    if (warp == kProducerWarp && lane == 0) {
        tma_prefetch_desc(&tmap_a);
        tma_prefetch_desc(&tmap_b);
        for (int s = 0; s < Cfg::kStages; ++s) {
            mbar_init(full + s, 1);
            mbar_init(empty + s, kConsumerWarps);   // one arrival per consumer warp
        }
        mbar_fence_init();
    }
    if (p.staged && warp == 0 && lane == 0)
        tma_prefetch_desc(&tmap_c);
    __syncthreads();
    pdl_trigger();   // set-up done: the next kernel may start its own; ...
    pdl_wait();      // ... our inputs are complete only once the previous kernel has finished

    // Bytes that one stage really receives (boxes may be smaller than the tile): A box rows * 128 B per 64-wide chunk.
    uint32_t const a_bytes = MODE == kWgrad ? static_cast<uint32_t>(kBM / E::kChunk) * box_rows * 128u : static_cast<uint32_t>(box_rows) * 128u;
    uint32_t const b_bytes = MODE == kWgrad ? (BN / E::kChunk) * box_rows * 128u : Cfg::kBBytes;

    // item -> (m index, n tile, tap for wgrad, k split)
    // par_h / par_w: pixel parity of a strided dgrad item; first_kh / nkh (and _kw): the taps that reach that parity (kh = first_kh + stride * i)
    struct Item { int pw, ph, pn, n0, tap, kb_begin, nkb, m0, group, par_h, par_w, first_kh, first_kw, nkw; };
    auto decode = [&](int item) {
        Item it;
        it.group = item / (items_mn * splits);
        item -= it.group * items_mn * splits;
        int mn = item % items_mn;
        int const split = item / items_mn;
        it.par_h = it.par_w = it.first_kh = it.first_kw = 0;
        it.nkw = cp.k;
        int item_kblocks = total_kblocks;
        if (parities > 1) {
            int const per_parity = items_mn / parities;
            int const parity = mn / per_parity;
            mn -= parity * per_parity;
            it.par_h = parity / cp.stride;
            it.par_w = parity % cp.stride;
            it.first_kh = (it.par_h + cp.pad_t) % cp.stride;
            it.first_kw = (it.par_w + cp.pad_l) % cp.stride;
            int const nkh = it.first_kh < cp.k ? (cp.k - it.first_kh + cp.stride - 1) / cp.stride : 0;
            it.nkw = it.first_kw < cp.k ? (cp.k - it.first_kw + cp.stride - 1) / cp.stride : 0;
            item_kblocks = nkh * it.nkw * cchunks;
        }
        it.kb_begin = split * p.kblocks_per_split;
        int const kb_end = min(item_kblocks, it.kb_begin + p.kblocks_per_split);
        it.nkb = max(kb_end - it.kb_begin, 0);
        if (MODE == kWgrad) {
            int const m_tiles = (cp.Cout + kBM - 1) / kBM, n_tiles = (cp.Cin + BN - 1) / BN;
            it.tap = mn / (m_tiles * n_tiles);
            int const rest = mn % (m_tiles * n_tiles);
            it.m0 = (rest % m_tiles) * kBM;      // output-channel offset
            it.n0 = (rest / m_tiles) * BN;       // input-channel offset
            it.pw = it.ph = it.pn = 0;
        } else {
            int const tile = mn % pixel_tiles;
            it.n0 = (mn / pixel_tiles) * BN;
            it.pw = (tile % cp.tiles_w) * cp.bw;
            it.ph = ((tile / cp.tiles_w) % cp.tiles_h) * cp.bh;
            it.pn = (tile / (cp.tiles_w * cp.tiles_h)) * cp.bn;
            it.tap = 0;
            it.m0 = 0;
        }
        return it;
    };

    if (warp >= kProducerWarp) {
        producer_registers();
        if (warp == kProducerWarp && lane == 0) {
            uint32_t ring = 0;
            for (int item = blockIdx.x; item < total_items; item += gridDim.x) {
                Item const it = decode(item);
                for (int i = 0; i < it.nkb; ++i, ++ring) {
                    int const s = ring % Cfg::kStages;
                    mbar_wait(empty + s, ((ring / Cfg::kStages) & 1) ^ 1, 1);
                    uint8_t* a_dst = smem + s * Cfg::kStageBytes;
                    uint8_t* b_dst = a_dst + Cfg::kABytes;
                    int const kb = it.kb_begin + i;
                    mbar_expect_tx(full + s, a_bytes + b_bytes);
                    if (MODE == kWgrad) {
                        // K block = pixel box `kb` of the dy grid; A = dy[box, co chunk], B = x[box * stride shifted by the tap, ci chunk]
                        int const w0 = (kb % cp.tiles_w) * cp.bw, h0 = ((kb / cp.tiles_w) % cp.tiles_h) * cp.bh;
                        int const n0p = (kb / (cp.tiles_w * cp.tiles_h)) * cp.bn + it.group * cp.images_per_group;
                        int const kh = it.tap / cp.k, kw = it.tap % cp.k;
#pragma unroll
                        for (int c = 0; c < kBM / E::kChunk; ++c)
                            tma_load_4d(a_dst + c * kChunkBytes, &tmap_a, full + s, it.m0 + c * E::kChunk, w0, h0, n0p);
#pragma unroll
                        for (int c = 0; c < BN / E::kChunk; ++c)
                            tma_load_4d(b_dst + c * kChunkBytes, &tmap_b, full + s, it.n0 + c * E::kChunk, w0 * cp.stride + kw - cp.pad_l, h0 * cp.stride + kh - cp.pad_t, n0p);
                    } else {
                        int const tap_index = kb / cchunks, c0 = (kb % cchunks) * E::kChunk;
                        int kh, kw, dw, dh;
                        if (MODE == kFwd) {         // x[oh * s + kh - pad_t, ow * s + kw - pad_l]: the map's element strides do the "* s"
                            kh = tap_index / cp.k; kw = tap_index % cp.k;
                            dw = it.pw * (cp.stride - 1) + kw - cp.pad_l;
                            dh = it.ph * (cp.stride - 1) + kh - cp.pad_t;
                        } else if (parities == 1) { // dy[h + pad_t - kh, w + pad_l - kw]
                            kh = tap_index / cp.k; kw = tap_index % cp.k;
                            dw = cp.pad_l - kw; dh = cp.pad_t - kh;
                        } else {                    // pixel (s*i + par_h, s*j + par_w) <- dy[i + (par_h + pad_t - kh) / s, j + (par_w + pad_l - kw) / s], kh = par_h + pad_t (mod s)
                            kh = it.first_kh + cp.stride * (tap_index / it.nkw); kw = it.first_kw + cp.stride * (tap_index % it.nkw);
                            dh = (it.par_h + cp.pad_t - kh) / cp.stride;   // exact: the numerator is a multiple of the stride (may be negative)
                            dw = (it.par_w + cp.pad_l - kw) / cp.stride;
                        }
                        int const tap = kh * cp.k + kw;
                        tma_load_4d(a_dst, &tmap_a, full + s, c0, it.pw + dw, it.ph + dh, it.pn);
                        if (MODE == kFwd) {
                            tma_load_2d(b_dst, &tmap_b, full + s, tap * cp.Cin + c0, it.n0);
                        } else { // dgrad: B[k = co, n = ci] = W[co][tap][ci]: MN-major boxes of 64 ci x 64 co
#pragma unroll
                            for (int c = 0; c < BN / E::kChunk; ++c)
                                tma_load_2d(b_dst + c * kChunkBytes, &tmap_b, full + s, tap * cp.Cin + it.n0 + c * E::kChunk, c0);
                        }
                    }
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
        Item const it = decode(item);
        mainloop<BN, A_MN, B_MN, E>(smem, full, empty, ring, it.nkb, warp, acc);
        if (p.staged) {
            if (MODE == kWgrad) {   // output map (Cin, taps, Cout, groups)
                epilogue_staged<BN>(p, &tmap_c, acc, staging, issued, it.n0, [&](int col, int (&c)[4]) {
                    c[0] = col; c[1] = it.tap; c[2] = it.m0 + 16 * warp; c[3] = it.group;
                });
            } else if (16 * warp < box_rows) {   // output map (C, W, H, N) of y / dx; the slab is a sbw x sbh x sbn sub-box
                int const r = 16 * warp;
                int const bi_w = r % cp.bw, bi_h = (r / cp.bw) % cp.bh, bi_n = r / (cp.bw * cp.bh);
                epilogue_staged<BN>(p, &tmap_c, acc, staging, issued, it.n0, [&](int col, int (&c)[4]) {
                    c[0] = col; c[1] = it.pw + bi_w; c[2] = it.ph + bi_h; c[3] = it.pn + bi_n;
                });
            }
            continue;
        }
        epilogue_slab<BN>(p, acc, 16 * warp, it.n0, [&](int r, bool& valid, long long& offset) {
            if (MODE == kWgrad) {   // row = output channel; columns = (tap, ci) inside dW[Cout][k*k*Cin]
                int const co = it.m0 + r;
                valid = co < cp.Cout;
                offset = static_cast<long long>(co) * p.ldc + it.tap * cp.Cin + it.group * p.c_group_stride;
            } else {                // row = pixel of the box, (w fastest, then h, then n)
                int const bi_w = r % cp.bw, bi_h = (r / cp.bw) % cp.bh, bi_n = r / (cp.bw * cp.bh);
                int const gw = it.pw + bi_w, gh = it.ph + bi_h, n = it.pn + bi_n;
                valid = r < box_rows && gw < cp.GW && gh < cp.GH && n < cp.N;
                if (MODE == kFwd)      // y[n, gh, gw]
                    offset = ((static_cast<long long>(n) * cp.OH + gh) * cp.OW + gw) * p.ldc;
                else                   // dx[n, gh * s + parity_h, gw * s + parity_w] (s = 1: the pixel itself)
                    offset = ((static_cast<long long>(n) * cp.H + gh * cp.stride + it.par_h) * cp.W + gw * cp.stride + it.par_w) * p.ldc;
            }
        });
    }
    if (p.staged && lane == 0)
        bulk_wait_all();   // outputs complete (and staging read) before the CTA retires: PDL dependents and graph replays see them
}

// Output map of the staged epilogue; false leaves the register epilogue in charge: the strided data gradient (its rows scatter to
// one pixel parity of dx), pixel boxes whose 16-row slabs are not sub-boxes (7x1x16), outputs TMA cannot address.
template<int MODE>
bool conv_out_map(CUtensorMap* map, GemmParams const& p, ConvParams& cp) {
    if (MODE == kWgrad) {   // dW[group][Cout][taps][Cin]
        uint64_t const taps = static_cast<uint64_t>(cp.k) * cp.k, groups = cp.groups > 1 ? cp.groups : 1;
        uint64_t const gstride = groups > 1 ? static_cast<uint64_t>(p.c_group_stride) : static_cast<uint64_t>(p.ldc) * cp.Cout;
        uint64_t const dims[4] = {static_cast<uint64_t>(cp.Cin), taps, static_cast<uint64_t>(cp.Cout), groups};
        uint64_t const strides[3] = {static_cast<uint64_t>(cp.Cin), static_cast<uint64_t>(p.ldc), gstride};
        uint32_t const box[3] = {1, 16, 1};
        return make_tmap_out(map, p.C, p.out_fp32, dims, strides, box);
    }
    if (MODE == kDgrad && cp.stride > 1)
        return false;
    if (!slab_box(cp.bw, cp.bh, cp.bn, cp.sbw, cp.sbh, cp.sbn))
        return false;
    int const C = MODE == kFwd ? cp.Cout : cp.Cin, W = MODE == kFwd ? cp.OW : cp.W, H = MODE == kFwd ? cp.OH : cp.H;   // y or dx, NHWC
    uint64_t const dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(W), static_cast<uint64_t>(H), static_cast<uint64_t>(cp.N)};
    uint64_t const strides[3] = {static_cast<uint64_t>(C), static_cast<uint64_t>(W) * C, static_cast<uint64_t>(H) * W * C};
    uint32_t const box[3] = {static_cast<uint32_t>(cp.sbw), static_cast<uint32_t>(cp.sbh), static_cast<uint32_t>(cp.sbn)};
    return make_tmap_out(map, p.C, p.out_fp32, dims, strides, box);
}

template<int BN, int MODE, typename E = ElemBF16>
int launch_conv(CUtensorMap const& ta, CUtensorMap const& tb, GemmParams const& params, ConvParams const& conv, int items_mn, int splits, cudaStream_t stream) {
    using Cfg = Config<BN>;
    GemmParams p = params;
    ConvParams cp = conv;
    CUtensorMap tc;
    std::memset(&tc, 0, sizeof(tc));
    p.staged = agb_gemm_epilogue_staged() && conv_out_map<MODE>(&tc, p, cp);
    auto kernel = conv_sm90_kernel<BN, MODE, E>;
    static bool configured = false;
    if (!configured) {
        AGB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
        configured = true;
    }
    int const sms = sm_count();
    long long const items = static_cast<long long>(items_mn) * splits * ((MODE == kWgrad && cp.groups > 1) ? cp.groups : 1);
    int const grid = static_cast<int>(items < sms ? items : sms);
    AGB_CUDA_OK(launch_pdl(kernel, dim3(grid), dim3(kThreads), Cfg::kSmemBytes, stream, ta, tb, tc, p, cp, items_mn, splits));
    return 0;
}

// Pixel box (bw, bh, bn) with bw*bh*bn <= rows, bw | W-tiles etc. Prefers exact tilings of the feature map.
bool choose_box(int W, int H, int N, int rows, int& bw, int& bh, int& bn) {
    long long best = -1;
    for (int w = 1; w <= W && w <= rows; ++w) {
        if (W % w)
            continue;
        for (int h = 1; h <= H && w * h <= rows; ++h) {
            if (H % h)
                continue;
            int n = rows / (w * h);
            if (n > N)
                n = N;
            while (n > 1 && N % n)
                --n;
            // prefer full MMA tiles, then spatially compact boxes (halo reuse in L2), then wide rows (long TMA runs)
            long long const score = static_cast<long long>(w) * h * n * 1000000 + static_cast<long long>(w) * h * 1000 + w;
            if (score > best) {
                best = score;
                bw = w; bh = h; bn = n;
            }
        }
    }
    return best >= 0;
}

template<typename E>
int conv_implicit_impl(int mode, void const* act, void const* other, void* out, int N, int H, int W, int OH, int OW, int Cin, int Cout, int k, int stride, int pad_t, int pad_l,
                              void const* bias, int relu, int out_fp32, int splits, int bn, int groups, long long c_group_stride, void* stream) {
    if (k < 1 || Cin % E::kChunk || Cout % E::kChunk || N < 1 || (stride != 1 && stride != 2) || pad_t < 0 || pad_l < 0 || pad_t >= k || pad_l >= k)
        return 401;
    if (stride == 2 && ((H & 1) || (W & 1) || OH != H / 2 || OW != W / 2 || k < 2))
        return 405;
    if (stride == 1 && (OH != H || OW != W))
        return 405;
    if (groups < 1)
        groups = 1;
    if (groups > 1 && (mode != 2 || N % groups))
        return 404;
    ConvParams cp{};
    cp.N = N; cp.H = H; cp.W = W; cp.OH = OH; cp.OW = OW; cp.Cin = Cin; cp.Cout = Cout; cp.k = k; cp.stride = stride; cp.pad_t = pad_t; cp.pad_l = pad_l;
    cp.groups = groups; cp.images_per_group = N / groups;
    // the grid the boxes tile: output pixels (fwd, wgrad) or, for the data gradient, the pixels of one parity class of dx
    cp.GH = mode == 1 ? H / stride : OH;
    cp.GW = mode == 1 ? W / stride : OW;
    if (!choose_box(cp.GW, cp.GH, mode == 2 ? N / groups : N, mode == 2 ? E::kBK : 128, cp.bw, cp.bh, cp.bn))   // boxes never straddle two workers
        return 402;
    cp.tiles_w = cp.GW / cp.bw; cp.tiles_h = cp.GH / cp.bh; cp.tiles_n = N / cp.bn;
    int const pixel_tiles = cp.tiles_w * cp.tiles_h * cp.tiles_n;
    GemmParams p{};
    p.C = out;
    p.bias = static_cast<float const*>(bias);
    p.relu = relu;
    p.out_fp32 = out_fp32;
    CUtensorMap ta, tb;
    int status, items_mn, total_kblocks;
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (mode == 0) {
        p.M = N * OH * OW; p.N = Cout; p.K = k * k * Cin; p.ldc = Cout;
        if (bn == 0)
            bn = Cout <= 64 ? 64 : 128;
        if ((status = make_tmap_4d<E>(&ta, act, Cin, W, H, N, cp.bw, cp.bh, cp.bn, stride)))
            return status;
        if ((status = make_tmap_2d(&tb, other, static_cast<uint64_t>(k) * k * Cin, Cout, static_cast<uint64_t>(k) * k * Cin, E::kBK, bn, E::kBytes)))
            return status;
        items_mn = pixel_tiles * ((Cout + bn - 1) / bn);
        total_kblocks = k * k * (Cin / E::kChunk);
    } else if (mode == 1) {
        p.M = N * H * W; p.N = Cin; p.K = k * k * Cout; p.ldc = Cin;
        if (bn == 0)
            bn = Cin <= 64 ? 64 : 128;
        if ((status = make_tmap_4d<E>(&ta, act, Cout, OW, OH, N, cp.bw, cp.bh, cp.bn)))
            return status;
        if ((status = make_tmap_2d(&tb, other, static_cast<uint64_t>(k) * k * Cin, Cout, static_cast<uint64_t>(k) * k * Cin, E::kChunk, E::kBK, E::kBytes)))
            return status;
        items_mn = pixel_tiles * ((Cin + bn - 1) / bn) * stride * stride;   // one sub-problem per pixel parity
        total_kblocks = k * k * (Cout / E::kChunk);
        if (stride > 1 && splits > 1)
            return 406;
    } else if (mode == 2) {
        p.M = Cout; p.N = Cin; p.K = N * OH * OW; p.ldc = static_cast<long long>(k) * k * Cin;
        if (!out_fp32)
            return 205;
        if (bn == 0)
            bn = Cin <= 64 ? 64 : 128;
        if ((status = make_tmap_4d<E>(&ta, act, Cout, OW, OH, N, cp.bw, cp.bh, cp.bn)))
            return status;
        if ((status = make_tmap_4d<E>(&tb, other, Cin, W, H, N, cp.bw, cp.bh, cp.bn, stride)))
            return status;
        items_mn = k * k * ((Cout + kBM - 1) / kBM) * ((Cin + bn - 1) / bn);
        total_kblocks = pixel_tiles / groups;
    } else {
        return 403;
    }
    if (splits < 1)
        splits = 1;
    if (splits > total_kblocks)
        splits = total_kblocks;
    if (splits > 1 && !out_fp32)
        return 205;
    p.atomic = splits > 1;
    p.groups = groups; p.c_group_stride = c_group_stride;
    p.kblocks_per_split = (total_kblocks + splits - 1) / splits;
    splits = (total_kblocks + p.kblocks_per_split - 1) / p.kblocks_per_split;
#define AGB_CONV_DISPATCH(MODE) \
    switch (bn) { \
        case 64: return launch_conv<64, MODE, E>(ta, tb, p, cp, items_mn, splits, s); \
        case 128: return launch_conv<128, MODE, E>(ta, tb, p, cp, items_mn, splits, s); \
    } \
    return 203;
    if (mode == 0) { AGB_CONV_DISPATCH(kFwd) }
    if (mode == 1) { AGB_CONV_DISPATCH(kDgrad) }
    AGB_CONV_DISPATCH(kWgrad)
#undef AGB_CONV_DISPATCH
}

} // namespace

extern "C" {

// mode 0: y = conv(x, W) (+bias, ReLU) ; mode 1: dx = conv_transpose(dy, W) ; mode 2: dW (+)= dy^T * x (fp32, atomics; caller zeroes).
// x / dx are NHWC bf16 with N x H x W pixels, y / dy with N x OH x OW pixels, OH = (H + pad_t + pad_b - k) / stride + 1 (the bottom / right
// padding is implied: whatever the boxes read beyond the image is zero). stride 1 or 2; W is [Cout][k][k][Cin] bf16; dW is
// [Cout][k][k][Cin] fp32. Cin % 64 == 0 and Cout % 64 == 0. For stride 2: H, W even, OH = H / 2, OW = W / 2.
int agb_conv_implicit_strided(int mode, void const* act, void const* other, void* out, int N, int H, int W, int OH, int OW, int Cin, int Cout, int k, int stride, int pad_t, int pad_l,
                              void const* bias, int relu, int out_fp32, int splits, int bn, int groups, long long c_group_stride, void* stream);

int agb_conv_implicit_grouped(int mode, void const* act, void const* other, void* out, int N, int H, int W, int Cin, int Cout, int k, void const* bias, int relu,
                              int out_fp32, int splits, int bn, int groups, long long c_group_stride, void* stream) {
    if ((k & 1) == 0)
        return 401;
    return agb_conv_implicit_strided(mode, act, other, out, N, H, W, H, W, Cin, Cout, k, 1, (k - 1) / 2, (k - 1) / 2, bias, relu, out_fp32, splits, bn, groups, c_group_stride, stream);
}

int agb_conv_implicit(int mode, void const* act, void const* other, void* out, int N, int H, int W, int Cin, int Cout, int k, void const* bias, int relu,
                      int out_fp32, int splits, int bn, void* stream) {
    return agb_conv_implicit_grouped(mode, act, other, out, N, H, W, Cin, Cout, k, bias, relu, out_fp32, splits, bn, 1, 0, stream);
}

// `groups` > 1 (mode 2 only): the N images are `groups` consecutive batches of N / groups images; group g accumulates its weight gradient
// into out + g * c_group_stride.
int agb_conv_implicit_strided(int mode, void const* act, void const* other, void* out, int N, int H, int W, int OH, int OW, int Cin, int Cout, int k, int stride, int pad_t, int pad_l,
                              void const* bias, int relu, int out_fp32, int splits, int bn, int groups, long long c_group_stride, void* stream) {
    return conv_implicit_impl<ElemBF16>(mode, act, other, out, N, H, W, OH, OW, Cin, Cout, k, stride, pad_t, pad_l, bias, relu, out_fp32, splits, bn, groups, c_group_stride, stream);
}

// fp32 activations / weights multiplied as TF32; channel counts multiples of 32; outputs are fp32.
int agb_conv_implicit_strided_tf32(int mode, void const* act, void const* other, void* out, int N, int H, int W, int OH, int OW, int Cin, int Cout, int k, int stride, int pad_t, int pad_l,
                                   void const* bias, int relu, int splits, int bn, int groups, long long c_group_stride, void* stream) {
    return conv_implicit_impl<ElemTF32>(mode, act, other, out, N, H, W, OH, OW, Cin, Cout, k, stride, pad_t, pad_l, bias, relu, 1, splits, bn, groups, c_group_stride, stream);
}

} // extern "C"
