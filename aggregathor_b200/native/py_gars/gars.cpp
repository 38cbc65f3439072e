// Host (CPU) gradient aggregation rules — C ABI, loaded through ctypes.
//
// These are the gloo/CPU-mode implementations and the oracles of the sm_90a
// kernels. They cover what the reference spreads over `native/op_krum/cpu.cpp`,
// `native/op_bulyan/cpu.cpp` and `aggregators/deprecated_native/native.cpp`
// (median :678-705, averaged-median :714-748, average-nan :756-783, squared
// distance :637-668), with two deliberate differences required by SPMD use:
//   * every reduction has a fixed summation order (chunked, folded in chunk order);
//   * every ordering is total: finite values first (ascending), non-finite last,
//     ties broken by the lower worker index. All ranks therefore select the same set.
// Inputs are a row-major [n, d] matrix (one flattened gradient per row).

#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <limits>
#include <vector>

#include <agb_threadpool.hpp>

namespace {

using agb::global_pool;
using agb::ThreadPool;

constexpr size_t kGrainCoord = 1 << 14; // coordinates per chunk for coordinate-wise loops
constexpr size_t kMaxWorkers = 1024;

// (finite, value, index) strict weak order: finite ascending, then non-finite, ties by index.
template<class T> inline bool before(T a, size_t ia, T b, size_t ib) {
    bool fa = std::isfinite(a), fb = std::isfinite(b);
    if (fa != fb)
        return fa;
    if (fa && a != b)
        return a < b;
    return ia < ib;
}

// ------------------------------------------------------------------------ //
// Pairwise squared distances, deterministic: per-chunk partial matrices folded in chunk order.
// sum_{k in [b, e)} (x[k] - y[k])^2 with 16 interleaved partial sums folded in a fixed tree: the association is fixed (hence
// deterministic) but no longer one serial chain, so the loop vectorises instead of waiting 4 cycles per addition.
template<class T> inline T squared_difference(T const* x, T const* y, size_t b, size_t e) {
    constexpr size_t kLanes = 16;
    T acc[kLanes];
    for (size_t u = 0; u < kLanes; ++u)
        acc[u] = T(0);
    size_t k = b;
    for (; k + kLanes <= e; k += kLanes)
        for (size_t u = 0; u < kLanes; ++u) {
            T const delta = x[k + u] - y[k + u];
            acc[u] += delta * delta;
        }
    for (size_t u = 0; k < e; ++k, ++u) {
        T const delta = x[k] - y[k];
        acc[u] += delta * delta;
    }
    for (size_t width = kLanes / 2; width > 0; width /= 2)
        for (size_t u = 0; u < width; ++u)
            acc[u] += acc[u + width];
    return acc[0];
}

template<class T> void pairwise_distances(T const* g, size_t n, size_t d, T* dist /* [n*n] */) {
    size_t const grain = kGrainCoord;
    size_t const chunks = ThreadPool::chunk_count(0, d, grain);
    size_t const pairs = n * (n - 1) / 2;
    std::vector<T> partial(chunks * pairs, T(0));
    global_pool().run(0, d, grain, [&](size_t chunk, size_t b, size_t e) {
        T* out = partial.data() + chunk * pairs;
        size_t p = 0;
        for (size_t i = 0; i + 1 < n; ++i) {
            T const* x = g + i * d;
            for (size_t j = i + 1; j < n; ++j, ++p) {
                T const* y = g + j * d;
                out[p] = squared_difference(x, y, b, e);
            }
        }
    });
    size_t p = 0;
    for (size_t i = 0; i < n; ++i)
        dist[i * n + i] = 0;
    for (size_t i = 0; i + 1 < n; ++i) {
        for (size_t j = i + 1; j < n; ++j, ++p) {
            T sum = 0;
            for (size_t c = 0; c < chunks; ++c)
                sum += partial[c * pairs + p];
            if (!std::isfinite(sum))
                sum = std::numeric_limits<T>::infinity();
            dist[i * n + j] = sum;
            dist[j * n + i] = sum;
        }
    }
}

// Krum scores: sum of the `count` smallest distances of each row (self excluded).
// `order` (optional, [n*(n-1)]) receives, per row, the other workers sorted by distance.
template<class T> void krum_scores(T const* dist, size_t n, size_t count, T* scores, size_t* order) {
    std::vector<size_t> idx(n);
    for (size_t i = 0; i < n; ++i) {
        size_t len = 0;
        for (size_t j = 0; j < n; ++j)
            if (j != i)
                idx[len++] = j;
        T const* row = dist + i * n;
        std::sort(idx.begin(), idx.begin() + len, [&](size_t a, size_t b) { return before(row[a], a, row[b], b); });
        T score = 0;
        for (size_t k = 0; k < count && k < len; ++k)
            score += row[idx[k]];
        scores[i] = score;
        if (order)
            for (size_t k = 0; k < len; ++k)
                order[i * (n - 1) + k] = idx[k];
    }
}

// out[x] = sum_i w[i] * g[i][x] over the workers with non-zero weight, in index order.
template<class T> void weighted_sum(T const* g, size_t n, size_t d, T const* w, T* out) {
    std::vector<size_t> sel;
    for (size_t i = 0; i < n; ++i)
        if (w[i] != T(0))
            sel.push_back(i);
    agb::parallel_for(0, d, kGrainCoord, [&](size_t b, size_t e) {
        for (size_t x = b; x < e; ++x) {
            T sum = 0;
            for (size_t i: sel)
                sum += w[i] * g[i * d + x];
            out[x] = sum;
        }
    });
}

// out[x] = (sum_{i in sel} g[i][x]) / |sel|, in index order (Multi-Krum output).
template<class T> void selection_mean(T const* g, size_t d, std::vector<size_t> sel, T* out) {
    std::sort(sel.begin(), sel.end());
    T const count = static_cast<T>(sel.size());
    agb::parallel_for(0, d, kGrainCoord, [&](size_t b, size_t e) {
        for (size_t x = b; x < e; ++x) {
            T sum = 0;
            for (size_t i: sel)
                sum += g[i * d + x];
            out[x] = sum / count;
        }
    });
}

// ------------------------------------------------------------------------ //
template<class T> int average(T const* g, size_t n, size_t d, T* out) {
    if (n == 0 || n > kMaxWorkers)
        return 1;
    T const count = static_cast<T>(n);
    agb::parallel_for(0, d, kGrainCoord, [&](size_t b, size_t e) {
        for (size_t x = b; x < e; ++x) {
            T sum = 0;
            for (size_t i = 0; i < n; ++i)
                sum += g[i * d + x];
            out[x] = sum / count;
        }
    });
    return 0;
}

template<class T> int average_nan(T const* g, size_t n, size_t d, T* out) {
    if (n == 0 || n > kMaxWorkers)
        return 1;
    agb::parallel_for(0, d, kGrainCoord, [&](size_t b, size_t e) {
        for (size_t x = b; x < e; ++x) {
            T sum = 0;
            size_t count = 0;
            for (size_t i = 0; i < n; ++i) {
                T v = g[i * d + x];
                if (std::isfinite(v)) {
                    sum += v;
                    ++count;
                }
            }
            out[x] = sum / static_cast<T>(count); // 0/0 = NaN when no worker is finite (lets the NaN-loss guard fire)
        }
    });
    return 0;
}

// ------------------------------------------------------------------------ //
// Coordinate-wise selections. For up to kRankWorkers workers the order statistics come from rank counting on blocks of
// coordinates: rank_i = #{j : before(v_j, j, v_i, i)} with the keys made total (non-finite -> +inf, ties -> lower index), i.e. n^2
// branch-free compare-and-adds per coordinate over kBlock contiguous coordinates of every row — streaming loads and loops the
// compiler vectorises, instead of an index sort per coordinate with strided gathers. Larger n: std::nth_element on indices.
// (Same definition as the device kernels, `native/op_gar/gar.cu`; the reference does nth_element per coordinate, `native.cpp:678-748`.)
constexpr size_t kRankWorkers = 32;
constexpr size_t kBlock = 32;

template<class T> struct Block {
    T val[kRankWorkers][kBlock];     // original values
    T key[kRankWorkers][kBlock];     // non-finite -> +inf
    int rank[kRankWorkers][kBlock];
};

template<class T> inline void load_block(T const* g, size_t n, size_t d, size_t x0, size_t len, Block<T>& blk) {
    T const inf = std::numeric_limits<T>::infinity();
    for (size_t i = 0; i < n; ++i) {
        T const* row = g + i * d + x0;
        for (size_t c = 0; c < kBlock; ++c) {
            T const v = c < len ? row[c] : T(0);
            blk.val[i][c] = v;
            blk.key[i][c] = (v - v == T(0)) ? v : inf;   // v - v is NaN for NaN and +-inf
        }
    }
}

template<class T> inline void rank_block(size_t n, T const (*key)[kBlock], int (*rank)[kBlock]) {
    for (size_t i = 0; i < n; ++i) {
        int* const r = rank[i];
        for (size_t c = 0; c < kBlock; ++c)
            r[c] = 0;
        for (size_t j = 0; j < n; ++j) {
            T const* kj = key[j];
            T const* ki = key[i];
            if (j < i) {
                for (size_t c = 0; c < kBlock; ++c)
                    r[c] += kj[c] <= ki[c];       // equal keys: the lower index comes first
            } else if (j > i) {
                for (size_t c = 0; c < kBlock; ++c)
                    r[c] += kj[c] < ki[c];
            }
        }
    }
}

template<class T> inline void make_keys(size_t rows, Block<T>& blk) {
    T const inf = std::numeric_limits<T>::infinity();
    for (size_t i = 0; i < rows; ++i)
        for (size_t c = 0; c < kBlock; ++c) {
            T const v = blk.val[i][c];
            blk.key[i][c] = (v - v == T(0)) ? v : inf;
        }
}

// res[c] = mean of the `beta` values of column c of blk.val[0 .. rows) closest to their (upper) median, added in row order.
template<class T> inline void averaged_median_of_block(size_t rows, size_t beta, Block<T>& blk, T* res) {
    int const target = static_cast<int>(rows / 2), keep = static_cast<int>(beta);
    T const inf = std::numeric_limits<T>::infinity();
    rank_block<T>(rows, blk.key, blk.rank);
    T med[kBlock];
    for (size_t c = 0; c < kBlock; ++c)
        med[c] = T(0);
    for (size_t i = 0; i < rows; ++i)
        for (size_t c = 0; c < kBlock; ++c)
            med[c] = blk.rank[i][c] == target ? blk.val[i][c] : med[c];
    for (size_t i = 0; i < rows; ++i)           // second key: distance to the median (non-finite -> +inf)
        for (size_t c = 0; c < kBlock; ++c) {
            T const dev = std::fabs(blk.val[i][c] - med[c]);
            blk.key[i][c] = (dev - dev == T(0)) ? dev : inf;
        }
    rank_block<T>(rows, blk.key, blk.rank);
    for (size_t c = 0; c < kBlock; ++c)
        res[c] = T(0);
    for (size_t i = 0; i < rows; ++i)
        for (size_t c = 0; c < kBlock; ++c)
            res[c] += blk.rank[i][c] < keep ? blk.val[i][c] : T(0);
    for (size_t c = 0; c < kBlock; ++c)
        res[c] /= static_cast<T>(beta);
}

template<class T> int median(T const* g, size_t n, size_t d, T* out) {
    if (n == 0 || n > kMaxWorkers)
        return 1;
    if (n <= kRankWorkers) {
        agb::parallel_for(0, (d + kBlock - 1) / kBlock, kGrainCoord / kBlock, [&](size_t b, size_t e) {
            Block<T> blk;
            int const target = static_cast<int>(n / 2);   // upper median for even n
            for (size_t blk_i = b; blk_i < e; ++blk_i) {
                size_t const x0 = blk_i * kBlock, len = std::min(kBlock, d - x0);
                load_block(g, n, d, x0, len, blk);
                rank_block<T>(n, blk.key, blk.rank);
                T res[kBlock];
                for (size_t c = 0; c < kBlock; ++c)
                    res[c] = T(0);
                for (size_t i = 0; i < n; ++i)
                    for (size_t c = 0; c < kBlock; ++c)
                        res[c] = blk.rank[i][c] == target ? blk.val[i][c] : res[c];
                for (size_t c = 0; c < len; ++c)
                    out[x0 + c] = res[c];
            }
        });
        return 0;
    }
    agb::parallel_for(0, d, kGrainCoord, [&](size_t b, size_t e) {
        std::vector<size_t> idx(n);
        for (size_t x = b; x < e; ++x) {
            for (size_t i = 0; i < n; ++i)
                idx[i] = i;
            auto cmp = [&](size_t a, size_t c) { return before(g[a * d + x], a, g[c * d + x], c); };
            std::nth_element(idx.begin(), idx.begin() + n / 2, idx.end(), cmp);
            out[x] = g[idx[n / 2] * d + x]; // upper median for even n
        }
    });
    return 0;
}

// Mean of the `beta` values closest to the (upper) median, per coordinate.
template<class T> int averaged_median(T const* g, size_t n, size_t d, size_t beta, T* out) {
    if (n == 0 || n > kMaxWorkers || beta == 0 || beta > n)
        return 1;
    if (n <= kRankWorkers) {
        agb::parallel_for(0, (d + kBlock - 1) / kBlock, kGrainCoord / kBlock, [&](size_t b, size_t e) {
            Block<T> blk;
            T res[kBlock];
            for (size_t blk_i = b; blk_i < e; ++blk_i) {
                size_t const x0 = blk_i * kBlock, len = std::min(kBlock, d - x0);
                load_block(g, n, d, x0, len, blk);
                averaged_median_of_block<T>(n, beta, blk, res);
                for (size_t c = 0; c < len; ++c)
                    out[x0 + c] = res[c];
            }
        });
        return 0;
    }
    agb::parallel_for(0, d, kGrainCoord, [&](size_t b, size_t e) {
        std::vector<size_t> idx(n);
        std::vector<T> dev(n);
        std::vector<char> keep(n);
        for (size_t x = b; x < e; ++x) {
            for (size_t i = 0; i < n; ++i)
                idx[i] = i;
            auto cmp = [&](size_t a, size_t c) { return before(g[a * d + x], a, g[c * d + x], c); };
            std::nth_element(idx.begin(), idx.begin() + n / 2, idx.end(), cmp);
            T const zero = g[idx[n / 2] * d + x];
            for (size_t i = 0; i < n; ++i) {
                dev[i] = std::fabs(g[i * d + x] - zero);
                idx[i] = i;
            }
            auto closer = [&](size_t a, size_t c) { return before(dev[a], a, dev[c], c); };
            std::nth_element(idx.begin(), idx.begin() + (beta - 1), idx.end(), closer);
            std::fill(keep.begin(), keep.end(), 0);
            for (size_t k = 0; k < beta; ++k)
                keep[idx[k]] = 1;
            T sum = 0;
            for (size_t i = 0; i < n; ++i)
                if (keep[i])
                    sum += g[i * d + x];
            out[x] = sum / static_cast<T>(beta);
        }
    });
    return 0;
}

// Coordinate-wise trimmed mean: per coordinate, the values ranked [f, n - f) (the f smallest and the f largest or non-finite ones are
// dropped), added in index order, divided once by n - 2f. Same order of operations as the device kernel, hence the same bits.
template<class T> int trimmed_mean(T const* g, size_t n, size_t d, size_t f, T* out) {
    if (n == 0 || n > kMaxWorkers || 2 * f >= n)
        return 1;
    T const count = static_cast<T>(n - 2 * f);
    if (n <= kRankWorkers) {
        int const lo = static_cast<int>(f), hi = static_cast<int>(n - f);
        agb::parallel_for(0, (d + kBlock - 1) / kBlock, kGrainCoord / kBlock, [&](size_t b, size_t e) {
            Block<T> blk;
            T res[kBlock];
            for (size_t blk_i = b; blk_i < e; ++blk_i) {
                size_t const x0 = blk_i * kBlock, len = std::min(kBlock, d - x0);
                load_block(g, n, d, x0, len, blk);
                rank_block<T>(n, blk.key, blk.rank);
                for (size_t c = 0; c < kBlock; ++c)
                    res[c] = T(0);
                for (size_t i = 0; i < n; ++i)
                    for (size_t c = 0; c < kBlock; ++c)
                        res[c] += (blk.rank[i][c] >= lo && blk.rank[i][c] < hi) ? blk.val[i][c] : T(0);
                for (size_t c = 0; c < len; ++c)
                    out[x0 + c] = res[c] / count;
            }
        });
        return 0;
    }
    agb::parallel_for(0, d, kGrainCoord, [&](size_t b, size_t e) {
        std::vector<size_t> idx(n);
        std::vector<char> keep(n);
        for (size_t x = b; x < e; ++x) {
            for (size_t i = 0; i < n; ++i)
                idx[i] = i;
            auto cmp = [&](size_t a, size_t c) { return before(g[a * d + x], a, g[c * d + x], c); };
            std::nth_element(idx.begin(), idx.begin() + f, idx.end(), cmp);                 // ranks [0, f) first
            std::nth_element(idx.begin() + f, idx.begin() + (n - f), idx.end(), cmp);       // then [f, n - f)
            std::fill(keep.begin(), keep.end(), 0);
            for (size_t k = f; k < n - f; ++k)
                keep[idx[k]] = 1;
            T sum = 0;
            for (size_t i = 0; i < n; ++i)
                if (keep[i])
                    sum += g[i * d + x];
            out[x] = sum / count;
        }
    });
    return 0;
}

// ------------------------------------------------------------------------ //
// MDA (minimum-diameter averaging): the kept set S, |S| = n - f, whose diameter (largest pairwise distance inside S, non-finite
// distances = +inf) is smallest; ties -> the lexicographically smallest sorted index list of S. The removal sets R, |R| = f, are
// enumerated in lexicographic order: a later R is lexicographically larger, so its S is smaller and wins a tie. A set's diameter is
// the first pair, in descending distance order, with both ends kept.
constexpr size_t kMdaMaxSets = size_t(1) << 20;

inline bool mda_params_ok(size_t n, size_t f) {
    if (n == 0 || n > kMaxWorkers || 2 * f >= n)
        return false;
    size_t sets = 1;   // C(n, f), exact while it stays below the bound
    for (size_t t = 0; t < f && sets <= kMdaMaxSets; ++t)
        sets = sets * (n - t) / (t + 1);
    return sets <= kMdaMaxSets;
}

template<class T> int mda_select(T const* dist, size_t n, size_t f, int64_t* selected) {
    if (!mda_params_ok(n, f))
        return 1;
    T const inf = std::numeric_limits<T>::infinity();
    std::vector<std::pair<size_t, size_t>> pairs;
    std::vector<T> value;
    for (size_t i = 0; i + 1 < n; ++i)
        for (size_t j = i + 1; j < n; ++j) {
            T const v = dist[i * n + j];
            pairs.emplace_back(i, j);
            value.push_back(std::isfinite(v) ? v : inf);
        }
    std::vector<size_t> order(pairs.size());
    for (size_t p = 0; p < order.size(); ++p)
        order[p] = p;
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return value[a] > value[b]; });
    std::vector<size_t> removal(f), best_removal(f);
    for (size_t k = 0; k < f; ++k)
        removal[k] = k;
    std::vector<char> removed(n, 0);
    T best = inf;
    bool found = false;
    for (;;) {
        for (size_t k = 0; k < f; ++k)
            removed[removal[k]] = 1;
        T diam = 0;
        for (size_t p: order)
            if (!removed[pairs[p].first] && !removed[pairs[p].second]) {
                diam = value[p];
                break;
            }
        if (!found || diam <= best) {
            best = diam;
            best_removal = removal;
            found = true;
        }
        for (size_t k = 0; k < f; ++k)
            removed[removal[k]] = 0;
        size_t k = f;   // next removal set in lexicographic order
        while (k > 0 && removal[k - 1] == n - f + k - 1)
            --k;
        if (k == 0)
            break;
        ++removal[k - 1];
        for (size_t t = k; t < f; ++t)
            removal[t] = removal[t - 1] + 1;
    }
    for (size_t k = 0; k < f; ++k)
        removed[best_removal[k]] = 1;
    size_t count = 0;
    for (size_t i = 0; i < n; ++i)
        if (!removed[i])
            selected[count++] = static_cast<int64_t>(i);
    return 0;
}

// MDA: mean of the selected rows, added in index order, divided once by n - f; `selected` (optional, [n - f]) receives their ids.
template<class T> int mda(T const* g, size_t n, size_t d, size_t f, T* out, int64_t* selected, T* dist_out) {
    if (!mda_params_ok(n, f))
        return 1;
    std::vector<T> dist(n * n);
    std::vector<int64_t> ids(n - f);
    pairwise_distances(g, n, d, dist.data());
    if (dist_out)
        std::copy(dist.begin(), dist.end(), dist_out);
    if (int status = mda_select(dist.data(), n, f, ids.data()))
        return status;
    if (selected)
        std::copy(ids.begin(), ids.end(), selected);
    selection_mean(g, d, std::vector<size_t>(ids.begin(), ids.end()), out);
    return 0;
}

// ------------------------------------------------------------------------ //
// Geometric median, smoothed Weiszfeld iterations (RFA, Pillutla et al.): z_0 = the coordinate-wise median; for t < T,
// D_i = ||z_t - x_i||^2 (chunked, folded in chunk order), rows with a non-finite D_i are skipped, beta_i = 1 / max(nu, sqrt(D_i)),
// z_{t+1} = (sum beta_i x_i) / (sum beta_i), both sums over the kept rows in index order from +0, one rounding per operation (the
// device kernel's definition: given the distances, the same bits). No kept row: z_{t+1} = z_t. `dist` (optional, [T, n]) receives D.
constexpr size_t kGeoMaxIterations = 16;

template<class T> int geometric_median(T const* g, size_t n, size_t d, size_t iterations, double nu_arg, T* out, T* dist_out) {
    T const nu = static_cast<T>(nu_arg);
    if (n == 0 || n > kMaxWorkers || iterations < 1 || iterations > kGeoMaxIterations || !(nu > T(0)) || !std::isfinite(nu))
        return 1;
    if (int status = median<T>(g, n, d, out))
        return status;
    size_t const chunks = ThreadPool::chunk_count(0, d, kGrainCoord);
    std::vector<T> next(d), partial(chunks * n), beta(n);
    T* z = out;
    T* z_next = next.data();
    for (size_t t = 0; t < iterations; ++t) {
        global_pool().run(0, d, kGrainCoord, [&](size_t chunk, size_t b, size_t e) {
            for (size_t i = 0; i < n; ++i)
                partial[chunk * n + i] = squared_difference(z, g + i * d, b, e);
        });
        std::vector<size_t> kept;
        T sum = 0;
        for (size_t i = 0; i < n; ++i) {
            T D = 0;
            for (size_t c = 0; c < chunks; ++c)
                D += partial[c * n + i];
            if (dist_out)
                dist_out[t * n + i] = D;
            if (std::isfinite(D)) {   // skipped, not weighted by 0: 0 * NaN is NaN
                beta[i] = T(1) / std::max(nu, std::sqrt(D));
                sum += beta[i];
                kept.push_back(i);
            }
        }
        if (kept.empty())
            continue;   // z_{t+1} = z_t: the next iteration sees the same distances
        agb::parallel_for(0, d, kGrainCoord, [&](size_t b, size_t e) {
            for (size_t x = b; x < e; ++x) {
                T num = 0;
                for (size_t i: kept)
                    num += beta[i] * g[i * d + x];
                z_next[x] = num / sum;
            }
        });
        std::swap(z, z_next);
    }
    if (z != out)
        std::copy(z, z + d, out);
    return 0;
}

// ------------------------------------------------------------------------ //
// Centered clipping (Karimireddy, He and Jaggi, "Learning from History for Byzantine Robust Optimization"): z_0 = the center v; for
// t < T, D_i = ||x_i - z_t||^2 (chunked, folded in chunk order), rows with a non-finite D_i are skipped, s_i = sqrt(D_i),
// c_i = 1 if s_i <= tau else tau / s_i, z_{t+1} = z_t + (sum c_i (x_i - z_t)) / n, the sum over the kept rows in index order from +0
// and divided by all n rows, one rounding per operation (the device kernel's definition: given the distances, the same bits). No
// kept row: z_{t+1} = z_t. `center` is v on entry and z_T on return; `dist` (optional, [T, n]) receives D.
template<class T> int centered_clipping(T const* g, size_t n, size_t d, size_t iterations, double tau_arg, T* center, T* dist_out) {
    T const tau = static_cast<T>(tau_arg);
    if (n == 0 || n > kMaxWorkers || iterations < 1 || iterations > kGeoMaxIterations || !(tau > T(0)) || !std::isfinite(tau) || !center)
        return 1;
    size_t const chunks = ThreadPool::chunk_count(0, d, kGrainCoord);
    std::vector<T> partial(chunks * n), clip(n);
    T const count = static_cast<T>(n);
    for (size_t t = 0; t < iterations; ++t) {
        global_pool().run(0, d, kGrainCoord, [&](size_t chunk, size_t b, size_t e) {
            for (size_t i = 0; i < n; ++i)
                partial[chunk * n + i] = squared_difference(center, g + i * d, b, e);
        });
        std::vector<size_t> kept;
        for (size_t i = 0; i < n; ++i) {
            T D = 0;
            for (size_t c = 0; c < chunks; ++c)
                D += partial[c * n + i];
            if (dist_out)
                dist_out[t * n + i] = D;
            if (std::isfinite(D)) {   // skipped, not weighted by 0: 0 * NaN is NaN
                T const s = std::sqrt(D);
                clip[i] = s <= tau ? T(1) : tau / s;
                kept.push_back(i);
            }
        }
        if (kept.empty())
            continue;   // z_{t+1} = z_t
        agb::parallel_for(0, d, kGrainCoord, [&](size_t b, size_t e) {
            for (size_t x = b; x < e; ++x) {
                T u = 0;
                for (size_t i: kept) {
                    T const diff = g[i * d + x] - center[x];
                    u += clip[i] * diff;
                }
                center[x] = center[x] + u / count;
            }
        });
    }
    return 0;
}

// Multi-Krum: average of the m smallest-scoring gradients; `selected` (optional, [m]) receives their ids.
template<class T> int krum(T const* g, size_t n, size_t d, size_t f, size_t m, T* out, int64_t* selected, T* dist_out) {
    if (n == 0 || n > kMaxWorkers || n < f + 3 || m < 1 || m > n)
        return 1;
    std::vector<T> dist(n * n), scores(n);
    pairwise_distances(g, n, d, dist.data());
    if (dist_out)
        std::copy(dist.begin(), dist.end(), dist_out);
    krum_scores(dist.data(), n, n - f - 2, scores.data(), nullptr);
    std::vector<size_t> idx(n);
    for (size_t i = 0; i < n; ++i)
        idx[i] = i;
    std::sort(idx.begin(), idx.end(), [&](size_t a, size_t b) { return before(scores[a], a, scores[b], b); });
    idx.resize(m);
    if (selected)
        for (size_t k = 0; k < m; ++k)
            selected[k] = static_cast<int64_t>(idx[k]);
    selection_mean(g, d, idx, out);
    return 0;
}

// Bulyan's selection stage: fills the [theta, n] weight matrix W such that intermediate k = sum_i W[k][i] g_i.
template<class T> int bulyan_weights(T const* dist, size_t n, size_t f, size_t m, T* weights) {
    if (n < 4 * f + 3 || m < 1 || m > n)
        return 1;
    size_t const theta = n - 2 * f - 2;
    if (m < theta) // round k averages m - k >= 1 gradients
        return 1;
    std::vector<T> scores(n), pruned(dist, dist + n * n);
    std::vector<size_t> order(n * (n - 1));
    size_t const inscore = n - f - 2;
    krum_scores(dist, n, inscore, scores.data(), order.data());
    for (size_t i = 0; i < n; ++i) // distances not counted in the score of i never get subtracted from it
        for (size_t k = inscore; k < n - 1; ++k)
            pruned[i * n + order[i * (n - 1) + k]] = 0;
    std::vector<char> removed(n, 0);
    std::vector<size_t> idx(n);
    for (size_t k = 0; k < theta; ++k) {
        for (size_t i = 0; i < n; ++i)
            idx[i] = i;
        std::sort(idx.begin(), idx.end(), [&](size_t a, size_t b) {
            if (removed[a] != removed[b])
                return !removed[a];
            return before(scores[a], a, scores[b], b);
        });
        size_t const count = m - k;
        for (size_t i = 0; i < n; ++i)
            weights[k * n + i] = 0;
        for (size_t r = 0; r < count; ++r)
            weights[k * n + idx[r]] = T(1) / static_cast<T>(count);
        size_t const best = idx[0];
        removed[best] = 1;
        for (size_t i = 0; i < n; ++i)
            if (!removed[i])
                scores[i] -= pruned[i * n + best];
    }
    return 0;
}

template<class T> int bulyan(T const* g, size_t n, size_t d, size_t f, size_t m, T* out, T* weights_out) {
    if (n == 0 || n > kMaxWorkers || n < 4 * f + 3)
        return 1;
    size_t const theta = n - 2 * f - 2;
    size_t const beta = theta - 2 * f;
    std::vector<T> dist(n * n), weights(theta * n);
    pairwise_distances(g, n, d, dist.data());
    if (int status = bulyan_weights(dist.data(), n, f, m, weights.data()))
        return status;
    if (weights_out)
        std::copy(weights.begin(), weights.end(), weights_out);
    // Sparse view of the weight rows (index order), then the coordinate-wise averaged median of the theta intermediates.
    std::vector<std::vector<size_t>> members(theta);
    for (size_t k = 0; k < theta; ++k)
        for (size_t i = 0; i < n; ++i)
            if (weights[k * n + i] != T(0))
                members[k].push_back(i);
    if (theta <= kRankWorkers) {
        agb::parallel_for(0, (d + kBlock - 1) / kBlock, kGrainCoord / 4 / kBlock, [&](size_t b, size_t e) {
            Block<T> blk;
            T res[kBlock];
            for (size_t blk_i = b; blk_i < e; ++blk_i) {
                size_t const x0 = blk_i * kBlock, len = std::min(kBlock, d - x0);
                for (size_t k = 0; k < theta; ++k) {     // the theta intermediate gradients of this block (members added in index order)
                    T* const row = blk.val[k];
                    for (size_t c = 0; c < kBlock; ++c)
                        row[c] = T(0);
                    for (size_t i: members[k]) {
                        T const* src = g + i * d + x0;
                        for (size_t c = 0; c < len; ++c)
                            row[c] += src[c];
                    }
                    T const count = static_cast<T>(members[k].size());
                    for (size_t c = 0; c < kBlock; ++c)
                        row[c] /= count;
                }
                make_keys<T>(theta, blk);
                averaged_median_of_block<T>(theta, beta, blk, res);
                for (size_t c = 0; c < len; ++c)
                    out[x0 + c] = res[c];
            }
        });
        return 0;
    }
    agb::parallel_for(0, d, kGrainCoord / 4, [&](size_t b, size_t e) {
        std::vector<T> inter(theta), dev(theta);
        std::vector<size_t> idx(theta);
        std::vector<char> keep(theta);
        for (size_t x = b; x < e; ++x) {
            for (size_t k = 0; k < theta; ++k) {
                T sum = 0;
                for (size_t i: members[k])
                    sum += g[i * d + x];
                inter[k] = sum / static_cast<T>(members[k].size());
                idx[k] = k;
            }
            auto cmp = [&](size_t a, size_t c) { return before(inter[a], a, inter[c], c); };
            std::nth_element(idx.begin(), idx.begin() + theta / 2, idx.end(), cmp);
            T const zero = inter[idx[theta / 2]];
            for (size_t k = 0; k < theta; ++k) {
                dev[k] = std::fabs(inter[k] - zero);
                idx[k] = k;
            }
            auto closer = [&](size_t a, size_t c) { return before(dev[a], a, dev[c], c); };
            std::nth_element(idx.begin(), idx.begin() + (beta - 1), idx.end(), closer);
            std::fill(keep.begin(), keep.end(), 0);
            for (size_t k = 0; k < beta; ++k)
                keep[idx[k]] = 1;
            T sum = 0;
            for (size_t k = 0; k < theta; ++k)
                if (keep[k])
                    sum += inter[k];
            out[x] = sum / static_cast<T>(beta);
        }
    });
    return 0;
}

// ------------------------------------------------------------------------ //
// DnC's sampled distances (`native/op_gar/gar.cu` defines the sampler): for t < T, D^t_ij = sum_k (x_i[s_k] - x_j[s_k])^2 over the
// b' = min(b, domain) coordinates s_k = P(k) of iteration t, added in ascending k; non-finite -> +inf. The selection runs in Python
// (`_ops.dnc_select`), so that its float64 Jacobi exists once on the host.
inline uint64_t splitmix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

template<class T> int dnc_sample_distances(T const* g, size_t n, size_t d, size_t iterations, size_t b, uint64_t seed, uint64_t step,
                                           size_t domain, T* dist /* [T, n, n] */) {
    if (n < 1 || iterations < 1 || iterations > 8 || b < 1 || b > (size_t(1) << 20) || domain < 1 || domain > d || domain > (size_t(1) << 48))
        return 1;
    size_t const count = std::min(b, domain);
    int width = 0;
    while (width < 64 && ((domain - 1) >> width) != 0)
        ++width;
    int const h = (width < 2 ? 2 : width + (width & 1)) / 2;
    uint64_t const mask = (uint64_t(1) << h) - 1;
    std::vector<T> sample(n * count);
    for (size_t t = 0; t < iterations; ++t) {
        uint64_t const key = splitmix64(splitmix64(splitmix64(seed) ^ step) ^ t);
        for (size_t k = 0; k < count; ++k) {
            uint64_t y = k;
            do {
                uint64_t L = y >> h, R = y & mask;
                for (uint64_t r = 0; r < 4; ++r) {
                    uint64_t const next = L ^ (splitmix64(key ^ (r << 48) ^ R) & mask);
                    L = R;
                    R = next;
                }
                y = (L << h) | R;
            } while (y >= domain);
            for (size_t i = 0; i < n; ++i)
                sample[i * count + k] = g[i * d + y];
        }
        T* out = dist + t * n * n;
        for (size_t i = 0; i < n; ++i) {
            out[i * n + i] = T(0);
            for (size_t j = i + 1; j < n; ++j) {
                T sum = T(0);
                for (size_t k = 0; k < count; ++k) {
                    T const delta = sample[i * count + k] - sample[j * count + k];
                    sum += delta * delta;
                }
                if (!std::isfinite(sum))
                    sum = std::numeric_limits<T>::infinity();
                out[i * n + j] = sum;
                out[j * n + i] = sum;
            }
        }
    }
    return 0;
}

template<class T> int selection_mean_of(T const* g, size_t n, size_t d, int64_t const* selected, size_t count, T* out) {
    if (count < 1)
        return 1;
    std::vector<size_t> sel(count);
    for (size_t k = 0; k < count; ++k) {
        if (selected[k] < 0 || static_cast<size_t>(selected[k]) >= n)
            return 1;
        sel[k] = static_cast<size_t>(selected[k]);
    }
    selection_mean<T>(g, d, sel, out);
    return 0;
}

// sum_{k in [b, e)} x[k] * y[k], with `squared_difference`'s 16 interleaved partial sums and fixed fold
template<class T> inline T dot(T const* x, T const* y, size_t b, size_t e) {
    constexpr size_t kLanes = 16;
    T acc[kLanes];
    for (size_t u = 0; u < kLanes; ++u)
        acc[u] = T(0);
    size_t k = b;
    for (; k + kLanes <= e; k += kLanes)
        for (size_t u = 0; u < kLanes; ++u)
            acc[u] += x[k + u] * y[k + u];
    for (size_t u = 0; k < e; ++k, ++u)
        acc[u] += x[k] * y[k];
    for (size_t width = kLanes / 2; width > 0; width /= 2)
        for (size_t u = 0; u < width; ++u)
            acc[u] += acc[u + width];
    return acc[0];
}

// FLTrust's sums (`aggregators/_ops.py`): out = [P_0 .. P_{n-1}, N_0 .. N_{n-1}, N0] with P_i = <x_i, r>, N_i = ||x_i||^2, N0 = ||r||^2,
// per-chunk partials folded in chunk order. The coefficients and the weighted sum are computed by the callers (one copy of that arithmetic).
template<class T> int fltrust_sums(T const* g, size_t n, size_t d, T const* root, T* out) {
    if (n == 0 || n > kMaxWorkers)
        return 1;
    size_t const chunks = ThreadPool::chunk_count(0, d, kGrainCoord);
    size_t const width = 2 * n + 1;
    std::vector<T> partial(chunks * width, T(0));
    global_pool().run(0, d, kGrainCoord, [&](size_t chunk, size_t b, size_t e) {
        T* part = partial.data() + chunk * width;
        for (size_t i = 0; i < n; ++i) {
            part[i] = dot(g + i * d, root, b, e);
            part[n + i] = dot(g + i * d, g + i * d, b, e);
        }
        part[2 * n] = dot(root, root, b, e);
    });
    for (size_t k = 0; k < width; ++k) {
        T sum = 0;
        for (size_t c = 0; c < chunks; ++c)
            sum += partial[c * width + k];
        out[k] = sum;
    }
    return 0;
}

// FoolsGold's history step and sums (`aggregators/_ops.py`), one pass over the coordinates: every chunk first adds the finite values of
// the rows g_i to the histories H_i (in place), then accumulates the partial products <H_i, H_j>, i <= j, of its updated coordinates.
// out = [P (n x n, computed for i <= j and mirrored), the n bad flags (1: g_i holds a non-finite value)], the per-chunk partials folded
// in chunk order. The coefficients and the weighted sum are computed by the callers.
template<class T> int foolsgold_sums(T const* g, size_t n, size_t d, T* H, T* out) {
    if (n == 0 || n > kMaxWorkers)
        return 1;
    size_t const chunks = ThreadPool::chunk_count(0, d, kGrainCoord);
    size_t const pairs = n * (n + 1) / 2, width = pairs + n;
    std::vector<T> partial(chunks * width, T(0));
    global_pool().run(0, d, kGrainCoord, [&](size_t chunk, size_t b, size_t e) {
        T* part = partial.data() + chunk * width;
        for (size_t i = 0; i < n; ++i) {
            T const* gi = g + i * d;
            T* hi = H + i * d;
            bool bad = false;
            for (size_t k = b; k < e; ++k) {
                if (std::isfinite(gi[k]))
                    hi[k] += gi[k];
                else
                    bad = true;
            }
            part[pairs + i] = bad ? T(1) : T(0);
        }
        for (size_t i = 0, p = 0; i < n; ++i)
            for (size_t j = i; j < n; ++j, ++p)
                part[p] = dot(H + i * d, H + j * d, b, e);
    });
    for (size_t i = 0, p = 0; i < n; ++i)
        for (size_t j = i; j < n; ++j, ++p) {
            T sum = 0;
            for (size_t c = 0; c < chunks; ++c)
                sum += partial[c * width + p];
            out[i * n + j] = sum;
            out[j * n + i] = sum;
        }
    for (size_t i = 0; i < n; ++i) {
        T flag = 0;
        for (size_t c = 0; c < chunks; ++c)
            flag = partial[c * width + pairs + i] != T(0) ? T(1) : flag;
        out[n * n + i] = flag;
    }
    return 0;
}

template<class T> T squared_distance(T const* a, T const* b, size_t d) {
    size_t const chunks = ThreadPool::chunk_count(0, d, kGrainCoord);
    std::vector<T> partial(chunks, T(0));
    global_pool().run(0, d, kGrainCoord, [&](size_t chunk, size_t lo, size_t hi) { partial[chunk] = squared_difference(a, b, lo, hi); });
    T sum = 0;
    for (T v: partial)
        sum += v;
    return sum;
}

} // namespace

// CRC32C (Castagnoli), table driven, 8 bytes per step: checksums of TensorFlow-format files (checkpoint tensors, TFRecords).
extern "C" uint32_t agb_crc32c(uint8_t const* data, size_t size, uint32_t crc) {
    static uint32_t table[8][256];
    static bool ready = false;
    if (!ready) {
        for (uint32_t i = 0; i < 256; ++i) {
            uint32_t c = i;
            for (int k = 0; k < 8; ++k)
                c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
            table[0][i] = c;
        }
        for (uint32_t i = 0; i < 256; ++i)
            for (int t = 1; t < 8; ++t)
                table[t][i] = (table[t - 1][i] >> 8) ^ table[0][table[t - 1][i] & 0xFF];
        ready = true;
    }
    crc = ~crc;
    size_t i = 0;
    for (; i + 8 <= size; i += 8) {
        uint32_t const lo = crc ^ (static_cast<uint32_t>(data[i]) | static_cast<uint32_t>(data[i + 1]) << 8 | static_cast<uint32_t>(data[i + 2]) << 16 | static_cast<uint32_t>(data[i + 3]) << 24);
        crc = table[7][lo & 0xFF] ^ table[6][(lo >> 8) & 0xFF] ^ table[5][(lo >> 16) & 0xFF] ^ table[4][lo >> 24]
            ^ table[3][data[i + 4]] ^ table[2][data[i + 5]] ^ table[1][data[i + 6]] ^ table[0][data[i + 7]];
    }
    for (; i < size; ++i)
        crc = table[0][(crc ^ data[i]) & 0xFF] ^ (crc >> 8);
    return ~crc;
}

#define AGB_EXPORT(T, S) \
    extern "C" int agb_cpu_average_##S(T const* g, size_t n, size_t d, T* out) { return average<T>(g, n, d, out); } \
    extern "C" int agb_cpu_average_nan_##S(T const* g, size_t n, size_t d, T* out) { return average_nan<T>(g, n, d, out); } \
    extern "C" int agb_cpu_median_##S(T const* g, size_t n, size_t d, T* out) { return median<T>(g, n, d, out); } \
    extern "C" int agb_cpu_averaged_median_##S(T const* g, size_t n, size_t d, size_t beta, T* out) { return averaged_median<T>(g, n, d, beta, out); } \
    extern "C" int agb_cpu_krum_##S(T const* g, size_t n, size_t d, size_t f, size_t m, T* out, int64_t* selected, T* dist) { return krum<T>(g, n, d, f, m, out, selected, dist); } \
    extern "C" int agb_cpu_bulyan_##S(T const* g, size_t n, size_t d, size_t f, size_t m, T* out, T* weights) { return bulyan<T>(g, n, d, f, m, out, weights); } \
    extern "C" int agb_cpu_bulyan_weights_##S(T const* dist, size_t n, size_t f, size_t m, T* weights) { return bulyan_weights<T>(dist, n, f, m, weights); } \
    extern "C" int agb_cpu_trimmed_mean_##S(T const* g, size_t n, size_t d, size_t f, T* out) { return trimmed_mean<T>(g, n, d, f, out); } \
    extern "C" int agb_cpu_mda_##S(T const* g, size_t n, size_t d, size_t f, T* out, int64_t* selected, T* dist) { return mda<T>(g, n, d, f, out, selected, dist); } \
    extern "C" int agb_cpu_mda_select_##S(T const* dist, size_t n, size_t f, int64_t* selected) { return mda_select<T>(dist, n, f, selected); } \
    extern "C" int agb_cpu_geometric_median_##S(T const* g, size_t n, size_t d, size_t iterations, double nu, T* out, T* dist) { return geometric_median<T>(g, n, d, iterations, nu, out, dist); } \
    extern "C" int agb_cpu_centered_clipping_##S(T const* g, size_t n, size_t d, size_t iterations, double tau, T* center, T* dist) { return centered_clipping<T>(g, n, d, iterations, tau, center, dist); } \
    extern "C" int agb_cpu_pairwise_distances_##S(T const* g, size_t n, size_t d, T* dist) { if (n < 1) return 1; pairwise_distances<T>(g, n, d, dist); return 0; } \
    extern "C" int agb_cpu_weighted_sum_##S(T const* g, size_t n, size_t d, T const* w, T* out) { weighted_sum<T>(g, n, d, w, out); return 0; } \
    extern "C" int agb_cpu_dnc_sample_distances_##S(T const* g, size_t n, size_t d, size_t iterations, size_t b, uint64_t seed, uint64_t step, size_t domain, T* dist) { return dnc_sample_distances<T>(g, n, d, iterations, b, seed, step, domain, dist); } \
    extern "C" int agb_cpu_selection_mean_##S(T const* g, size_t n, size_t d, int64_t const* selected, size_t count, T* out) { return selection_mean_of<T>(g, n, d, selected, count, out); } \
    extern "C" int agb_cpu_fltrust_sums_##S(T const* g, size_t n, size_t d, T const* root, T* out) { return fltrust_sums<T>(g, n, d, root, out); } \
    extern "C" int agb_cpu_foolsgold_sums_##S(T const* g, size_t n, size_t d, T* history, T* out) { return foolsgold_sums<T>(g, n, d, history, out); } \
    extern "C" T agb_cpu_squared_distance_##S(T const* a, T const* b, size_t d) { return squared_distance<T>(a, b, d); }

AGB_EXPORT(float, float)
AGB_EXPORT(double, double)

extern "C" size_t agb_cpu_pool_size() { return agb::global_pool().size(); }
