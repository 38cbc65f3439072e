// Streaming shard reader: N reader threads -> shuffle pool -> caller-provided (pinned) batch buffers.
//
// GPU-side equivalent of the input pipeline the reference borrows from TensorFlow / slim
// (`experiments/slims.py:100-111`, `experiments/cnnet.py:123-132`: `DatasetDataProvider(num_readers=...)` over the TFRecord shards,
// a `RandomShuffleQueue`, `tf.train.batch(num_threads=...)`, `prefetch_queue`). A dataset is a list of shard files of fixed-size
// records (`tools/datasets.py --shards`): 64-byte header, then `count` records of `record_bytes` image bytes (uint8 HWC at the
// storage resolution), then `count` int64 labels. Nothing is ever loaded whole: readers `pread` records in a per-epoch random
// order (shard order shuffled per epoch, records shuffled inside the shard), push them into a bounded pool, and `next()` fills
// one batch by drawing uniformly from the pool once it holds `min_after_dequeue` records (the RandomShuffleQueue discipline),
// copying each record straight into the caller's buffer — pinned host memory from which the H2D copy is issued.
//
// A reader opened with `agb_loader_open_subset` serves only the records of a membership bitmap over the global record index (the
// shards in the order given, then the records of each shard), e.g. one worker's part of a label-skewed split; the others are skipped
// before any read.
//
// C ABI (ctypes): agb_loader_open / agb_loader_open_subset / agb_loader_next / agb_loader_info / agb_loader_close.

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <vector>

namespace {

constexpr char kMagic[8] = {'A', 'G', 'B', 'S', 'H', 'R', 'D', '1'};

struct ShardHeader {          // 64 bytes, little endian
    char magic[8];
    uint64_t count;           // records in this shard
    uint32_t height, width, channels;
    uint32_t label_bytes;     // 8 (int64)
    uint64_t record_bytes;    // height * width * channels
    uint8_t reserved[24];
};
static_assert(sizeof(ShardHeader) == 64, "shard header is 64 bytes");

struct Shard {
    std::string path;
    int fd = -1;
    uint64_t count = 0;
    uint64_t first = 0;       // global index of its record 0 (records of the shards before it)
};

struct Record {
    std::vector<uint8_t> pixels;
    int64_t label = 0;
};

class Loader {
public:
    Loader(std::vector<Shard> shards, ShardHeader const& proto, int batch, int nthreads, uint64_t seed, bool shuffle, size_t pool_capacity, size_t min_after_dequeue, int part, int parts,
           std::vector<uint64_t> members = {})
        : shards_(std::move(shards)), proto_(proto), batch_(batch), shuffle_(shuffle), capacity_(pool_capacity), min_after_(min_after_dequeue), part_(part), parts_(parts),
          members_(std::move(members)), draw_rng_(seed ^ 0x9E3779B97F4A7C15ull) {
        if (!shuffle_)
            nthreads = 1;   // sequential order is only defined with one reader
        total_ = 0;   // records this reader can ever serve per epoch (its residue class of every shard, or its subset)
        if (!members_.empty()) {
            for (uint64_t word : members_)
                total_ += static_cast<uint64_t>(__builtin_popcountll(word));
        } else {
            for (auto const& s : shards_)
                total_ += parts_ > 1 ? (s.count + parts_ - 1 - part_) / parts_ : s.count;
        }
        for (int t = 0; t < nthreads; ++t)
            readers_.emplace_back([this, t, nthreads, seed] { read_loop(t, nthreads, seed); });
    }

    ~Loader() {
        {
            std::lock_guard<std::mutex> guard(mutex_);
            stop_ = true;
        }
        not_full_.notify_all();
        not_empty_.notify_all();
        for (auto& thread : readers_)
            thread.join();
        for (auto& s : shards_)
            if (s.fd >= 0)
                ::close(s.fd);
    }

    // Fill `batch_` records; returns 0, or -1 when a reader failed (message in `error()`).
    int next(uint8_t* images, int64_t* labels) {
        for (int b = 0; b < batch_; ++b) {
            Record record;
            {
                std::unique_lock<std::mutex> lock(mutex_);
                size_t const need = shuffle_ ? std::min(min_after_, total_ ? static_cast<size_t>(total_) - 1 : size_t(0)) + 1 : 1;
                not_empty_.wait(lock, [&] { return stop_ || failed_ || pool_.size() >= need; });
                if (failed_ || stop_)
                    return -1;
                size_t pick = 0;
                if (shuffle_)
                    pick = std::uniform_int_distribution<size_t>(0, pool_.size() - 1)(draw_rng_);
                record = std::move(pool_[pick]);
                if (shuffle_) {
                    if (pick + 1 != pool_.size())
                        pool_[pick] = std::move(pool_.back());
                    pool_.pop_back();
                } else {
                    pool_.erase(pool_.begin());
                }
                ++served_;
            }
            not_full_.notify_one();
            std::memcpy(images + static_cast<size_t>(b) * proto_.record_bytes, record.pixels.data(), proto_.record_bytes);
            labels[b] = record.label;
        }
        return 0;
    }

    std::string error() {
        std::lock_guard<std::mutex> guard(mutex_);
        return error_;
    }
    uint64_t total() const { return total_; }
    uint64_t served() const { return served_; }
    ShardHeader const& proto() const { return proto_; }

private:
    void fail(std::string const& what) {
        {
            std::lock_guard<std::mutex> guard(mutex_);
            failed_ = true;
            error_ = what;
        }
        not_empty_.notify_all();
    }

    // Reader t handles the shards at positions t, t + nthreads, ... of every epoch's shard permutation (all readers derive the
    // same permutation from (seed, epoch)); `part`/`parts` restrict a worker to every parts-th record (disjoint data per worker).
    void read_loop(int t, int nthreads, uint64_t seed) {
        std::vector<uint32_t> order;
        for (uint64_t epoch = 0;; ++epoch) {
            std::vector<size_t> perm(shards_.size());
            for (size_t i = 0; i < perm.size(); ++i)
                perm[i] = i;
            if (shuffle_) {
                std::mt19937_64 rng(seed * 0x100000001B3ull + epoch);
                std::shuffle(perm.begin(), perm.end(), rng);
            }
            for (size_t pos = t; pos < perm.size(); pos += nthreads) {
                Shard const& shard = shards_[perm[pos]];
                order.resize(shard.count);
                for (uint32_t i = 0; i < shard.count; ++i)
                    order[i] = i;
                if (shuffle_) {
                    std::mt19937_64 rng((seed + 0x51ED27ull * (perm[pos] + 1)) ^ (epoch << 20));
                    std::shuffle(order.begin(), order.end(), rng);
                }
                off_t const labels_at = static_cast<off_t>(sizeof(ShardHeader) + shard.count * proto_.record_bytes);
                for (uint32_t index : order) {
                    if (parts_ > 1 && static_cast<int>(index % parts_) != part_)
                        continue;
                    uint64_t const global = shard.first + index;
                    if (!members_.empty() && !((members_[global >> 6] >> (global & 63)) & 1ull))
                        continue;
                    Record record;
                    record.pixels.resize(proto_.record_bytes);
                    off_t const at = static_cast<off_t>(sizeof(ShardHeader) + static_cast<uint64_t>(index) * proto_.record_bytes);
                    if (!read_all(shard.fd, record.pixels.data(), proto_.record_bytes, at) || !read_all(shard.fd, &record.label, 8, labels_at + static_cast<off_t>(index) * 8)) {
                        fail("short read in shard " + shard.path);
                        return;
                    }
                    std::unique_lock<std::mutex> lock(mutex_);
                    not_full_.wait(lock, [&] { return stop_ || pool_.size() < capacity_; });
                    if (stop_)
                        return;
                    pool_.push_back(std::move(record));
                    lock.unlock();
                    not_empty_.notify_one();
                }
            }
            {
                std::lock_guard<std::mutex> guard(mutex_);
                if (stop_)
                    return;
            }
        }
    }

    static bool read_all(int fd, void* dst, size_t bytes, off_t at) {
        uint8_t* out = static_cast<uint8_t*>(dst);
        while (bytes > 0) {
            ssize_t got = ::pread(fd, out, bytes, at);
            if (got <= 0)
                return false;
            out += got;
            at += got;
            bytes -= static_cast<size_t>(got);
        }
        return true;
    }

    std::vector<Shard> shards_;
    ShardHeader proto_;
    int batch_;
    bool shuffle_;
    size_t capacity_, min_after_;
    int part_, parts_;
    std::vector<uint64_t> members_;   // membership bitmap over the global record index (empty: every record)
    uint64_t total_ = 0;
    std::atomic<uint64_t> served_{0};
    std::mutex mutex_;
    std::condition_variable not_full_, not_empty_;
    std::vector<Record> pool_;
    std::vector<std::thread> readers_;
    std::mt19937_64 draw_rng_;
    bool stop_ = false, failed_ = false;
    std::string error_;
};

thread_local std::string g_last_error;

void* open_loader(char const* const* paths, int nshards, int batch, int nthreads, unsigned long long seed, int shuffle, long long pool_capacity, long long min_after_dequeue,
                  int part, int parts, unsigned long long const* bitmap, unsigned long long nbits) {
    if (nshards < 1 || batch < 1) {
        g_last_error = "need at least one shard and a positive batch size";
        return nullptr;
    }
    std::vector<Shard> shards;
    ShardHeader proto{};
    uint64_t total = 0;
    for (int i = 0; i < nshards; ++i) {
        Shard shard;
        shard.path = paths[i];
        shard.fd = ::open(paths[i], O_RDONLY);
        ShardHeader header{};
        if (shard.fd < 0 || ::pread(shard.fd, &header, sizeof(header), 0) != static_cast<ssize_t>(sizeof(header)) || std::memcmp(header.magic, kMagic, 8) != 0) {
            g_last_error = std::string("not a shard file: ") + paths[i];
            for (auto& s : shards)
                ::close(s.fd);
            if (shard.fd >= 0)
                ::close(shard.fd);
            return nullptr;
        }
        struct stat st{};
        if (::fstat(shard.fd, &st) != 0 || static_cast<uint64_t>(st.st_size) < sizeof(header) + header.count * (header.record_bytes + 8) ||
            header.record_bytes != static_cast<uint64_t>(header.height) * header.width * header.channels || header.label_bytes != 8) {
            g_last_error = std::string("truncated or inconsistent shard: ") + paths[i];
            for (auto& s : shards)
                ::close(s.fd);
            ::close(shard.fd);
            return nullptr;
        }
        if (i == 0) {
            proto = header;
        } else if (header.record_bytes != proto.record_bytes || header.height != proto.height || header.width != proto.width || header.channels != proto.channels) {
            g_last_error = std::string("shards with different image shapes: ") + paths[i];
            for (auto& s : shards)
                ::close(s.fd);
            ::close(shard.fd);
            return nullptr;
        }
        shard.count = header.count;
        shard.first = total;
        total += header.count;
        shards.push_back(shard);
    }
    std::vector<uint64_t> members;
    if (bitmap) {
        uint64_t set = 0;
        if (nbits == total) {
            members.assign(bitmap, bitmap + (total + 63) / 64);
            if (total % 64)
                members.back() &= (1ull << (total % 64)) - 1;
            for (uint64_t word : members)
                set += static_cast<uint64_t>(__builtin_popcountll(word));
        }
        if (nbits != total || set == 0) {
            g_last_error = "the membership bitmap must cover the " + std::to_string(total) + " records of the shards and select at least one";
            for (auto& s : shards)
                ::close(s.fd);
            return nullptr;
        }
    }
    if (nthreads < 1)
        nthreads = 1;
    if (nthreads > nshards && shuffle)
        nthreads = nshards;
    if (parts < 1)
        parts = 1;
    size_t capacity = pool_capacity > 0 ? static_cast<size_t>(pool_capacity) : static_cast<size_t>(batch) * 16;
    size_t min_after = min_after_dequeue >= 0 ? static_cast<size_t>(min_after_dequeue) : capacity / 2;
    if (capacity < static_cast<size_t>(batch))
        capacity = static_cast<size_t>(batch);
    if (min_after >= capacity)
        min_after = capacity - 1;
    return new Loader(std::move(shards), proto, batch, nthreads, seed, shuffle != 0, capacity, min_after, part, parts, std::move(members));
}

} // namespace

extern "C" {

// `paths`: nshards NUL-terminated file names. Returns an opaque handle or null (see agb_loader_last_error).
// `part` / `parts`: this reader only serves records whose index in their shard is congruent to part modulo parts.
void* agb_loader_open(char const* const* paths, int nshards, int batch, int nthreads, unsigned long long seed, int shuffle, long long pool_capacity, long long min_after_dequeue,
                      int part, int parts) {
    return open_loader(paths, nshards, batch, nthreads, seed, shuffle, pool_capacity, min_after_dequeue, part, parts, nullptr, 0);
}

// As `agb_loader_open` without part / parts, serving only the records whose bit is set in `bitmap` (64-bit words, bit g % 64 of word
// g / 64 for global record g: the shards in the order given, then the records of each). `nbits` must be the total number of records,
// and at least one bit must be set.
void* agb_loader_open_subset(char const* const* paths, int nshards, int batch, int nthreads, unsigned long long seed, int shuffle, long long pool_capacity,
                             long long min_after_dequeue, unsigned long long const* bitmap, unsigned long long nbits) {
    if (!bitmap) {
        g_last_error = "the subset reader needs a membership bitmap";
        return nullptr;
    }
    return open_loader(paths, nshards, batch, nthreads, seed, shuffle, pool_capacity, min_after_dequeue, 0, 1, bitmap, nbits);
}
int agb_loader_next(void* handle, void* images, void* labels) {
    Loader* loader = static_cast<Loader*>(handle);
    int status = loader->next(static_cast<uint8_t*>(images), static_cast<int64_t*>(labels));
    if (status != 0)
        g_last_error = loader->error();
    return status;
}

// out[0..5] = total records, records served so far, height, width, channels, record bytes
int agb_loader_info(void* handle, unsigned long long* out) {
    Loader* loader = static_cast<Loader*>(handle);
    out[0] = loader->total();
    out[1] = loader->served();
    out[2] = loader->proto().height;
    out[3] = loader->proto().width;
    out[4] = loader->proto().channels;
    out[5] = loader->proto().record_bytes;
    return 0;
}

void agb_loader_close(void* handle) {
    delete static_cast<Loader*>(handle);
}

char const* agb_loader_last_error() {
    return g_last_error.c_str();
}

} // extern "C"
