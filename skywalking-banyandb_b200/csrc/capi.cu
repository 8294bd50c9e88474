// capi.cu -- the C ABI of libbydbgpu.so (include/bydb_gpu.h): context, HBM part cache, query
// orchestration on CUDA streams.  Host logic only; every byte of page decoding happens in
// scan_kernels.cu.  There is no CPU fallback here: unsupported encodings surface as BYDB_ENOTSUP.
#include <cuda_runtime.h>
#include <unistd.h>

#include <algorithm>
#include <cstdio>
#include <chrono>
#include <condition_variable>
#include <cstddef>
#include <cstdlib>
#include <deque>
#include <functional>
#include <thread>
#include <future>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/bydb_gpu.h"
#include "part_dir.hpp"
#include "scan_kernels.cuh"
#include "index_kernels.cuh"

using namespace bydb;

namespace {

thread_local std::string g_last_error;
thread_local uint32_t g_last_dev_err = 0;  // DevErr of the last failed scan on this thread (drives the lazy unpack retry)
int fail(int code, const std::string &msg) {
    g_last_error = msg;
    return code;
}
// No exception may cross the C ABI ("never abort"): allocation failures and anything a hostile part provokes in the
// standard library become error codes.
template <class F>
int guarded(F &&f) {
    try {
        return f();
    } catch (const std::bad_alloc &) {
        return fail(BYDB_ENOMEM, "out of host memory");
    } catch (const std::exception &e) {
        return fail(BYDB_EINVAL, std::string("internal error: ") + e.what());
    } catch (...) {
        return fail(BYDB_EIO, "internal error: unknown exception");
    }
}
#define CUDA_TRY(expr)                                                                          \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess)                                                                  \
            return fail(BYDB_EIO, std::string(#expr) + ": " + cudaGetErrorString(_e));          \
    } while (0)

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// the layout of one device scratch allocation: each call carves `bytes` and returns their offset; regions start 256 B aligned
struct Carve {
    size_t o = 0;  // bytes carved so far
    size_t operator()(size_t bytes) {
        const size_t at = o;
        o = align_up(o + bytes, 256);
        return at;
    }
};

struct Part {
    uint64_t id = 0;
    PartDir dir;
    uint8_t *d_arena = nullptr;       // all file images, each 256 B aligned and padded
    uint8_t *d_dir = nullptr;         // DevBlock[] | DevCol[] | file pointer table
    uint8_t *d_unpack = nullptr;      // fallback pages rewritten at admission (unpack_kernels.cu); file slot `n_files`
    uint64_t unpacked_pages = 0, unpack_skipped = 0;
    const DevBlock *d_blocks = nullptr;
    const DevCol *d_cols = nullptr;
    const uint8_t *const *d_files = nullptr;
    uint64_t hbm_bytes = 0;
    int device = 0;
    cudaStream_t pool_stream = nullptr;  // transient parts (host path) live in the stream-ordered pool
    ~Part() {
        if (pool_stream) {
            if (d_arena) cudaFreeAsync(d_arena, pool_stream);
            if (d_dir) cudaFreeAsync(d_dir, pool_stream);
            if (d_unpack) cudaFreeAsync(d_unpack, pool_stream);
        } else {
            if (d_arena) cudaFree(d_arena);
            if (d_dir) cudaFree(d_dir);
            if (d_unpack) cudaFree(d_unpack);
        }
    }
};

// The zero page of a scan: zeroed on the device before plan_blocks, written by the kernels, and read back whole behind the
// last kernel of the step (errors + counters).
struct ZeroPage {
    uint32_t work_count, work_next;   // work list cursor
    uint32_t err[2];                  // DevErr (first error wins), block / series index
    unsigned long long stats[6];      // see ScanParams::stats
    int32_t col_type[kMaxFcols];
    unsigned long long dd_counts[2];  // version dedup: flagged blocks, flagged rows
    uint32_t slow_count, slow_next;   // slow-lane list cursor
    uint32_t rest_count, rest_next;   // express lane only: cursor of the blocks it left to the regular fast lane
};
static_assert(offsetof(ZeroPage, err) == 8 && offsetof(ZeroPage, stats) == 16 && offsetof(ZeroPage, col_type) == 64 &&
                  offsetof(ZeroPage, dd_counts) == 96 && offsetof(ZeroPage, slow_count) == 112 && offsetof(ZeroPage, rest_count) == 120,
              "zero page layout");
constexpr size_t kZeroPageBytes = 256;  // zeroed and read back per scan
static_assert(sizeof(ZeroPage) <= kZeroPageBytes, "zero page size");

// One in-flight call: stream, events and a pinned staging buffer.
struct ExecSlot {
    cudaStream_t stream = nullptr;
    static constexpr int kMaxBatches = 8;  // pipelined cold path: one set of events / zero page per batch
    cudaEvent_t ev[4 * kMaxBatches] = {};
    uint8_t *pinned = nullptr;
    size_t pinned_bytes = 0;
    uint8_t *zpage = nullptr;  // pinned, kZeroPageBytes per batch: read-back of the zero pages
    ZeroPage *page(int batch) { return reinterpret_cast<ZeroPage *>(zpage + kZeroPageBytes * static_cast<size_t>(batch)); }
    bool express[kMaxBatches] = {};  // per batch: run_scan launched the express lane (its zero-page counter is meaningful)
    cudaEvent_t busy = nullptr;  // recorded by a call that returned before its work finished (asynchronous scan_partials)
    bool busy_pending = false;
    void wait_idle() {
        if (busy_pending) cudaEventSynchronize(busy);
        busy_pending = false;
    }
    // Page-locked allocations (and frees) are implicit synchronisation points of the device: no kernel issued after one starts
    // before every kernel issued before it has finished.  When several ranks share a device, a rank whose wait kernel is spinning
    // for a peer would then never see that peer's kernels start (the peer's call just allocated staging memory) -- a 60 s
    // stall ending in BYDB_EIO.  So: every slot is created with kInitialPinned bytes at bydb_init, grows geometrically and
    // rarely, and nothing is freed before bydb_shutdown.
    static constexpr size_t kInitialPinned = 1u << 20;
    std::vector<uint8_t *> retired;
    int ensure_pinned(size_t n) {
        if (n <= pinned_bytes) return 0;
        size_t want = align_up(std::max(n, 2 * pinned_bytes), 1 << 16);
        uint8_t *fresh = nullptr;
        if (cudaMallocHost(reinterpret_cast<void **>(&fresh), want) != cudaSuccess) {
            cudaGetLastError();
            want = align_up(n, 1 << 16);
            if (cudaMallocHost(reinterpret_cast<void **>(&fresh), want) != cudaSuccess) return -1;
        }
        if (pinned) retired.push_back(pinned);  // copies from it may still be in flight; freed at shutdown
        pinned = fresh;
        pinned_bytes = want;
        return 0;
    }
    int create() {
        if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess) return -1;
        for (auto &e : ev)
            if (cudaEventCreate(&e) != cudaSuccess) return -1;
        if (cudaMallocHost(reinterpret_cast<void **>(&zpage), kZeroPageBytes * kMaxBatches) != cudaSuccess) return -1;
        if (cudaEventCreateWithFlags(&busy, cudaEventDisableTiming) != cudaSuccess) return -1;
        return ensure_pinned(kInitialPinned);
    }
    ExecSlot() = default;
    ExecSlot(const ExecSlot &) = delete;
    ExecSlot &operator=(const ExecSlot &) = delete;
    // with the slot's device current and none of its work in flight
    ~ExecSlot() {
        if (stream) cudaStreamDestroy(stream);
        for (auto &e : ev)
            if (e) cudaEventDestroy(e);
        if (busy) cudaEventDestroy(busy);
        if (pinned) cudaFreeHost(pinned);
        for (uint8_t *r : retired) cudaFreeHost(r);
        if (zpage) cudaFreeHost(zpage);
    }
};

}  // namespace

// A few persistent host threads for the cold path's block-index parsing: creating a dozen threads per query costs
// more (serialised on the calling thread) than parsing the first primary block.
class WorkPool {
  public:
    ~WorkPool() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
        }
        cv_.notify_all();
        for (auto &t : th_) t.join();
    }
    void submit(std::function<void()> fn) {
        {
            std::lock_guard<std::mutex> lk(mu_);
            if (th_.empty()) {
                unsigned hw = std::thread::hardware_concurrency();
                const unsigned n = std::max(2u, std::min(32u, hw ? hw / 2 : 4u));  // index parsing + page gathering: memory-bound helpers
                for (unsigned i = 0; i < n; ++i) th_.emplace_back([this] { run(); });
            }
            q_.push_back(std::move(fn));
        }
        cv_.notify_one();
    }

  private:
    void run() {
        for (;;) {
            std::function<void()> fn;
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [this] { return stop_ || !q_.empty(); });
                if (q_.empty()) return;  // stop_ and drained
                fn = std::move(q_.front());
                q_.pop_front();
            }
            fn();
        }
    }
    std::mutex mu_;
    std::condition_variable cv_;
    std::deque<std::function<void()>> q_;
    std::vector<std::thread> th_;
    bool stop_ = false;
};

// Peer mailboxes of the multi-GPU reduce (bydb_comm_*).  Layout of one rank's mailbox (device memory of that rank):
//   [0, 4096)        control: arrival flags (u64 epoch per writer rank) at 0, status words (epoch << 32 | host-side error of
//                    that rank's call) at 1024, `done` epoch at 2048, error word of this rank's wait kernels at 2056
//   [4096, ...)      2 parities x nranks slots of slot_bytes each (partial tables written by the peers)
constexpr int kCommMaxRanks = 64;
constexpr size_t kCommCtl = 4096, kCommStatusOff = 1024, kCommDoneOff = 2048, kCommErrOff = 2056, kCommArgsOff = 2112;
struct Comm {
    int rank = -1, nranks = 0;
    uint8_t *mine = nullptr;            // this rank's mailbox (cudaMalloc)
    size_t slot_bytes = 0, mailbox_bytes = 0;
    std::vector<uint8_t *> peer;        // device-visible base of every rank's mailbox
    std::vector<bool> ipc_opened;
    std::vector<size_t> peer_slot_bytes;
    uint64_t epoch = 0;
    std::vector<uint64_t> last_use;     // [root * 2 + parity] epoch of the previous collective that used that root's slots of that parity
    std::mutex mu;                      // collective calls are issued one at a time per context
    // A peer lives on THIS GPU (tests on a one-GPU box, more ranks than GPUs): no wait kernel may spin there.  CUDA gives no
    // forward-progress guarantee between streams of one device -- they share a handful of hardware queues, and work queued
    // behind the dependants of a spinning kernel in the same queue never launches, so a rank could wait forever for a peer
    // whose kernels sit behind its own wait kernel (seen as collectives that stalled until the 60 s bound, depending on how
    // many streams the process had created before).  In this mode the HOST polls the flags and the prepared form keeps the
    // plain path.  Ranks on different GPUs keep the device-side waits.
    bool shared_device = false;
    cudaStream_t poll_stream = nullptr;
    unsigned long long *poll_buf = nullptr;  // pinned, kCommMaxRanks words
};

// Pinned staging ring of the gather path (host images in PAGEABLE memory): the pages a query touches are collected into
// these buffers by the worker pool and go up with asynchronous copies, chunk k+1 being gathered while chunk k is on the bus.
struct StageRing {
    static constexpr int kBufs = 3;
    static constexpr size_t kBytes = 64u << 20;
    uint8_t *buf[kBufs] = {};
    cudaEvent_t done[kBufs] = {};
    bool pending[kBufs] = {};
    int next = 0;
    std::mutex mu;  // one gathering call at a time per context
};

struct bydb_ctx {
    int device = 0;
    int sm_count = 0;
    int ctas_per_sm = 2;       // slow lane (general decoder)
    int ctas_per_sm_fast = 2;  // fast lane
    int ctas_per_sm_express = 2;  // express lane (its own shared-memory ring)
    uint64_t hbm_budget = 0;
    uint64_t hbm_used = 0;
    bool host_index = false;   // BYDB_CFG_HOST_INDEX: parse the block index of resident parts on the host (part_dir.cc)
    std::mutex mu;
    NameTable names;
    std::unordered_map<bydb_part_h, std::shared_ptr<Part>> parts;
    std::unordered_map<uint64_t, bydb_part_h> by_id;
    bydb_part_h next_handle = 1;
    std::vector<std::unique_ptr<ExecSlot>> free_slots;
    WorkPool pool;
    Comm comm;
    StageRing stage;
};

namespace {

// The HBM budget (bydb_cfg.hbm_budget_bytes, 0 = none) is an account of the device memory the context holds for parts and the
// mailbox: every reservation is given back with hbm_release when that memory goes, or when its allocation fails.
int hbm_reserve(bydb_ctx *ctx, uint64_t bytes, const char *msg = "HBM budget exceeded") {
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->hbm_budget && ctx->hbm_used + bytes > ctx->hbm_budget) return fail(BYDB_ENOMEM, msg);
    ctx->hbm_used += bytes;
    return 0;
}
void hbm_release(bydb_ctx *ctx, uint64_t bytes) {
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->hbm_used -= bytes;
}

struct SlotLease {
    bydb_ctx *ctx;
    std::unique_ptr<ExecSlot> slot;
    SlotLease(bydb_ctx *c) : ctx(c) {
        std::lock_guard<std::mutex> lk(c->mu);
        if (!c->free_slots.empty()) {
            slot = std::move(c->free_slots.back());
            c->free_slots.pop_back();
        }
    }
    int init() {
        if (slot) {
            slot->wait_idle();  // its pinned staging may still feed an asynchronous call's copies
            return 0;
        }
        slot.reset(new ExecSlot());   // more concurrent callers than slots made at bydb_init
        return slot->create();
    }
    ~SlotLease() {
        if (!slot) return;
        std::lock_guard<std::mutex> lk(ctx->mu);
        ctx->free_slots.push_back(std::move(slot));
    }
};

struct ResultOwner {
    std::vector<int32_t> group_id;
    std::vector<int64_t> rows;
    std::vector<uint8_t> is_float;
    std::vector<int64_t> val_i64;
    std::vector<double> val_f64;
};

// query after name resolution
struct Plan {
    std::vector<std::shared_ptr<Part>> parts;
    std::vector<std::string> fcols;       // distinct aggregated fields
    std::vector<int> agg_fcol;
    int32_t n_groups = 1;
    TableLayout tl = TableLayout(1, 1);   // the partial table of n_groups x fcols
    uint32_t total_blocks = 0;
    uint64_t n_series = 0;
};

const char *dev_err_text(uint32_t code) {
    switch (code) {
        case kErrPlainPage: return "numeric fallback page (EncodeTypePlain: null cells or non-decimal floats) is not decoded on the device yet";
        case kErrZstdDict: return "dictionary page with a zstd-compressed value block is not decoded on the device yet";
        case kErrBigBlock: return "row predicate on a block larger than the shared-memory row mask (8448 rows)";
        case kErrCorrupt: return "corrupt page: varint stream / header does not match the block's row count";
        case kErrTypeMix: return "a field is stored with different value types across blocks";
        case kErrBadEnc: return "unknown encode type byte";
        case kErrTagPlain: return "high-cardinality string tag page (plain bytes block) is not decoded on the device yet";
        case kErrOverlap: return "a series lives in several parts with overlapping time spans and the dedup pass did not run (internal error)";
        case kErrPredType: return "predicate literal type does not match the stored tag column type";
        case kErrTmaTimeout: return "internal error: a TMA bulk copy did not complete";
        case kErrPeerTimeout: return "multi-GPU reduce: a peer rank did not deliver its partial table in time";
        case kErrKeyCap: return "per-row group key: more distinct key values than bydb_group_key.max_values";
        case kErrKeyLong: return "per-row group key: a key value longer than 64 bytes";
        case kErrRankOverlap: return "keyed collective: a series lives on several ranks over time spans that intersect";
    }
    return "unknown device error";
}
int dev_err_code(uint32_t code) { return code == kErrKeyCap ? BYDB_ENOMEM : (code == kErrCorrupt || code == kErrBadEnc || code == kErrTypeMix || code == kErrPredType) ? BYDB_EINVAL : (code == kErrTmaTimeout || code == kErrPeerTimeout) ? BYDB_EIO : BYDB_ENOTSUP; }

int validate_query(const bydb_query *q, bool need_parts) {
    if (!q) return fail(BYDB_EINVAL, "query is NULL");
    if (need_parts && (q->n_parts == 0 || !q->parts)) return fail(BYDB_EINVAL, "query has no parts");
    if (q->n_parts > kMaxParts) return fail(BYDB_EINVAL, "too many parts in one query (max 64)");
    if (q->n_series > 0 && !q->series_ids) return fail(BYDB_EINVAL, "series_ids is NULL");
    if (q->n_series > 0x7fffffffull) return fail(BYDB_EINVAL, "too many series");
    if (q->n_aggs == 0 || q->n_aggs > 32 || !q->aggs) return fail(BYDB_EINVAL, "need 1..32 aggregations");
    if (q->n_preds > kMaxPreds) return fail(BYDB_EINVAL, "too many predicates (max 8)");
    if (q->n_preds > 0 && !q->preds) return fail(BYDB_EINVAL, "preds is NULL");
    if (q->series_group && q->n_groups < 1) return fail(BYDB_EINVAL, "n_groups must be >= 1 when series_group is given");
    for (uint64_t i = 1; i < q->n_series; ++i)
        if (q->series_ids[i] <= q->series_ids[i - 1]) return fail(BYDB_EINVAL, "series_ids must be ascending and unique (query.go:601)");
    if (q->series_group)
        for (uint64_t i = 0; i < q->n_series; ++i)
            if (q->series_group[i] < 0 || q->series_group[i] >= q->n_groups) return fail(BYDB_EINVAL, "series_group out of range");
    for (uint32_t a = 0; a < q->n_aggs; ++a) {
        if (!q->aggs[a].field) return fail(BYDB_EINVAL, "aggregation without a field");
        if (q->aggs[a].func < BYDB_AGG_MEAN || q->aggs[a].func > BYDB_AGG_SUM) return fail(BYDB_EINVAL, "unknown aggregation function");
    }
    for (uint32_t i = 0; i < q->n_preds; ++i) {
        const bydb_pred &p = q->preds[i];
        if (!p.family || !p.tag) return fail(BYDB_EINVAL, "predicate without family/tag");
        if (p.op < BYDB_OP_EQ || p.op > BYDB_OP_GE) return fail(BYDB_EINVAL, "unknown predicate operator");
        if (p.value_type != BYDB_VT_INT64 && p.value_type != BYDB_VT_STR && p.value_type != BYDB_VT_BINARY)
            return fail(BYDB_EINVAL, "predicate literal must be int64, string or binary");
        if (p.value_type != BYDB_VT_INT64 && p.lit_len > kMaxLit) return fail(BYDB_ENOTSUP, "string predicate literal longer than 64 bytes");
        if (p.value_type != BYDB_VT_INT64 && p.lit_len > 0 && !p.lit) return fail(BYDB_EINVAL, "predicate literal is NULL");
    }
    if (q->top_n < 0 || (q->top_n > 0 && (q->top_agg < 0 || static_cast<uint32_t>(q->top_agg) >= q->n_aggs)))
        return fail(BYDB_EINVAL, "bad top_n / top_agg");
    // checked before anything is enqueued: a refusal after run_scan would leave work in flight on a pooled stream
    if (q->top_n > kMaxDeviceTopN) return fail(BYDB_ENOTSUP, "top_n larger than 2048 is not supported on the device path");
    return 0;
}

// The shape of a (validated) query's partial table, into `plan`: its distinct aggregated fields, the field of each
// aggregation, the series groups and the table layout.  Fills all of them, then refuses more fields than a table holds.
int query_shape(const bydb_query *q, Plan &plan) {
    for (uint32_t a = 0; a < q->n_aggs; ++a) {
        std::string f = q->aggs[a].field;
        int idx = -1;
        for (size_t i = 0; i < plan.fcols.size(); ++i)
            if (plan.fcols[i] == f) idx = static_cast<int>(i);
        if (idx < 0) {
            plan.fcols.push_back(f);
            idx = static_cast<int>(plan.fcols.size() - 1);
        }
        plan.agg_fcol.push_back(idx);
    }
    plan.n_groups = q->series_group ? q->n_groups : 1;
    plan.n_series = q->n_series;
    plan.tl = TableLayout(static_cast<size_t>(plan.n_groups), plan.fcols.size());
    if (plan.fcols.size() > kMaxFcols) return fail(BYDB_EINVAL, "too many distinct aggregated fields (max 8)");
    return 0;
}

// the caller's file list of one part, checked
int file_images(const bydb_part_files *files, std::vector<FileImage> &imgs) {
    if (!files || files->n_files == 0 || !files->files) return fail(BYDB_EINVAL, "no files");
    for (uint32_t i = 0; i < files->n_files; ++i) {
        const bydb_file &f = files->files[i];
        if (!f.name || (!f.data && f.len)) return fail(BYDB_EINVAL, "file without name/data");
        imgs.push_back(FileImage{f.name, f.data, f.len});
    }
    return 0;
}

int unpack_fallback_pages(bydb_ctx *ctx, Part &part, size_t n_files, cudaStream_t s);
int build_part_dir_device(bydb_ctx *ctx, const std::vector<FileImage> &imgs, Part &part, const std::vector<std::string> &families, cudaStream_t s, size_t n_files,
                          size_t *dir_bytes_out);

// how register_part_locked_free admits a part
struct AdmitOptions {
    bool zero_copy = false;     // the data files stay in (pinned, device-mapped) host memory and the kernels read the pages they
                                // need straight over PCIe; only the block directory is uploaded
    bool transient = false;     // for the length of one call: device memory from the stream-ordered pool
    bool unpack = false;        // fallback pages are rewritten at admission (unpack_fallback_pages)
    PartDir *parsed = nullptr;  // the block index as the caller parsed it already
    bool device_index = false;  // the block index is parsed by kernels (resident parts without `parsed`)
};

int register_part_locked_free(bydb_ctx *ctx, uint64_t part_id, const bydb_part_files *files, std::shared_ptr<Part> &out, uint64_t *h2d,
                              const AdmitOptions &opt) {
    std::vector<FileImage> imgs;
    if (int rc = file_images(files, imgs)) return rc;
    auto part = std::make_shared<Part>();
    part->id = part_id;
    part->device = ctx->device;
    std::string err;
    // resident parts: the block index is inflated and parsed by kernels (index_kernels.cu); the host only decides the file table
    const bool dev_index = opt.device_index && !opt.parsed && !opt.zero_copy;
    std::vector<std::string> families;
    if (dev_index) {
        for (const auto &f : imgs)
            if (f.name.size() > 4 && f.name.compare(f.name.size() - 4, 4, ".tfm") == 0) families.push_back(f.name.substr(0, f.name.size() - 4));
        std::sort(families.begin(), families.end());
        if (families.size() > 250) return fail(BYDB_EINVAL, "too many tag family files");
        part->dir.files = {"timestamps.bin", "fv.bin"};
        for (const auto &fam : families) part->dir.files.push_back(fam + ".tf");
    } else if (opt.parsed) {
        part->dir = std::move(*opt.parsed);  // the caller parsed this slice of the block index already (cold path, in the background)
    } else {
        int rc = build_part_dir(imgs, ctx->names, part->dir, err);
        if (rc) return fail(rc, "part " + std::to_string(part_id) + ": " + err);
    }
    // arena: each data file 256 B aligned with >= 256 B of slack after it (TMA over-read, bit windows)
    std::vector<size_t> offs;
    size_t arena = 0;
    std::vector<const FileImage *> order;
    for (const auto &name : part->dir.files) {
        const FileImage *img = nullptr;
        for (const auto &f : imgs)
            if (f.name == name) img = &f;
        if (!img) return fail(BYDB_ENOENT, "missing file " + name);
        order.push_back(img);
        offs.push_back(arena);
        arena = align_up(arena + img->len + 256, 256);
    }
    std::vector<const uint8_t *> mapped(order.size(), nullptr);
    if (opt.zero_copy) {
        for (size_t i = 0; i < order.size(); ++i) {
            if (order[i]->len == 0) continue;
            cudaPointerAttributes at;
            if (cudaPointerGetAttributes(&at, order[i]->data) != cudaSuccess || at.type != cudaMemoryTypeHost || !at.devicePointer) {
                cudaGetLastError();
                return fail(BYDB_EINVAL, "BYDB_Q_HOST_ZERO_COPY needs file images in pinned, device-mapped host memory (" + order[i]->name + ")");
            }
            if (reinterpret_cast<uintptr_t>(at.devicePointer) & 15) return fail(BYDB_EINVAL, "zero-copy file images must be 16-byte aligned");
            mapped[i] = static_cast<const uint8_t *>(at.devicePointer);
        }
        arena = 0;
    }
    const size_t nb = part->dir.blocks.size(), nc = part->dir.cols.size(), nf = order.size();
    const size_t dir_bytes = dev_index ? 0 : align_up(nb * sizeof(DevBlock), 256) + align_up(nc * sizeof(DevCol), 256) + align_up((nf + 1) * sizeof(void *), 256);
    if (int rc = hbm_reserve(ctx, arena + dir_bytes)) return rc;
    part->hbm_bytes = arena + dir_bytes;
    // every failure from here on gives the part's reservation back; the directory and the unpack arena add to it
    struct Undo {
        bydb_ctx *ctx;
        const Part *part;
        bool keep = false;
        ~Undo() {
            if (!keep) hbm_release(ctx, part->hbm_bytes);
        }
    } undo{ctx, part.get()};
    SlotLease lease(ctx);
    if (lease.init()) return fail(BYDB_EIO, "cannot create stream");
    cudaStream_t s = lease.slot->stream;
    bool alloc_ok;
    if (opt.transient) {
        part->pool_stream = s;
        alloc_ok = cudaMallocAsync(reinterpret_cast<void **>(&part->d_arena), arena ? arena : 256, s) == cudaSuccess &&
                   (dev_index || cudaMallocAsync(reinterpret_cast<void **>(&part->d_dir), dir_bytes ? dir_bytes : 256, s) == cudaSuccess);
    } else {
        alloc_ok = cudaMalloc(reinterpret_cast<void **>(&part->d_arena), arena ? arena : 256) == cudaSuccess &&
                   (dev_index || cudaMalloc(reinterpret_cast<void **>(&part->d_dir), dir_bytes ? dir_bytes : 256) == cudaSuccess);
    }
    if (!alloc_ok) return fail(BYDB_ENOMEM, "device allocation failed for part " + std::to_string(part_id));
    cudaError_t e = cudaSuccess;
    if (!opt.zero_copy) {
        e = cudaMemsetAsync(part->d_arena, 0, arena ? arena : 256, s);
        for (size_t i = 0; i < nf && e == cudaSuccess; ++i)
            if (order[i]->len) e = cudaMemcpyAsync(part->d_arena + offs[i], order[i]->data, order[i]->len, cudaMemcpyHostToDevice, s);
    }
    if (dev_index) {
        if (e != cudaSuccess) return fail(BYDB_EIO, std::string("part upload: ") + cudaGetErrorString(e));
        size_t dbytes = 0;
        int rc = build_part_dir_device(ctx, imgs, *part, families, s, nf, &dbytes);
        std::vector<const uint8_t *> table(nf + 1, nullptr);
        for (size_t i = 0; i < nf; ++i) table[i] = part->d_arena + offs[i];
        if (!rc && cudaMemcpyAsync(const_cast<uint8_t **>(reinterpret_cast<const uint8_t *const *>(part->d_files)), table.data(), nf * sizeof(void *),
                                   cudaMemcpyHostToDevice, s) != cudaSuccess)
            rc = fail(BYDB_EIO, "part upload: file table");
        if (!rc && cudaStreamSynchronize(s) != cudaSuccess) rc = fail(BYDB_EIO, "part upload: synchronize");
        if (rc) {
            cudaStreamSynchronize(s);
            return rc;
        }
        if (h2d) {
            for (size_t i = 0; i < nf; ++i) *h2d += order[i]->len;
            *h2d += dbytes;
        }
        if (opt.unpack) {
            rc = unpack_fallback_pages(ctx, *part, nf, s);
            if (rc) return rc;
        }
        undo.keep = true;
        out = part;
        return 0;
    }
    // directory
    if (lease.slot->ensure_pinned(dir_bytes ? dir_bytes : 256)) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
    uint8_t *hdir = lease.slot->pinned;  // the directory goes up from pinned staging in one copy
    if (nb) memcpy(hdir, part->dir.blocks.data(), nb * sizeof(DevBlock));
    const size_t off_cols = align_up(nb * sizeof(DevBlock), 256);
    if (nc) memcpy(hdir + off_cols, part->dir.cols.data(), nc * sizeof(DevCol));
    const size_t off_files = off_cols + align_up(nc * sizeof(DevCol), 256);
    for (size_t i = 0; i < nf; ++i) {
        const uint8_t *pfile = opt.zero_copy ? mapped[i] : part->d_arena + offs[i];
        memcpy(hdir + off_files + i * sizeof(void *), &pfile, sizeof(void *));
    }
    if (e == cudaSuccess && dir_bytes) e = cudaMemcpyAsync(part->d_dir, hdir, dir_bytes, cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) return fail(BYDB_EIO, std::string("part upload: ") + cudaGetErrorString(e));
    part->d_blocks = reinterpret_cast<const DevBlock *>(part->d_dir);
    part->d_cols = reinterpret_cast<const DevCol *>(part->d_dir + off_cols);
    part->d_files = reinterpret_cast<const uint8_t *const *>(part->d_dir + off_files);
    if (h2d) {
        if (!opt.zero_copy)
            for (size_t i = 0; i < nf; ++i) *h2d += order[i]->len;
        *h2d += dir_bytes;
    }
    if (opt.unpack) {
        const int rc = unpack_fallback_pages(ctx, *part, nf, s);
        if (rc) return rc;
    }
    undo.keep = true;
    out = part;
    return 0;
}

// The parts a host-image entry point admits for the length of one call, with ids ~0, ~0 - 1, ...: their budget goes back when
// this goes away, their memory (stream-ordered) once the last holder lets go.
struct TransientParts {
    bydb_ctx *ctx;
    std::vector<std::shared_ptr<Part>> parts;
    explicit TransientParts(bydb_ctx *c) : ctx(c) {}
    TransientParts(const TransientParts &) = delete;
    TransientParts &operator=(const TransientParts &) = delete;
    ~TransientParts() {
        for (auto &p : parts) hbm_release(ctx, p->hbm_bytes);
    }
    uint64_t next_id() const { return ~0ull - parts.size(); }
    int admit(const bydb_part_files *files, uint64_t *h2d, AdmitOptions opt) {
        opt.transient = true;
        std::shared_ptr<Part> p;
        const int rc = register_part_locked_free(ctx, next_id(), files, p, h2d, opt);
        if (!rc) parts.push_back(std::move(p));
        return rc;
    }
};


// ------------------------------------------------------------------------------------------------
// Block index on the device (index_kernels.cu): meta.bin / primary.bin / *.tfm go up as they are, the zstd frames are
// inflated and the blockMetadata records walked by kernels; the host only sizes the buffers between the phases and maps
// the handful of interned column names to the context's ids.  Fills part.dir (host copy of the directory) and writes
// DevBlock[] / DevCol[] straight into the part's device directory.
// ------------------------------------------------------------------------------------------------
// device memory from the stream-ordered pool, freed on its stream (behind the work that uses it) when this goes out of scope
struct Scratch {
    uint8_t *base = nullptr;
    cudaStream_t stream = nullptr;
    ~Scratch() {
        if (base) cudaFreeAsync(base, stream);
    }
    cudaError_t alloc(size_t n, cudaStream_t s) {
        stream = s;
        return cudaMallocAsync(reinterpret_cast<void **>(&base), n ? n : 256, s);
    }
};

const char *index_err_text(uint32_t e) {
    switch (e) {
        case kIdxBadMeta: return "meta.bin: not a zstd frame of 40-byte primaryBlockMetadata records in order inside primary.bin";
        case kIdxBadFrame: return "primary block does not inflate to its declared size";
        case kIdxBadBlock: return "corrupt blockMetadata";
        case kIdxBadEnc: return "unexpected timestamps encode type";
        case kIdxBadColumn: return "corrupt columnMetadata";
        case kIdxFamily: return "tag family: missing or truncated .tf/.tfm";
        case kIdxOrder: return "blockMetadata out of order";
        case kIdxNames: return "too many / too long column names for the device index";
        case kIdxTooManyFamilies: return "more than 16 tag families in a block";
    }
    return "block index error";
}

// The part's device directory [DevBlock[nb] | DevCol[nc] | file table], charged to the part: sets d_dir / d_blocks /
// d_cols / d_files.
int alloc_part_dir(bydb_ctx *ctx, Part &part, size_t nb, size_t nc, size_t n_files, cudaStream_t s, size_t *dir_bytes_out) {
    const size_t off_cols = align_up(nb * sizeof(DevBlock), 256);
    const size_t off_files = off_cols + align_up(nc * sizeof(DevCol), 256);
    const size_t dir_bytes = off_files + align_up((n_files + 1) * sizeof(void *), 256);
    if (int rc = hbm_reserve(ctx, dir_bytes)) return rc;
    part.hbm_bytes += dir_bytes;
    *dir_bytes_out = dir_bytes;
    const cudaError_t ae = part.pool_stream ? cudaMallocAsync(reinterpret_cast<void **>(&part.d_dir), dir_bytes, s) : cudaMalloc(reinterpret_cast<void **>(&part.d_dir), dir_bytes);
    if (ae != cudaSuccess) {
        part.d_dir = nullptr;
        return fail(BYDB_ENOMEM, "device allocation failed for the directory of part " + std::to_string(part.id));
    }
    part.d_blocks = reinterpret_cast<const DevBlock *>(part.d_dir);
    part.d_cols = reinterpret_cast<const DevCol *>(part.d_dir + off_cols);
    part.d_files = reinterpret_cast<const uint8_t *const *>(part.d_dir + off_files);
    return 0;
}

// A part whose column names do not fit the device walker's table (more than kIndexMaxNames distinct names, or one longer
// than kIndexNameMax bytes) is still a valid part: its directory comes from the host parser, with the host's file ids
// (first use) renumbered onto the file table the caller laid the arena out by (sorted families).
int build_part_dir_host_for_device(bydb_ctx *ctx, const std::vector<FileImage> &imgs, Part &part, cudaStream_t s, size_t n_files, size_t *dir_bytes_out) {
    PartDir dir;
    std::string err;
    if (int rc = build_part_dir(imgs, ctx->names, dir, err)) return fail(rc, "part " + std::to_string(part.id) + ": " + err);
    std::vector<uint8_t> remap(dir.files.size(), 0);
    for (size_t i = 0; i < dir.files.size(); ++i) {
        size_t k = 0;
        while (k < part.dir.files.size() && part.dir.files[k] != dir.files[i]) ++k;
        if (k == part.dir.files.size()) return fail(BYDB_EINVAL, "part " + std::to_string(part.id) + ": " + dir.files[i] + " is not in the file table");
        remap[i] = static_cast<uint8_t>(k);
    }
    for (DevCol &c : dir.cols) c.file_id = remap[c.file_id];
    dir.files = std::move(part.dir.files);
    part.dir = std::move(dir);
    const size_t nb = part.dir.blocks.size(), nc = part.dir.cols.size();
    if (int rc = alloc_part_dir(ctx, part, nb, nc, n_files, s, dir_bytes_out)) return rc;
    if (nb) CUDA_TRY(cudaMemcpyAsync(const_cast<DevBlock *>(part.d_blocks), part.dir.blocks.data(), nb * sizeof(DevBlock), cudaMemcpyHostToDevice, s));
    if (nc) CUDA_TRY(cudaMemcpyAsync(const_cast<DevCol *>(part.d_cols), part.dir.cols.data(), nc * sizeof(DevCol), cudaMemcpyHostToDevice, s));
    return 0;
}

// files: the part's file table (timestamps.bin, fv.bin, <family>.tf ...) is already decided by the caller; d_dir_* are
// allocated here once the counts are known.
int build_part_dir_device(bydb_ctx *ctx, const std::vector<FileImage> &imgs, Part &part, const std::vector<std::string> &families, cudaStream_t s,
                          size_t n_files, size_t *dir_bytes_out) {
    auto find = [&](const std::string &name) -> const FileImage * {
        for (const auto &f : imgs)
            if (f.name == name) return &f;
        return nullptr;
    };
    const FileImage *meta = find("meta.bin"), *primary = find("primary.bin"), *tsf = find("timestamps.bin"), *fvf = find("fv.bin");
    if (!meta || !primary || !tsf || !fvf) return fail(BYDB_ENOENT, "part needs meta.bin, primary.bin, timestamps.bin and fv.bin");
    // ---- the index files go up verbatim: [meta | primary | tfm ... | family names]
    std::vector<const FileImage *> tfm(families.size()), tf(families.size());
    size_t up = align_up(meta->len, 256) + align_up(primary->len, 256);
    const size_t off_primary = align_up(meta->len, 256);
    std::vector<size_t> off_tfm(families.size()), off_name(families.size());
    for (size_t i = 0; i < families.size(); ++i) {
        tfm[i] = find(families[i] + ".tfm");
        tf[i] = find(families[i] + ".tf");
        if (!tfm[i] || !tf[i]) return fail(BYDB_EINVAL, "tag family '" + families[i] + "': missing .tf/.tfm");
        off_tfm[i] = up;
        up += align_up(tfm[i]->len, 256);
    }
    for (size_t i = 0; i < families.size(); ++i) {
        off_name[i] = up;
        up += align_up(families[i].size(), 16);
    }
    const size_t off_fams = align_up(up, 256);
    up = off_fams + align_up(families.size() * sizeof(IndexFamily), 256);
    const size_t off_ctl = up;
    up += 256;
    const size_t off_names = up;
    up += kIndexMaxNames * sizeof(IndexName);
    const size_t off_map = up;
    up += align_up(kIndexMaxNames * sizeof(uint16_t), 256);
    Scratch in;
    if (in.alloc(up, s)) return fail(BYDB_ENOMEM, "device allocation failed (index files)");
    CUDA_TRY(cudaMemsetAsync(in.base + off_ctl, 0, 256 + kIndexMaxNames * sizeof(IndexName), s));
    if (meta->len) CUDA_TRY(cudaMemcpyAsync(in.base, meta->data, meta->len, cudaMemcpyHostToDevice, s));
    if (primary->len) CUDA_TRY(cudaMemcpyAsync(in.base + off_primary, primary->data, primary->len, cudaMemcpyHostToDevice, s));
    std::vector<IndexFamily> fams(families.size());
    for (size_t i = 0; i < families.size(); ++i) {
        if (tfm[i]->len) CUDA_TRY(cudaMemcpyAsync(in.base + off_tfm[i], tfm[i]->data, tfm[i]->len, cudaMemcpyHostToDevice, s));
        CUDA_TRY(cudaMemcpyAsync(in.base + off_name[i], families[i].data(), families[i].size(), cudaMemcpyHostToDevice, s));
        memset(&fams[i], 0, sizeof fams[i]);
        fams[i].name = in.base + off_name[i];
        fams[i].name_len = static_cast<uint32_t>(families[i].size());
        fams[i].tfm = in.base + off_tfm[i];
        fams[i].tfm_len = tfm[i]->len;
        fams[i].tf_len = tf[i]->len;
        fams[i].file_id = static_cast<uint8_t>(2 + i);
    }
    if (!fams.empty()) CUDA_TRY(cudaMemcpyAsync(in.base + off_fams, fams.data(), fams.size() * sizeof(IndexFamily), cudaMemcpyHostToDevice, s));
    IndexCtl ctl0;
    memset(&ctl0, 0, sizeof ctl0);
    ctl0.min_ts = INT64_MAX;
    ctl0.max_ts = INT64_MIN;
    CUDA_TRY(cudaMemcpyAsync(in.base + off_ctl, &ctl0, sizeof ctl0, cudaMemcpyHostToDevice, s));
    IndexParams ip;
    memset(&ip, 0, sizeof ip);
    ip.meta = in.base;
    ip.primary = in.base + off_primary;
    ip.meta_len = meta->len;
    ip.primary_len = primary->len;
    ip.ts_len = tsf->len;
    ip.fv_len = fvf->len;
    ip.n_families = static_cast<uint32_t>(families.size());
    ip.families = reinterpret_cast<const IndexFamily *>(in.base + off_fams);
    ip.ctl = reinterpret_cast<IndexCtl *>(in.base + off_ctl);
    ip.names = reinterpret_cast<IndexName *>(in.base + off_names);
    ip.name_map = reinterpret_cast<const uint16_t *>(in.base + off_map);
    IndexCtl ctl;
    auto read_ctl = [&]() -> int {
        CUDA_TRY(cudaMemcpyAsync(&ctl, in.base + off_ctl, sizeof ctl, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        // more than 16 families in a block: a valid part this library does not read, as part_dir.cc says too
        const int code = ctl.err == kIdxTooManyFamilies ? BYDB_ENOTSUP : BYDB_EINVAL;
        if (ctl.err) return fail(code, "part " + std::to_string(part.id) + ": " + index_err_text(ctl.err) + " (#" + std::to_string(ctl.err_where) + ")");
        return 0;
    };
    // ---- meta.bin: size, then inflate + the primary frames' sizes
    Scratch scratch0;
    if (scratch0.alloc(index_scratch_stride(), s)) return fail(BYDB_ENOMEM, "device allocation failed (index scratch)");
    ip.scratch = scratch0.base;
    launch_index_meta(ip, 0, s);
    int rc = read_ctl();
    if (rc) return rc;
    const size_t n_primary = static_cast<size_t>(ctl.meta_raw / 40);
    Scratch meta_raw, pbs;
    if (meta_raw.alloc(ctl.meta_raw, s) || pbs.alloc(n_primary * sizeof(IndexPrimary), s)) return fail(BYDB_ENOMEM, "device allocation failed (index)");
    CUDA_TRY(cudaMemsetAsync(pbs.base, 0, n_primary ? n_primary * sizeof(IndexPrimary) : 256, s));
    ip.meta_raw = meta_raw.base;
    ip.meta_raw_cap = ctl.meta_raw;
    ip.pb = reinterpret_cast<IndexPrimary *>(pbs.base);
    launch_index_meta(ip, 1, s);
    rc = read_ctl();
    if (rc) return rc;
    // ---- primary blocks: inflate, count
    ip.n_primary = static_cast<uint32_t>(n_primary);
    Scratch raw, scratch;
    if (raw.alloc(ctl.raw_total + 256, s) || scratch.alloc(std::max<size_t>(1, n_primary) * index_scratch_stride(), s))
        return fail(BYDB_ENOMEM, "device allocation failed (inflated index)");
    ip.raw = raw.base;
    ip.scratch = scratch.base;
    launch_index_inflate(ip, s);
    launch_index_walk(ip, false, s);
    std::vector<IndexPrimary> hpb(n_primary);
    std::vector<IndexName> hnames(kIndexMaxNames);
    if (n_primary) CUDA_TRY(cudaMemcpyAsync(hpb.data(), pbs.base, n_primary * sizeof(IndexPrimary), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(hnames.data(), in.base + off_names, kIndexMaxNames * sizeof(IndexName), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaMemcpyAsync(&ctl, in.base + off_ctl, sizeof ctl, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    if (ctl.err == kIdxNames) return build_part_dir_host_for_device(ctx, imgs, part, s, n_files, dir_bytes_out);
    rc = read_ctl();
    if (rc) return rc;
    uint64_t nb = 0, nc = 0;
    for (auto &e : hpb) {
        e.block_base = nb;
        e.col_base = nc;
        nb += e.n_blocks;
        nc += e.n_cols;
    }
    if (nb > 0x7fffffffull || nc > 0xffffffffull) return fail(BYDB_EINVAL, "too many blocks / columns");
    // ---- the interned names -> the context's ids (a few dozen short strings: the only index bytes the host looks at)
    std::vector<uint16_t> map(kIndexMaxNames, 0);
    for (uint32_t i = 0; i < ctl.n_names && i < kIndexMaxNames; ++i) {
        const IndexName &e = hnames[i];
        std::string key = e.kind == 'f' ? "f:" : "t:" + families[e.fam] + "/";
        key.append(reinterpret_cast<const char *>(e.bytes), e.len);
        map[i] = ctx->names.intern(key);
    }
    if (n_primary) CUDA_TRY(cudaMemcpyAsync(pbs.base, hpb.data(), n_primary * sizeof(IndexPrimary), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemcpyAsync(in.base + off_map, map.data(), kIndexMaxNames * sizeof(uint16_t), cudaMemcpyHostToDevice, s));
    // ---- the part's device directory, filled by the second walk
    rc = alloc_part_dir(ctx, part, nb, nc, n_files, s, dir_bytes_out);
    if (rc) return rc;
    ip.blocks = const_cast<DevBlock *>(part.d_blocks);
    ip.cols = const_cast<DevCol *>(part.d_cols);
    ip.n_blocks = nb;
    launch_index_walk(ip, true, s);
    launch_index_order(ip, s);
    part.dir.blocks.resize(nb);
    part.dir.cols.resize(nc);
    if (nb) CUDA_TRY(cudaMemcpyAsync(part.dir.blocks.data(), ip.blocks, nb * sizeof(DevBlock), cudaMemcpyDeviceToHost, s));
    if (nc) CUDA_TRY(cudaMemcpyAsync(part.dir.cols.data(), ip.cols, nc * sizeof(DevCol), cudaMemcpyDeviceToHost, s));
    rc = read_ctl();
    if (rc) return rc;
    part.dir.total_rows = ctl.total_rows;
    part.dir.max_block_rows = ctl.max_block_rows;
    part.dir.min_ts = nb ? ctl.min_ts : 0;
    part.dir.max_ts = nb ? ctl.max_ts : 0;
    return 0;
}

// Rewrites the part's fallback pages (EncodeTypePlain numeric pages, zstd-compressed string blocks) into a side
// arena in HBM so the scan kernels never meet zstd or per-cell byte strings; see unpack_kernels.cu.
int unpack_fallback_pages(bydb_ctx *ctx, Part &part, size_t n_files, cudaStream_t s) {
    const size_t nb = part.dir.blocks.size(), nc = part.dir.cols.size();
    if (nb == 0 || nc == 0) return 0;
    if (n_files >= 255) return 0;
    Scratch jobs, scratch;
    const size_t jobs_off = 256;
    CUDA_TRY(jobs.alloc(jobs_off + nc * sizeof(UnpackJob), s));
    CUDA_TRY(cudaMemsetAsync(jobs.base, 0, jobs_off, s));
    UnpackParams up{};
    up.blocks = part.d_blocks;
    up.cols = const_cast<DevCol *>(part.d_cols);
    up.files = part.d_files;
    up.n_blocks = static_cast<uint32_t>(nb);
    up.arena_file_id = static_cast<uint32_t>(n_files);
    up.counters = reinterpret_cast<unsigned long long *>(jobs.base);
    up.jobs = reinterpret_cast<UnpackJob *>(jobs.base + jobs_off);
    up.max_jobs = nc;
    launch_classify_pages(up, s);
    unsigned long long cnt[5] = {0, 0, 0, 0, 0};
    CUDA_TRY(cudaMemcpyAsync(cnt, jobs.base, sizeof cnt, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    part.unpack_skipped = cnt[3];
    if (cnt[0] == 0) return 0;
    const size_t arena = align_up(cnt[1] + 256, 256);
    if (int rc = hbm_reserve(ctx, arena, "HBM budget exceeded while unpacking fallback pages")) return rc;
    part.hbm_bytes += arena;
    cudaError_t e = part.pool_stream ? cudaMallocAsync(reinterpret_cast<void **>(&part.d_unpack), arena, s)
                                     : cudaMalloc(reinterpret_cast<void **>(&part.d_unpack), arena);
    if (e != cudaSuccess) return fail(BYDB_ENOMEM, "device allocation failed for the unpack arena");
    const int n_warps = static_cast<int>(std::min<unsigned long long>(cnt[0], 8ull * static_cast<unsigned long long>(ctx->sm_count)));
    const int n_warps4 = (n_warps + 3) / 4 * 4;
    CUDA_TRY(scratch.alloc(static_cast<size_t>(n_warps4) * unpack_scratch_stride(), s));
    // publish the arena as one more file of the part
    const uint8_t *ap = part.d_unpack;
    CUDA_TRY(cudaMemcpyAsync(const_cast<uint8_t **>(reinterpret_cast<const uint8_t *const *>(part.d_files)) + n_files, &ap, sizeof ap,
                             cudaMemcpyHostToDevice, s));
    up.n_jobs = cnt[0];
    up.arena = part.d_unpack;
    up.scratch = scratch.base;
    launch_unpack_pages(up, n_warps4, s);
    CUDA_TRY(cudaMemcpyAsync(cnt, jobs.base, sizeof cnt, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    part.unpacked_pages = cnt[4];
    part.unpack_skipped = cnt[3];
    return 0;
}

// staging of one step, in pinned memory and on the device alike: series ids | order (query-series indices sorted by
// (group, series)) | group_start (where each group begins in order), back to back so that one copy takes all three
struct StageLayout {
    size_t NS, G, off_order, off_gstart, bytes, stride;
};
StageLayout stage_layout(size_t NS, size_t G) {
    const size_t bytes = NS * 12 + (G + 1) * 4;
    return StageLayout{NS, G, NS * 8, NS * 12, bytes, align_up(bytes, 256)};
}

void stage_series(const bydb_query *q, const StageLayout &st, uint8_t *h) {
    int32_t *order = reinterpret_cast<int32_t *>(h + st.off_order), *gstart = reinterpret_cast<int32_t *>(h + st.off_gstart);
    if (st.NS) memcpy(h, q->series_ids, st.NS * 8);
    std::fill(gstart, gstart + st.G + 1, 0);
    if (q->series_group) {
        for (size_t i = 0; i < st.NS; ++i) gstart[static_cast<size_t>(q->series_group[i]) + 1]++;
        for (size_t g = 0; g < st.G; ++g) gstart[g + 1] += gstart[g];
        std::vector<int32_t> cur(gstart, gstart + st.G);
        for (size_t i = 0; i < st.NS; ++i) order[cur[q->series_group[i]]++] = static_cast<int32_t>(i);
    } else {
        for (size_t i = 0; i < st.NS; ++i) order[i] = static_cast<int32_t>(i);
        gstart[1] = static_cast<int32_t>(st.NS);
    }
}

// device scratch of the finalisation and row selection; [o_out, o_out + out_bytes) is read back: selected-row count and the
// table's status word (o_cnt) | is_float | the selected rows
struct FinalLayout {
    size_t o_vi, o_vf, o_keys, o_kst, o_out, o_cnt, o_isf, o_sg, o_sr, o_si, o_sf, out_bytes, total, cap, A;
};
FinalLayout final_layout(size_t G, size_t A, int32_t top_n) {
    FinalLayout fl;
    Carve carve;
    fl.cap = top_n > 0 ? std::min<size_t>(static_cast<size_t>(top_n), G) : G;
    fl.A = A;
    fl.o_vi = carve(G * A * 8);
    fl.o_vf = carve(G * A * 8);
    fl.o_keys = carve(G * 8);
    fl.o_kst = carve(G);
    fl.o_out = carve.o;
    fl.o_cnt = carve(16);
    fl.o_isf = carve(A);
    fl.o_sg = carve(fl.cap * 4);
    fl.o_sr = carve(fl.cap * 8);
    fl.o_si = carve(fl.cap * A * 8);
    fl.o_sf = carve(fl.cap * A * 8);
    fl.out_bytes = carve.o - fl.o_out;
    fl.total = carve.o;
    return fl;
}

// pinned bytes of a step over G series groups whose finalisation sees out_groups groups: run_scan's staging of each batch, then
// the read-back of the results.  A prepared graph keeps the two apart (its results land at host_off = the staging's stride).
size_t step_pinned_bytes(const bydb_query *q, size_t G, size_t out_groups, size_t batches = 1) {
    return stage_layout(q->n_series, G).stride * batches + final_layout(out_groups, q->n_aggs, q->top_n).out_bytes;
}

// the partial-table pointers of ReduceParams / FinalizeParams (the names and order of TablePtrs)
template <class P>
void set_table(P &p, const TablePtrs &t) {
    p.sum_f64 = t.sum_f64;
    p.max_f64 = t.max_f64;
    p.negmin_f64 = t.negmin_f64;
    p.sum_i64 = t.sum_i64;
    p.cnt = t.cnt;
    p.rows = t.rows;
    p.max_i64 = t.max_i64;
    p.notmin_i64 = t.notmin_i64;
    p.coltype = t.coltype;
}

// the parts of a query as the kernels see them: blocks numbered globally in part order
void part_refs(const std::vector<std::shared_ptr<Part>> &parts, DevPartRef *out) {
    uint32_t base = 0;
    for (size_t i = 0; i < parts.size(); ++i) {
        const Part &p = *parts[i];
        out[i] = DevPartRef{p.d_blocks, p.d_cols, p.d_files, static_cast<uint32_t>(p.dir.blocks.size()), base};
        base += out[i].n_blocks;
    }
}

// two parts hold rows of one time span inside [tmin, tmax]: the scan then runs the version dedup, whose precheck synchronises
bool parts_overlap(const std::vector<std::shared_ptr<Part>> &parts, int64_t tmin, int64_t tmax) {
    for (size_t a = 0; a < parts.size(); ++a)
        for (size_t b = a + 1; b < parts.size(); ++b) {
            const PartDir &x = parts[a]->dir, &y = parts[b]->dir;
            if (x.blocks.empty() || y.blocks.empty()) continue;
            if (std::max(std::max(x.min_ts, y.min_ts), tmin) <= std::min(std::min(x.max_ts, y.max_ts), tmax)) return true;
        }
    return false;
}

// Runs plan -> scan -> series_reduce -> group_reduce on `stream`, leaving the partial table at
// `d_table` (device).  Synchronises the stream.  Fills stats.
// one pass of a group-key query (bydb_scan_agg_keyed): where in the composite table the pass writes, and its side outputs
struct KeyedPass {
    size_t group_off;   // first group row of this pass's slice
    int64_t *coltype;   // [F] the pass's own column types + status (merged by permute_table)
    int64_t *kts;       // [n_series] see ReduceParams::Kts
    uint32_t *krow;     // [n_series]
    int64_t *span;      // [2 * n_series] see ReduceParams::span, or NULL
};

int run_scan(bydb_ctx *ctx, const bydb_query *q, Plan &plan, ExecSlot &slot, cudaStream_t stream, uint8_t *d_table, const TableLayout &tl,
             bydb_stats *stats, int batch = 0, const KeyedPass *kp = nullptr) {
    cudaEvent_t *ev = slot.ev + 4 * batch;
    ZeroPage *hz = slot.page(batch);
    memset(hz, 0, kZeroPageBytes);  // a failure before the read-back is enqueued must not leave a previous call's status behind
    const size_t F = plan.fcols.size();
    const size_t NS = q->n_series;
    const size_t NB = plan.total_blocks;
    const int32_t G = plan.n_groups;
    // ---- host staging: sids | order | group_start
    const StageLayout st = stage_layout(NS, static_cast<size_t>(G));
    if (slot.ensure_pinned(st.stride * static_cast<size_t>(batch + 1))) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
    uint8_t *h = slot.pinned + st.stride * static_cast<size_t>(batch);
    stage_series(q, st, h);
    // ---- device scratch layout
    Carve carve;
    const size_t off_zero = carve(kZeroPageBytes);
    const size_t off_sids = carve(st.bytes);  // the staging as it is: one copy brings sids, order and group_start
    const size_t off_worklist = carve(NB * 4);
    const size_t off_slowlist = carve(NB * 4);
    const size_t off_restlist = carve(NB * 4);
    const size_t off_qsid = carve(NB * 4);
    const size_t off_P = carve(NB * F * sizeof(BlockPartial));
    const size_t off_Prows = carve(NB * 4);
    const size_t off_Pfirst = carve(kp ? NB * 4 : 0);
    const size_t off_S = carve(NS * F * sizeof(BlockPartial));
    const size_t off_Srows = carve(NS * 8);
    const size_t n_first = NS * plan.parts.size();
    const bool use_first = n_first > 0 && n_first <= (16u << 20);
    const size_t off_first = carve(use_first ? n_first * 4 : 0);
    const size_t off_dd_index = carve(NB * 4), off_dd_rowoff = carve(NB * 8), off_dd_list = carve(NB * 4);
    Scratch sc;
    CUDA_TRY(sc.alloc(carve.o, stream));
    uint8_t *d = sc.base;
    ZeroPage *z = reinterpret_cast<ZeroPage *>(d + off_zero);
    CUDA_TRY(cudaMemsetAsync(z, 0, kZeroPageBytes, stream));
    if (use_first) CUDA_TRY(cudaMemsetAsync(d + off_first, 0xff, n_first * 4, stream));
    CUDA_TRY(cudaMemcpyAsync(d + off_sids, h, st.bytes, cudaMemcpyHostToDevice, stream));
    if (stats) stats->h2d_bytes += st.bytes;

    ScanParams sp;
    memset(&sp, 0, sizeof sp);
    ReduceParams rp;
    memset(&rp, 0, sizeof rp);
    part_refs(plan.parts, sp.parts);
    std::copy(sp.parts, sp.parts + plan.parts.size(), rp.parts);
    sp.n_parts = rp.n_parts = static_cast<uint32_t>(plan.parts.size());
    sp.total_blocks = static_cast<uint32_t>(NB);
    sp.q_sids = reinterpret_cast<const uint64_t *>(d + off_sids);
    sp.n_series = static_cast<uint32_t>(NS);
    sp.n_fcols = static_cast<uint32_t>(F);
    sp.n_preds = q->n_preds;
    sp.tmin = q->tmin;
    sp.tmax = q->tmax;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        for (size_t c = 0; c < F; ++c) sp.fcol_name[c] = ctx->names.find("f:" + plan.fcols[c]);
        for (uint32_t a = 0; a < q->n_aggs; ++a) {
            const int fn = q->aggs[a].func;
            uint8_t need = (fn == BYDB_AGG_SUM || fn == BYDB_AGG_MEAN) ? 1 : (fn == BYDB_AGG_MIN || fn == BYDB_AGG_MAX) ? 2 : 0;
            sp.fcol_need[plan.agg_fcol[a]] |= need;
        }
        for (uint32_t i = 0; i < q->n_preds; ++i) {
            const bydb_pred &p = q->preds[i];
            DevPred &dp = sp.preds[i];
            dp.name_id = ctx->names.find(std::string("t:") + p.family + "/" + p.tag);
            dp.op = static_cast<uint8_t>(p.op);
            dp.value_type = static_cast<uint8_t>(p.value_type == BYDB_VT_BINARY ? BYDB_VT_STR : p.value_type);
            dp.lit_i64 = p.lit_i64;
            dp.lit_len = p.value_type == BYDB_VT_INT64 ? 0 : static_cast<uint32_t>(p.lit_len);
            if (dp.lit_len) memcpy(dp.lit, p.lit, dp.lit_len);
        }
    }
    sp.worklist = reinterpret_cast<uint32_t *>(d + off_worklist);
    sp.work_count = &z->work_count;
    sp.work_next = &z->work_next;
    sp.slow_list = reinterpret_cast<uint32_t *>(d + off_slowlist);
    sp.slow_count = &z->slow_count;
    sp.slow_next = &z->slow_next;
    sp.err = z->err;
    sp.stats = z->stats;
    sp.col_type = z->col_type;
    sp.block_qsid = reinterpret_cast<int32_t *>(d + off_qsid);
    sp.first_block = use_first ? reinterpret_cast<uint32_t *>(d + off_first) : nullptr;
    sp.P = reinterpret_cast<BlockPartial *>(d + off_P);
    sp.Prows = reinterpret_cast<uint32_t *>(d + off_Prows);
    sp.Pfirst = kp ? reinterpret_cast<uint32_t *>(d + off_Pfirst) : nullptr;

    rp.n_series = static_cast<uint32_t>(NS);
    rp.n_fcols = static_cast<uint32_t>(F);
    rp.n_groups = G;
    rp.q_sids = sp.q_sids;
    rp.order = reinterpret_cast<const int32_t *>(d + off_sids + st.off_order);
    rp.group_start = reinterpret_cast<const int32_t *>(d + off_sids + st.off_gstart);
    rp.block_qsid = sp.block_qsid;
    rp.first_block = sp.first_block;
    rp.P = sp.P;
    rp.Prows = sp.Prows;
    rp.col_type = sp.col_type;
    rp.S = reinterpret_cast<BlockPartial *>(d + off_S);
    rp.Srows = reinterpret_cast<int64_t *>(d + off_Srows);
    rp.err = sp.err;
    TablePtrs table = tl.at(d_table, kp ? kp->group_off : 0);
    if (kp) {
        table.coltype = kp->coltype;
        rp.Pfirst = sp.Pfirst;
        rp.Kts = kp->kts;
        rp.Krow = kp->krow;
        rp.span = kp->span;
    }
    set_table(rp, table);

    CUDA_TRY(cudaEventRecord(ev[0], stream));
    launch_plan_blocks(sp, stream);
    // ---- version dedup: only when two parts of the query overlap in time at all (host-side precheck on
    //      the part directories); then the device finds the series that really overlap
    Scratch dd_scratch;
    uint32_t extra_launches = 0;
    const bool overlap = parts_overlap(plan.parts, q->tmin, q->tmax);
    if (overlap && NB > 0 && NS > 0) {
        sp.dd_index = reinterpret_cast<int32_t *>(d + off_dd_index);
        sp.dd_row_off = reinterpret_cast<unsigned long long *>(d + off_dd_rowoff);
        sp.dd_list = reinterpret_cast<uint32_t *>(d + off_dd_list);
        sp.dd_counts = z->dd_counts;
        CUDA_TRY(cudaMemsetAsync(sp.dd_index, 0xff, NB * 4, stream));
        launch_detect_overlap(sp, stream);
        CUDA_TRY(cudaMemcpyAsync(hz->dd_counts, z->dd_counts, sizeof hz->dd_counts, cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        const unsigned long long n_ddb = hz->dd_counts[0], n_ddr = hz->dd_counts[1];
        extra_launches += 1;
        if (stats) stats->d2h_bytes += sizeof hz->dd_counts;
        if (n_ddb > 0) {
            const size_t b_ts = align_up(n_ddr * 8, 256), b_sh = align_up(n_ddb * kMaskWords * 4, 256);
            CUDA_TRY(dd_scratch.alloc(2 * b_ts + b_sh, stream));
            sp.dd_ts = reinterpret_cast<int64_t *>(dd_scratch.base);
            sp.dd_ver = reinterpret_cast<int64_t *>(dd_scratch.base + b_ts);
            sp.dd_shadow = reinterpret_cast<uint32_t *>(dd_scratch.base + 2 * b_ts);
            sp.n_dd_blocks = static_cast<uint32_t>(n_ddb);
            launch_dedup(sp, ctx->sm_count * ctx->ctas_per_sm, stream);
            extra_launches += 2;
        }
        rp.dedup_done = 1;
    }
    {
        // express lane (scan_sum_express_kernel): all-rows SUM / MEAN / COUNT without row predicates or version dedup -- the
        // group-by-sum shape; every block it cannot take (time-range cut, non-delta page, ...) goes on to the regular lane
        bool sums_only = q->n_preds == 0 && !overlap && NB > 0;
        for (size_t c = 0; c < F; ++c) sums_only = sums_only && (sp.fcol_need[c] & 2) == 0;
        slot.express[batch] = sums_only;
        if (sums_only) {
            sp.rest_list = reinterpret_cast<uint32_t *>(d + off_restlist);
            sp.rest_count = &z->rest_count;
            sp.rest_next = &z->rest_next;
            if (stats) stats->kernel_launches += 1;
        }
    }
    CUDA_TRY(cudaEventRecord(ev[1], stream));
    launch_scan_blocks(sp, ctx->sm_count * ctx->ctas_per_sm_express, ctx->sm_count * ctx->ctas_per_sm_fast, ctx->sm_count * ctx->ctas_per_sm, stream);
    CUDA_TRY(cudaEventRecord(ev[2], stream));
    launch_series_reduce(rp, stream);
    const int32_t *gstart = reinterpret_cast<const int32_t *>(h + st.off_gstart);
    bool small_groups = true;  // every group has at most 32 series: the warp-per-group reduce (bit-identical sums)
    for (int32_t g = 0; g < G && small_groups; ++g) small_groups = gstart[g + 1] - gstart[g] <= 32;
    launch_group_reduce(rp, stream, small_groups);
    CUDA_TRY(cudaEventRecord(ev[3], stream));
    // read back the zero page (errors + counters); the caller synchronises and then calls collect_scan
    CUDA_TRY(cudaMemcpyAsync(hz, z, kZeroPageBytes, cudaMemcpyDeviceToHost, stream));
    if (stats) {
        stats->kernel_launches += (NB ? 1u : 0u) + 2u + (NS ? 1u : 0u) + 1u + extra_launches;
        stats->d2h_bytes += kZeroPageBytes;
    }
    // the scratch must outlive the kernels: it is freed stream-ordered (after them) when `sc` goes out of scope
    return 0;
}

// a read-back zero page: its counters into `stats` (when given) and its device error as the result.  `express`: the step
// launched the express lane, which takes the whole work list and hands on to the regular lane what it cannot finish.
int read_zero_page(const ZeroPage &z, bool express, bydb_stats *stats) {
    if (stats) {
        stats->rows_scanned += z.stats[0];
        stats->rows_matched += z.stats[1];
        stats->page_bytes += z.stats[2];
        stats->blocks_scanned += z.stats[3];
        stats->blocks_slow_lane += static_cast<uint32_t>(z.stats[4]);
        stats->slow_lane_reasons |= static_cast<uint32_t>(z.stats[5]);
        stats->blocks_express_lane += express ? z.work_count - z.rest_count : 0u;
    }
    if (z.err[0] == 0) return 0;
    g_last_dev_err = z.err[0];  // reset by the API entry points; a later clean slice must not hide it
    char buf[96];
    snprintf(buf, sizeof buf, " (block/series #%u)", z.err[1]);
    return fail(dev_err_code(z.err[0]), std::string(dev_err_text(z.err[0])) + buf);
}

// after the stream is synchronised: device errors + counters of the scan
int collect_scan(ExecSlot &slot, bydb_stats *stats, int batch = 0) {
    if (stats) {
        cudaEvent_t *ev = slot.ev + 4 * batch;
        float ms = 0;
        cudaEventElapsedTime(&ms, ev[1], ev[2]);
        stats->scan_kernel_ms += ms;
        cudaEventElapsedTime(&ms, ev[0], ev[3]);
        stats->device_ms += ms;
    }
    return read_zero_page(*slot.page(batch), slot.express[batch], stats);
}

// the status a partial table carries in its coltype words (DevErr, 0 = none): tables of bydb_scan_partials and the peers'
// mailbox slots, possibly another rank's
int table_status(uint32_t e) {
    if (e == 0) return 0;
    g_last_dev_err = e;
    return fail(dev_err_code(e), std::string(dev_err_text(e)) + " (status carried in a partial table)");
}

// finalisation + row selection of the table at d_table, up to and including the read-back copy to slot.pinned + host_off;
// fl = final_layout() of the query, launches = kernels launched
int finalize_enqueue(const bydb_query *q, const Plan &plan, ExecSlot &slot, cudaStream_t stream, const uint8_t *d_table, const TableLayout &tl,
                     size_t host_off, Scratch &sc, FinalLayout &fl, uint32_t &launches) {
    const size_t F = plan.fcols.size();
    const int32_t G = plan.n_groups;
    const size_t A = q->n_aggs;
    fl = final_layout(static_cast<size_t>(G), A, q->top_n);
    CUDA_TRY(sc.alloc(fl.total, stream));
    uint8_t *d = sc.base;
    FinalizeParams fp;
    memset(&fp, 0, sizeof fp);
    fp.n_groups = G;
    fp.n_fcols = static_cast<uint32_t>(F);
    fp.n_aggs = static_cast<uint32_t>(A);
    fp.row_path_types = (q->flags & BYDB_Q_ROW_PATH_TYPES) ? 1u : 0u;
    for (size_t a = 0; a < A; ++a) {
        fp.agg_fcol[a] = plan.agg_fcol[a];
        fp.agg_func[a] = q->aggs[a].func;
    }
    set_table(fp, tl.at(const_cast<uint8_t *>(d_table)));  // read only
    fp.out_i64 = reinterpret_cast<int64_t *>(d + fl.o_vi);
    fp.out_f64 = reinterpret_cast<double *>(d + fl.o_vf);
    fp.out_is_float = d + fl.o_isf;
    fp.err_out = reinterpret_cast<uint32_t *>(d + fl.o_cnt + 8);
    SelectParams sp;
    memset(&sp, 0, sizeof sp);
    sp.n_groups = G;
    sp.n_fcols = static_cast<uint32_t>(F);
    sp.n_aggs = static_cast<uint32_t>(A);
    sp.top_n = q->top_n;
    sp.top_agg = q->top_n > 0 ? q->top_agg : 0;
    sp.top_desc = q->top_desc;
    sp.top_fcol = plan.agg_fcol[sp.top_agg];
    sp.top_is_count = q->aggs[sp.top_agg].func == BYDB_AGG_COUNT;
    sp.rows = fp.rows;
    sp.cnt = fp.cnt;
    sp.max_i64 = fp.max_i64;
    sp.max_f64 = fp.max_f64;
    sp.val_i64 = fp.out_i64;
    sp.val_f64 = fp.out_f64;
    sp.is_float = fp.out_is_float;
    sp.keys = reinterpret_cast<uint64_t *>(d + fl.o_keys);
    sp.kstate = d + fl.o_kst;
    sp.sel_count = reinterpret_cast<uint32_t *>(d + fl.o_cnt);
    sp.sel_group = reinterpret_cast<int32_t *>(d + fl.o_sg);
    sp.sel_rows = reinterpret_cast<int64_t *>(d + fl.o_sr);
    sp.sel_i64 = reinterpret_cast<int64_t *>(d + fl.o_si);
    sp.sel_f64 = reinterpret_cast<double *>(d + fl.o_sf);
    launches = launch_finalize_select(fp, sp, stream);
    if (slot.ensure_pinned(host_off + fl.out_bytes)) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
    CUDA_TRY(cudaMemcpyAsync(slot.pinned + host_off, d + fl.o_out, fl.out_bytes, cudaMemcpyDeviceToHost, stream));
    return 0;
}

// the read-back at h into *out; carried_status: the table came from bydb_scan_partials or a mailbox slot, so the status it
// carries is the outcome
int finalize_parse(const uint8_t *h, const FinalLayout &fl, bool carried_status, bydb_result *out) {
    if (carried_status) {
        const int rc = table_status(*reinterpret_cast<const uint32_t *>(h + (fl.o_cnt - fl.o_out) + 8));
        if (rc) return rc;
    }
    const size_t A = fl.A;
    const size_t R = std::min<size_t>(*reinterpret_cast<const uint32_t *>(h + (fl.o_cnt - fl.o_out)), fl.cap);
    auto owner = new ResultOwner();
    const int32_t *sg = reinterpret_cast<const int32_t *>(h + (fl.o_sg - fl.o_out));
    const int64_t *sr = reinterpret_cast<const int64_t *>(h + (fl.o_sr - fl.o_out));
    const int64_t *si = reinterpret_cast<const int64_t *>(h + (fl.o_si - fl.o_out));
    const double *sf = reinterpret_cast<const double *>(h + (fl.o_sf - fl.o_out));
    owner->group_id.assign(sg, sg + R);
    owner->rows.assign(sr, sr + R);
    owner->is_float.assign(h + (fl.o_isf - fl.o_out), h + (fl.o_isf - fl.o_out) + A);
    owner->val_i64.assign(si, si + R * A);
    owner->val_f64.assign(sf, sf + R * A);
    out->n_rows = static_cast<int32_t>(R);
    out->n_aggs = static_cast<int32_t>(A);
    out->group_id = owner->group_id.data();
    out->rows = owner->rows.data();
    out->is_float = owner->is_float.data();
    out->val_i64 = owner->val_i64.data();
    out->val_f64 = owner->val_f64.data();
    out->owner = owner;
    return 0;
}


// finalisation + row selection + read-back of the result rows, synchronised and parsed
int finalize_to_host(const bydb_query *q, const Plan &plan, ExecSlot &slot, cudaStream_t stream, const uint8_t *d_table, const TableLayout &tl,
                     bydb_result *out, bool carried_status = false) {
    FinalLayout fl;
    uint32_t launches = 0;
    Scratch sc;
    int rc = finalize_enqueue(q, plan, slot, stream, d_table, tl, 0, sc, fl, launches);
    if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(stream));
    CUDA_TRY(cudaGetLastError());
    out->stats.d2h_bytes += fl.out_bytes;
    out->stats.kernel_launches += launches;
    return finalize_parse(slot.pinned, fl, carried_status, out);
}
int make_plan(bydb_ctx *ctx, const bydb_query *q, const std::vector<std::shared_ptr<Part>> *given, Plan &plan) {
    if (given) {
        plan.parts = *given;
    } else {
        std::lock_guard<std::mutex> lk(ctx->mu);
        for (uint32_t i = 0; i < q->n_parts; ++i) {
            auto it = ctx->parts.find(q->parts[i]);
            if (it == ctx->parts.end()) return fail(BYDB_ENOENT, "unknown part handle");
            plan.parts.push_back(it->second);
        }
    }
    if (int rc = query_shape(q, plan)) return rc;
    uint64_t nb = 0;
    for (auto &p : plan.parts) nb += p->dir.blocks.size();
    if (nb > 0x7fffffffull) return fail(BYDB_EINVAL, "too many blocks");
    plan.total_blocks = static_cast<uint32_t>(nb);
    return 0;
}

int scan_agg_impl(bydb_ctx *ctx, const bydb_query *q, const std::vector<std::shared_ptr<Part>> *given, bydb_result *out, uint64_t h2d_pre) {
    Plan plan;
    int rc = make_plan(ctx, q, given, plan);
    if (rc) return rc;
    CUDA_TRY(cudaSetDevice(ctx->device));
    SlotLease lease(ctx);
    if (lease.init()) return fail(BYDB_EIO, "cannot create stream");
    ExecSlot &slot = *lease.slot;
    const TableLayout &tl = plan.tl;
    Scratch table;
    CUDA_TRY(table.alloc(tl.total, slot.stream));
    memset(&out->stats, 0, sizeof out->stats);
    out->stats.h2d_bytes = h2d_pre;
    // size the pinned staging once: it must not be reallocated while copies from/to it are in flight
    if (slot.ensure_pinned(step_pinned_bytes(q, tl.G, tl.G))) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
    rc = run_scan(ctx, q, plan, slot, slot.stream, table.base, tl, &out->stats);
    // finalisation is enqueued behind the scan; one synchronisation covers both
    if (!rc) rc = finalize_to_host(q, plan, slot, slot.stream, table.base, tl, out);
    if (rc) {
        // a failure after something was enqueued: the slot (and, on the host path, the transient parts the kernels read)
        // go back to their pools when this returns, so nothing may still be in flight
        cudaStreamSynchronize(slot.stream);
        const std::string keep = g_last_error;
        (void)collect_scan(slot, nullptr);  // a device-side error of the scan, if any, still drives the lazy-unpack retry
        g_last_error = keep;
        bydb_result_free(ctx, out);
        return rc;
    }
    int rc2 = collect_scan(slot, &out->stats);
    if (rc2) {
        bydb_result_free(ctx, out);
        return rc2;
    }
    return rc;
}


// ------------------------------------------------------------------------------------------------
// Prepared queries: the whole step (staging copy, plan, scan, reduce, finalize, row selection, read-back) captured once
// into a CUDA graph and replayed.  A query executed many times (dashboards, alert rules) then costs one graph launch and
// one synchronisation instead of ~20 runtime calls.  Everything here is additive: bydb_scan_agg is untouched.
// ------------------------------------------------------------------------------------------------
}  // namespace

struct bydb_prepared {
    // deep copy of the query: the caller's arrays only live for the duration of bydb_query_prepare
    std::vector<bydb_part_h> parts;
    std::vector<uint64_t> sids;
    std::vector<int32_t> groups;
    std::vector<std::string> agg_names, pred_family, pred_tag;
    std::vector<std::vector<uint8_t>> pred_lit;
    std::vector<bydb_agg> aggs;
    std::vector<bydb_pred> preds;
    bydb_query q{};
    std::mutex mu;                     // one execution at a time per prepared query
    std::unique_ptr<ExecSlot> slot;    // dedicated stream + pinned staging: their addresses are baked into the graph
    cudaGraphExec_t exec = nullptr;
    cudaEvent_t t0 = nullptr, t1 = nullptr;
    FinalLayout fl;
    size_t host_off = 0;
    std::vector<std::shared_ptr<Part>> held;  // the parts whose device pointers are baked into the graph stay alive with it
    bydb_stats captured{};             // host-side counters of one step (launch counts, byte counts)
    bool express = false;              // the captured step launches the express lane
    uint64_t runs = 0;
    bool capturable = true;
    // the collective form (bydb_scan_reduce_prepared): one captured graph per (root, slot parity)
    struct ReduceGraph {
        cudaGraphExec_t exec = nullptr;
        FinalLayout fl;
        bydb_stats captured{};
        bool express = false;
        std::vector<std::shared_ptr<Part>> held;
    };
    std::unordered_map<int, ReduceGraph> reduce_graphs;  // key = root * 2 + parity
    uint64_t reduce_runs = 0;
    bool reduce_capturable = true;
};

namespace {

void prepared_destroy(bydb_prepared *p) {
    if (!p) return;
    if (p->exec) cudaGraphExecDestroy(p->exec);
    for (auto &kv : p->reduce_graphs)
        if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    if (p->t0) cudaEventDestroy(p->t0);
    if (p->t1) cudaEventDestroy(p->t1);
    delete p;  // and with it the slot
}

// A graph reads its parts through the device pointers captured with it, so it may only replay while every handle still names
// the very part object it captured (`held`).  Otherwise the graph is dropped, to be captured again; returns false when a handle
// names no part any more (a released part makes the call fail like the plain path would).
bool check_held_parts(bydb_ctx *ctx, const std::vector<bydb_part_h> &parts, cudaGraphExec_t &exec, std::vector<std::shared_ptr<Part>> &held) {
    std::lock_guard<std::mutex> lk(ctx->mu);
    bool same = held.size() == parts.size(), missing = false;
    for (size_t i = 0; i < parts.size(); ++i) {
        auto it = ctx->parts.find(parts[i]);
        if (it == ctx->parts.end()) missing = true;
        else if (same && it->second != held[i]) same = false;
    }
    if (missing || !same) {
        cudaGraphExecDestroy(exec);
        exec = nullptr;
        held.clear();
    }
    return !missing;
}

// One replay of a captured step on the slot's stream, synchronised: the step's host-side counters as captured, device_ms from
// the events around the launch, then the counters and the device error of its zero page (batch 0).
int replay_graph(cudaGraphExec_t exec, ExecSlot &slot, cudaEvent_t t0, cudaEvent_t t1, const bydb_stats &captured, bool express, bydb_stats *stats) {
    CUDA_TRY(cudaEventRecord(t0, slot.stream));
    CUDA_TRY(cudaGraphLaunch(exec, slot.stream));
    CUDA_TRY(cudaEventRecord(t1, slot.stream));
    CUDA_TRY(cudaStreamSynchronize(slot.stream));
    CUDA_TRY(cudaGetLastError());
    *stats = captured;  // the zero-page counters are still 0 there
    float ms = 0;
    cudaEventElapsedTime(&ms, t0, t1);
    stats->device_ms = ms;
    stats->scan_kernel_ms = 0;  // per-kernel events are not available inside a graph replay
    return read_zero_page(*slot.page(0), express, stats);
}

// captures one step into p->exec; returns 0, or a code after leaving the stream out of capture mode
int prepared_capture(bydb_ctx *ctx, bydb_prepared *p) {
    Plan plan;
    int rc = make_plan(ctx, &p->q, nullptr, plan);
    if (rc) return rc;
    // the version-dedup precheck of run_scan synchronises: parts that overlap in time keep the uncaptured path
    if (parts_overlap(plan.parts, p->q.tmin, p->q.tmax)) {
        p->capturable = false;
        return 0;
    }
    ExecSlot &slot = *p->slot;
    const TableLayout &tl = plan.tl;
    p->host_off = stage_layout(p->q.n_series, tl.G).stride;  // results land behind the staging area, which must survive from replay to replay
    if (slot.ensure_pinned(step_pinned_bytes(&p->q, tl.G, tl.G))) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
    memset(&p->captured, 0, sizeof p->captured);
    cudaError_t e = cudaStreamBeginCapture(slot.stream, cudaStreamCaptureModeThreadLocal);
    if (e != cudaSuccess) return fail(BYDB_EIO, std::string("cudaStreamBeginCapture: ") + cudaGetErrorString(e));
    uint32_t fin_launches = 0;
    {
        Scratch table, fin;
        rc = table.alloc(tl.total, slot.stream) == cudaSuccess ? 0 : fail(BYDB_ENOMEM, "cudaMallocAsync (capture)");
        if (!rc) rc = run_scan(ctx, &p->q, plan, slot, slot.stream, table.base, tl, &p->captured);
        p->express = slot.express[0];
        if (!rc) rc = finalize_enqueue(&p->q, plan, slot, slot.stream, table.base, tl, p->host_off, fin, p->fl, fin_launches);
        // table / fin are released here: inside the capture, i.e. as free nodes of the graph
    }
    cudaGraph_t graph = nullptr;
    e = cudaStreamEndCapture(slot.stream, &graph);
    if (rc || e != cudaSuccess || !graph) {
        if (graph) cudaGraphDestroy(graph);
        cudaGetLastError();
        p->capturable = false;  // fall back to the uncaptured path for good
        return rc ? rc : 0;
    }
    e = cudaGraphInstantiate(&p->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) {
        cudaGetLastError();
        p->exec = nullptr;
        p->capturable = false;
    }
    p->captured.kernel_launches += fin_launches;  // finalize + select_rows (one fused launch for few groups)
    p->captured.d2h_bytes += p->fl.out_bytes;
    p->held = plan.parts;
    return 0;
}

}  // namespace

// ================================================================================================
extern "C" {

const char *bydb_last_error(void) { return g_last_error.c_str(); }
const char *bydb_version(void) { return "bydb-b200 0.1 (sm_90a)"; }

int bydb_init(const bydb_cfg *cfg, bydb_ctx **out) {
    return guarded([&]() -> int {
    if (!out) return fail(BYDB_EINVAL, "out is NULL");
    *out = nullptr;
    int dev = cfg ? cfg->device : 0;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return fail(BYDB_EIO, "no CUDA device: libbydbgpu has no CPU fallback");
    if (dev < 0 || dev >= n) return fail(BYDB_EINVAL, "bad device ordinal");
    CUDA_TRY(cudaSetDevice(dev));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
    // sm_90a code (arch-specific: TMA bulk copies, mbarrier transaction counts) loads on compute capability 9.0 only
    if (prop.major != 9 || prop.minor != 0)
        return fail(BYDB_ENOTSUP, std::string("device '") + prop.name + "' is not sm_90 (Hopper); this library is built for sm_90a only");
    auto ctx = new bydb_ctx();
    ctx->device = dev;
    ctx->sm_count = prop.multiProcessorCount;
    ctx->hbm_budget = cfg ? cfg->hbm_budget_bytes : 0;
    ctx->host_index = cfg && (cfg->flags & BYDB_CFG_HOST_INDEX) != 0;
    if (upload_pow10_table()) {
        delete ctx;
        return fail(BYDB_EIO, "cannot upload constant tables (is the library built for this GPU?)");
    }
    {
        // keep freed stream-ordered allocations in the pool: every query allocates its scratch with
        // cudaMallocAsync, and the default threshold (0) would hand the memory back at each sync
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            uint64_t thr = UINT64_MAX;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
            // never let the allocator satisfy a request by making the requesting stream wait for ANOTHER stream's pending free:
            // with several ranks on one device that other stream may sit behind a wait kernel spinning for this very rank
            // (the collective then stalls until the 60 s bound; seen as a test that failed only after the pool had history)
            int no = 0;
            cudaMemPoolSetAttribute(pool, cudaMemPoolReuseAllowInternalDependencies, &no);
        }
    }
    // execution slots (stream, events, pinned staging) for the first concurrent callers: made now, not inside a query
    for (int i = 0; i < 2; ++i) {
        std::unique_ptr<ExecSlot> sl(new ExecSlot());
        if (sl->create() != 0) {
            cudaGetLastError();
            break;
        }
        ctx->free_slots.push_back(std::move(sl));
    }
    preload_kernels();
    preload_unpack_kernels();
    preload_index_kernels();
    preload_encode_kernels();
    int occ_express = 1, occ_fast = 1, occ_slow = 1;
    scan_max_ctas_per_sm(&occ_express, &occ_fast, &occ_slow);
    int want = (cfg && cfg->warps_per_sm > 0) ? (cfg->warps_per_sm + kWarpsPerCta - 1) / kWarpsPerCta : 64;
    ctx->ctas_per_sm = std::max(1, std::min(want, occ_slow));
    ctx->ctas_per_sm_fast = std::max(1, std::min(want, occ_fast));
    ctx->ctas_per_sm_express = std::max(1, std::min(want, occ_express));
    *out = ctx;
    return 0;
    });
}

void bydb_shutdown(bydb_ctx *ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();  // before any slot goes away: no copy may still read its pinned staging
    ctx->free_slots.clear();
    ctx->parts.clear();
    for (int i = 0; i < StageRing::kBufs; ++i) {
        if (ctx->stage.buf[i]) cudaFreeHost(ctx->stage.buf[i]);
        if (ctx->stage.done[i]) cudaEventDestroy(ctx->stage.done[i]);
    }
    for (size_t r = 0; r < ctx->comm.peer.size(); ++r)
        if (ctx->comm.ipc_opened[r] && ctx->comm.peer[r]) cudaIpcCloseMemHandle(ctx->comm.peer[r]);
    if (ctx->comm.mine) cudaFree(ctx->comm.mine);
    if (ctx->comm.poll_stream) cudaStreamDestroy(ctx->comm.poll_stream);
    if (ctx->comm.poll_buf) cudaFreeHost(ctx->comm.poll_buf);
    delete ctx;
}

int bydb_part_register(bydb_ctx *ctx, uint64_t part_id, const bydb_part_files *files, bydb_part_h *out) {
    return guarded([&]() -> int {
    if (!ctx || !out) return fail(BYDB_EINVAL, "ctx/out is NULL");
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        auto it = ctx->by_id.find(part_id);
        if (it != ctx->by_id.end()) {  // idempotent per part_id
            *out = it->second;
            return 0;
        }
    }
    CUDA_TRY(cudaSetDevice(ctx->device));
    std::shared_ptr<Part> part;
    AdmitOptions opt;
    opt.unpack = true;
    opt.device_index = !ctx->host_index;
    int rc = register_part_locked_free(ctx, part_id, files, part, nullptr, opt);
    if (rc) return rc;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        auto again = ctx->by_id.find(part_id);
        if (again == ctx->by_id.end()) {
            bydb_part_h h = ctx->next_handle++;
            ctx->parts[h] = part;
            ctx->by_id[part_id] = h;
            *out = h;
            return 0;
        }
        *out = again->second;
    }
    // another thread registered the same part meanwhile: keep its copy, drop ours (idempotent per part_id)
    hbm_release(ctx, part->hbm_bytes);
    return 0;
    });
}

int bydb_part_release(bydb_ctx *ctx, bydb_part_h h) {
    return guarded([&]() -> int {
    if (!ctx) return fail(BYDB_EINVAL, "ctx is NULL");
    std::shared_ptr<Part> victim;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        auto it = ctx->parts.find(h);
        if (it == ctx->parts.end()) return fail(BYDB_ENOENT, "unknown part handle");
        victim = it->second;
        ctx->by_id.erase(victim->id);
        ctx->parts.erase(it);
    }
    hbm_release(ctx, victim->hbm_bytes);
    cudaSetDevice(ctx->device);
    victim.reset();  // frees HBM once no in-flight query holds the part
    return 0;
    });
}

int bydb_part_info(bydb_ctx *ctx, bydb_part_h h, uint64_t *hbm_bytes, uint64_t *n_blocks, uint64_t *n_rows) {
    return guarded([&]() -> int {
    if (!ctx) return fail(BYDB_EINVAL, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->parts.find(h);
    if (it == ctx->parts.end()) return fail(BYDB_ENOENT, "unknown part handle");
    if (hbm_bytes) *hbm_bytes = it->second->hbm_bytes;
    if (n_blocks) *n_blocks = it->second->dir.blocks.size();
    if (n_rows) *n_rows = it->second->dir.total_rows;
    return 0;
    });
}

int bydb_part_fallback_pages(bydb_ctx *ctx, bydb_part_h h, uint64_t *unpacked, uint64_t *left) {
    return guarded([&]() -> int {
    if (!ctx) return fail(BYDB_EINVAL, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->parts.find(h);
    if (it == ctx->parts.end()) return fail(BYDB_ENOENT, "unknown part handle");
    if (unpacked) *unpacked = it->second->unpacked_pages;
    if (left) *left = it->second->unpack_skipped;
    return 0;
    });
}

int bydb_part_directory(bydb_ctx *ctx, bydb_part_h h, void *blocks_out, uint64_t blocks_cap_bytes, void *cols_out, uint64_t cols_cap_bytes, uint64_t *n_blocks,
                        uint64_t *n_cols) {
    return guarded([&]() -> int {
    if (!ctx) return fail(BYDB_EINVAL, "ctx is NULL");
    std::shared_ptr<Part> part;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        auto it = ctx->parts.find(h);
        if (it == ctx->parts.end()) return fail(BYDB_ENOENT, "unknown part handle");
        part = it->second;
    }
    const uint64_t nb = part->dir.blocks.size(), nc = part->dir.cols.size();
    if (n_blocks) *n_blocks = nb;
    if (n_cols) *n_cols = nc;
    CUDA_TRY(cudaSetDevice(ctx->device));
    if (blocks_out) {
        if (blocks_cap_bytes < nb * sizeof(DevBlock)) return fail(BYDB_EINVAL, "blocks buffer too small");
        if (nb) CUDA_TRY(cudaMemcpy(blocks_out, part->d_blocks, nb * sizeof(DevBlock), cudaMemcpyDeviceToHost));
    }
    if (cols_out) {
        if (cols_cap_bytes < nc * sizeof(DevCol)) return fail(BYDB_EINVAL, "cols buffer too small");
        if (nc) CUDA_TRY(cudaMemcpy(cols_out, part->d_cols, nc * sizeof(DevCol), cudaMemcpyDeviceToHost));
    }
    return 0;
    });
}

int bydb_scan_agg(bydb_ctx *ctx, const bydb_query *q, bydb_result *out) {
    return guarded([&]() -> int {
    if (!ctx || !out) return fail(BYDB_EINVAL, "ctx/out is NULL");
    memset(out, 0, sizeof *out);
    int rc = validate_query(q, true);
    if (rc) return rc;
    return scan_agg_impl(ctx, q, nullptr, out, 0);
    });
}


// ------------------------------------------------------------------------------------------------
// Gather path of the cold query (host images in pageable memory, e.g. BanyanDB's mmap'd part files): instead of copying
// every file of the part to HBM (12.8 GB for the 1e9 bench part), the host selects the blocks
// like plan_blocks does and collects ONLY the pages the query reads -- the timestamps page, the aggregated fields, the
// predicate tags -- into one arena image per slice: [DevBlock[] | DevCol[] | file table | pages], every page offset
// rewritten into the arena.  The image goes up through the pinned staging ring in 64 MB chunks.
// ------------------------------------------------------------------------------------------------

namespace {
struct KeyedOwner {
    std::vector<int32_t> key_id;
    std::vector<uint32_t> key_off;
    std::vector<uint8_t> key_bytes;
};
using KeyValues = std::vector<std::vector<uint8_t>>;

// the checks of a group key that need no device; cap = the distinct values accepted (max_values, 0 = 64)
int check_group_key(const bydb_query *q, const bydb_group_key *key, uint32_t &cap) {
    if (!key || !key->family || !key->tag) return fail(BYDB_EINVAL, "group key without family/tag");
    if (key->value_type != 0 && key->value_type != BYDB_VT_STR && key->value_type != BYDB_VT_BINARY && key->value_type != BYDB_VT_INT64)
        return fail(BYDB_EINVAL, "bydb_group_key.value_type must be 0, BYDB_VT_STR, BYDB_VT_BINARY or BYDB_VT_INT64");
    cap = key->max_values ? key->max_values : 64u;
    if (cap > kMaxKeyValues) return fail(BYDB_EINVAL, "bydb_group_key.max_values above 256");
    if (q->n_preds + 1 > kMaxPreds) return fail(BYDB_ENOTSUP, "a group-key query takes at most 7 predicates");
    return 0;
}

// 1. the distinct key values of the selected blocks, on the slot's stream, synchronised
int discover_keys(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, uint32_t cap, const Plan &plan, ExecSlot &slot, bydb_stats *stats,
                  KeyValues &values) {
    const bool int64_key = key->value_type == BYDB_VT_INT64;
    const size_t NS = q->n_series, NB = plan.total_blocks;
    cudaStream_t stream = slot.stream;
    Carve carve;
    const size_t a_sids = carve(NS * 8), a_slots = carve(kKeySlots * 8), a_ctl = carve(16), a_vals = carve(static_cast<size_t>(cap) * kMaxLit),
                 a_lens = carve(static_cast<size_t>(cap) * 4);
    const size_t a_total = carve.o;
    Scratch ka;
    CUDA_TRY(ka.alloc(a_total, stream));
    const size_t back_bytes = a_total - a_ctl;  // ctl | vals | lens come back in one copy
    if (slot.ensure_pinned(std::max(back_bytes, NS * 8) + 256)) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
    if (NS) memcpy(slot.pinned, q->series_ids, NS * 8);
    if (NS) CUDA_TRY(cudaMemcpyAsync(ka.base + a_sids, slot.pinned, NS * 8, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemsetAsync(ka.base + a_slots, 0, a_total - a_slots, stream));
    KeyParams kpar;
    memset(&kpar, 0, sizeof kpar);
    part_refs(plan.parts, kpar.parts);
    kpar.n_parts = static_cast<uint32_t>(plan.parts.size());
    kpar.total_blocks = static_cast<uint32_t>(NB);
    kpar.q_sids = reinterpret_cast<const uint64_t *>(ka.base + a_sids);
    kpar.n_series = static_cast<uint32_t>(NS);
    kpar.cap = cap;
    kpar.tmin = q->tmin;
    kpar.tmax = q->tmax;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        kpar.key_name = ctx->names.find(std::string("t:") + key->family + "/" + key->tag);
    }
    kpar.slots = reinterpret_cast<unsigned long long *>(ka.base + a_slots);
    kpar.count = reinterpret_cast<uint32_t *>(ka.base + a_ctl);
    kpar.err = reinterpret_cast<uint32_t *>(ka.base + a_ctl) + 1;
    kpar.zero = reinterpret_cast<uint32_t *>(ka.base + a_ctl) + 3;
    kpar.vals = ka.base + a_vals;
    kpar.lens = reinterpret_cast<uint32_t *>(ka.base + a_lens);
    launch_key_values(kpar, int64_key, ctx->sm_count * 4, stream);
    CUDA_TRY(cudaStreamSynchronize(stream));  // the staging of the series ids must be consumed before the read-back reuses it
    CUDA_TRY(cudaMemcpyAsync(slot.pinned, ka.base + a_ctl, back_bytes, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    CUDA_TRY(cudaGetLastError());
    stats->kernel_launches += 2;
    stats->h2d_bytes += NS * 8;
    stats->d2h_bytes += back_bytes;
    const uint32_t *ctl = reinterpret_cast<const uint32_t *>(slot.pinned);
    if (ctl[1] != 0) {
        g_last_dev_err = ctl[1];
        char buf[64];
        snprintf(buf, sizeof buf, " (block #%u)", ctl[2]);
        return fail(dev_err_code(ctl[1]), std::string(dev_err_text(ctl[1])) + buf);
    }
    const size_t V = std::min<size_t>(ctl[0], cap);
    values.assign(V, {});
    const uint8_t *hv = slot.pinned + (a_vals - a_ctl);
    const uint32_t *hl = reinterpret_cast<const uint32_t *>(slot.pinned + (a_lens - a_ctl));
    for (size_t v = 0; v < V; ++v) {
        if (int64_key) values[v].assign(hv + v * 8, hv + v * 8 + 8);  // the reference's key bytes: little-endian int64
        else values[v].assign(hv + v * kMaxLit, hv + v * kMaxLit + hl[v]);
    }
    return 0;
}

// 2. one scan pass per value v (the key as an extra predicate) into slice v of the composite table tlc (V x G groups, value-major)
// at `table`, with the pass's column types at coltype + v * F and where each series first shows v at kts / krow + v * NS; the
// first pass also writes the series' spans when `span` is set.  Every pass is synchronised and its device errors collected.
int run_keyed_passes(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, Plan &plan, ExecSlot &slot, const KeyValues &values,
                     const TableLayout &tlc, uint8_t *table, int64_t *coltype, int64_t *kts, uint32_t *krow, int64_t *span, bydb_stats *stats) {
    const bool int64_key = key->value_type == BYDB_VT_INT64;
    const size_t F = plan.fcols.size(), NS = q->n_series, G = static_cast<size_t>(plan.n_groups);
    std::vector<bydb_pred> preds(q->preds, q->preds + q->n_preds);
    preds.emplace_back();
    bydb_query qv = *q;
    qv.n_preds = q->n_preds + 1;
    for (size_t v = 0; v < values.size(); ++v) {
        bydb_pred &kpred = preds.back();
        memset(&kpred, 0, sizeof kpred);
        kpred.family = key->family;
        kpred.tag = key->tag;
        if (int64_key) {
            int64_t lit = 0;
            memcpy(&lit, values[v].data(), 8);
            kpred.op = lit == 0 ? kOpEqOrNil : BYDB_OP_EQ;  // a nil cell is the column's zero value (typed_column.go:49-53)
            kpred.value_type = BYDB_VT_INT64;
            kpred.lit_i64 = lit;
        } else {
            kpred.op = values[v].empty() ? kOpEqOrNil : BYDB_OP_EQ;  // a nil cell and "" are the same key (groupby.go:226-254)
            kpred.value_type = BYDB_VT_STR;
            kpred.lit = values[v].data();
            kpred.lit_len = values[v].size();
        }
        qv.preds = preds.data();
        KeyedPass pass;
        pass.group_off = v * G;
        pass.coltype = coltype + v * F;
        pass.kts = kts + v * NS;
        pass.krow = krow + v * NS;
        pass.span = v == 0 ? span : nullptr;
        int rc = run_scan(ctx, &qv, plan, slot, slot.stream, table, tlc, stats, 0, &pass);
        cudaError_t ce = cudaStreamSynchronize(slot.stream);  // also on failure: nothing may be in flight when the slot goes back
        if (!rc && ce != cudaSuccess) rc = fail(BYDB_EIO, cudaGetErrorString(ce));
        if (!rc) rc = collect_scan(slot, stats);
        if (rc) return rc;
    }
    return 0;
}

// the key table of a keyed result: value k is `values[k]`
void set_key_table(bydb_keyed_result *out, KeyedOwner *owner, const KeyValues &values) {
    owner->key_off.assign(1, 0);
    owner->key_bytes.clear();
    for (const auto &v : values) {
        owner->key_bytes.insert(owner->key_bytes.end(), v.begin(), v.end());
        owner->key_off.push_back(static_cast<uint32_t>(owner->key_bytes.size()));
    }
    if (owner->key_bytes.empty()) owner->key_bytes.push_back(0);
    out->n_keys = static_cast<int32_t>(values.size());
    out->key_off = owner->key_off.data();
    out->key_bytes = owner->key_bytes.data();
}

// 3. insertion order of the V x G composite groups from where each series first shows each value (kts / krow), the table at
// `table` reordered, the ordinary finalisation / Top-N on it, and the rows mapped back to (series group, key value).  The
// caller sized the slot's pinned staging with step_pinned_bytes(q, G, V * G).
int keyed_finish(const bydb_query *q, const Plan &plan, ExecSlot &slot, size_t V, uint8_t *table, const TableLayout &tlc, const int64_t *coltype,
                 const int64_t *kts, const uint32_t *krow, bydb_keyed_result *out, KeyedOwner *owner) {
    cudaStream_t stream = slot.stream;
    const size_t F = plan.fcols.size(), NS = q->n_series, G = static_cast<size_t>(plan.n_groups), GP = G * V;
    const StageLayout st = stage_layout(NS, G);
    Carve carve;
    const size_t b_dst = carve(tlc.total), b_slot = carve(NS * V * 4), b_first = carve(GP * 4), b_perm = carve(GP * 4), b_np = carve(16),
                 b_stage = carve(st.bytes);
    Scratch kb;
    CUDA_TRY(kb.alloc(carve.o, stream));
    CUDA_TRY(cudaMemsetAsync(kb.base + b_slot, 0xff, NS * V * 4, stream));
    KeyOrderParams ko;
    memset(&ko, 0, sizeof ko);
    ko.n_groups = static_cast<int32_t>(G);
    ko.n_values = static_cast<uint32_t>(V);
    ko.n_series = static_cast<uint32_t>(NS);
    // order | group_start of the series groups: staged again (run_scan's copies live in its own scratch)
    stage_series(q, st, slot.pinned);
    CUDA_TRY(cudaMemcpyAsync(kb.base + b_stage, slot.pinned, st.bytes, cudaMemcpyHostToDevice, stream));
    ko.order = reinterpret_cast<const int32_t *>(kb.base + b_stage + st.off_order);
    ko.group_start = reinterpret_cast<const int32_t *>(kb.base + b_stage + st.off_gstart);
    ko.Kts = kts;
    ko.Krow = krow;
    ko.slot = reinterpret_cast<int32_t *>(kb.base + b_slot);
    ko.first_series = reinterpret_cast<int32_t *>(kb.base + b_first);
    ko.perm = reinterpret_cast<int32_t *>(kb.base + b_perm);
    ko.n_present = reinterpret_cast<uint32_t *>(kb.base + b_np);
    launch_key_order(ko, stream);
    launch_permute_table(tlc.at(kb.base + b_dst), tlc.at(table), ko.perm, static_cast<uint32_t>(GP), static_cast<uint32_t>(F), coltype,
                         static_cast<uint32_t>(V), stream);
    CUDA_TRY(cudaStreamSynchronize(stream));  // the staging above is reused by the finalisation's read-back
    out->base.stats.kernel_launches += 3;
    Plan planc = plan;
    planc.n_groups = static_cast<int32_t>(GP);
    int rc = finalize_to_host(q, planc, slot, stream, kb.base + b_dst, tlc, &out->base, true);
    if (rc) {
        cudaStreamSynchronize(stream);
        return rc;
    }
    std::vector<int32_t> perm(GP);
    CUDA_TRY(cudaMemcpyAsync(perm.data(), kb.base + b_perm, GP * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    out->base.stats.d2h_bytes += GP * 4;
    // rows carry the position in insertion order: back to (group of the series, key value)
    auto *ro = static_cast<ResultOwner *>(out->base.owner);
    owner->key_id.resize(ro->group_id.size());
    for (size_t r = 0; r < ro->group_id.size(); ++r) {
        const int32_t comp = perm[static_cast<size_t>(ro->group_id[r])];
        owner->key_id[r] = comp / static_cast<int32_t>(G);
        ro->group_id[r] = comp % static_cast<int32_t>(G);
    }
    out->key_id = owner->key_id.data();
    return 0;
}

// a failure past the point where the result owns memory must not leave a half-filled result with the caller
struct KeyedUndo {
    bydb_ctx *ctx;
    bydb_keyed_result *out;
    bool done = false;
    ~KeyedUndo() {
        if (!done) bydb_keyed_result_free(ctx, out);
    }
};
}  // namespace

void bydb_encoded_pages_free(bydb_ctx *ctx, bydb_encoded_pages *r);

// Group-by on a stored tag (per-row key): see "Group key" in scan_kernels.cu for the device side.
int bydb_scan_agg_keyed(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, bydb_keyed_result *out) {
    return guarded([&]() -> int {
    if (!ctx || !out) return fail(BYDB_EINVAL, "ctx/out is NULL");
    memset(out, 0, sizeof *out);
    int rc = validate_query(q, true);
    if (rc) return rc;
    uint32_t cap = 0;
    rc = check_group_key(q, key, cap);
    if (rc) return rc;
    g_last_dev_err = 0;
    Plan plan;
    rc = make_plan(ctx, q, nullptr, plan);
    if (rc) return rc;
    if (parts_overlap(plan.parts, q->tmin, q->tmax))
        return fail(BYDB_ENOTSUP, "group-key query over parts that overlap in time (version dedup) is not supported on the device path");
    CUDA_TRY(cudaSetDevice(ctx->device));
    SlotLease lease(ctx);
    if (lease.init()) return fail(BYDB_EIO, "cannot create stream");
    ExecSlot &slot = *lease.slot;
    cudaStream_t stream = slot.stream;
    const size_t F = plan.fcols.size(), NS = q->n_series, G = static_cast<size_t>(plan.n_groups);
    memset(&out->base.stats, 0, sizeof out->base.stats);

    KeyValues values;
    rc = discover_keys(ctx, q, key, cap, plan, slot, &out->base.stats, values);
    if (rc) return rc;
    const size_t V = values.size();
    auto owner = new KeyedOwner();
    out->owner = owner;
    KeyedUndo undo{ctx, out};
    set_key_table(out, owner, values);
    if (V == 0) {  // no block selected: no rows (n_rows = 0)
        undo.done = true;
        return 0;
    }

    const size_t GP = G * V;
    if (GP > 0x7fffffffull / std::max<size_t>(F, 1)) return fail(BYDB_ENOMEM, "group-key query: too many composite groups");
    TableLayout tlc(GP, F);
    Carve carve;
    const size_t b_src = carve(tlc.total), b_ct = carve(V * F * 8), b_kts = carve(V * NS * 8), b_krow = carve(V * NS * 4);
    Scratch kb;
    CUDA_TRY(kb.alloc(carve.o, stream));
    CUDA_TRY(cudaMemsetAsync(kb.base + b_ct, 0, V * F * 8, stream));
    if (slot.ensure_pinned(step_pinned_bytes(q, G, GP))) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
    int64_t *ct = reinterpret_cast<int64_t *>(kb.base + b_ct), *kts = reinterpret_cast<int64_t *>(kb.base + b_kts);
    uint32_t *krow = reinterpret_cast<uint32_t *>(kb.base + b_krow);
    rc = run_keyed_passes(ctx, q, key, plan, slot, values, tlc, kb.base + b_src, ct, kts, krow, nullptr, &out->base.stats);
    if (!rc) rc = keyed_finish(q, plan, slot, V, kb.base + b_src, tlc, ct, kts, krow, out, owner);
    if (rc) return rc;
    undo.done = true;
    return 0;
    });
}

void bydb_keyed_result_free(bydb_ctx *ctx, bydb_keyed_result *r) {
    if (!r) return;
    bydb_result_free(ctx, &r->base);
    delete static_cast<KeyedOwner *>(r->owner);
    memset(r, 0, sizeof *r);
}


namespace {
struct EncodedOwner {
    std::vector<uint64_t> page_off;
    std::vector<uint8_t> bytes, needs_cpu;
};
}  // namespace

// Write side (f4): numeric field pages encoded on the device, see encode_kernels.cu.
int bydb_encode_pages(bydb_ctx *ctx, const bydb_encode_input *in, bydb_encoded_pages *out) {
    return guarded([&]() -> int {
    if (!ctx || !in || !out) return fail(BYDB_EINVAL, "ctx/in/out is NULL");
    memset(out, 0, sizeof *out);
    if (in->value_type != BYDB_VT_INT64 && in->value_type != BYDB_VT_FLOAT64) return fail(BYDB_EINVAL, "bydb_encode_pages takes int64 or float64 columns");
    if (in->n_blocks > 0 && (!in->block_rows || !in->values)) return fail(BYDB_EINVAL, "block_rows / values is NULL");
    const size_t NB = in->n_blocks;
    const bool is_float = in->value_type == BYDB_VT_FLOAT64;
    std::vector<uint64_t> block_off(NB + 1, 0), slot_off(NB + 1, 0);
    for (size_t b = 0; b < NB; ++b) {
        if (in->block_rows[b] == 0) return fail(BYDB_EINVAL, "a block without rows");
        block_off[b + 1] = block_off[b] + in->block_rows[b];
        slot_off[b + 1] = slot_off[b] + align_up(11 + 10 * static_cast<size_t>(in->block_rows[b]), 16);  // a varint takes at most 10 bytes
    }
    const size_t NV = block_off[NB];
    auto owner = new EncodedOwner();
    out->owner = owner;
    out->n_blocks = in->n_blocks;
    owner->page_off.assign(NB + 1, 0);
    owner->needs_cpu.assign(std::max<size_t>(NB, 1), 0);
    owner->bytes.assign(1, 0);
    out->page_off = owner->page_off.data();
    out->needs_cpu = owner->needs_cpu.data();
    out->bytes = owner->bytes.data();
    if (NB == 0) return 0;
    bool done = false;
    struct Undo {
        bydb_ctx *ctx;
        bydb_encoded_pages *out;
        bool *done;
        ~Undo() {
            if (!*done) bydb_encoded_pages_free(ctx, out);
        }
    } undo{ctx, out, &done};
    CUDA_TRY(cudaSetDevice(ctx->device));
    SlotLease lease(ctx);
    if (lease.init()) return fail(BYDB_EIO, "cannot create stream");
    cudaStream_t stream = lease.slot->stream;
    Carve carve;
    const size_t d_vals = carve(NV * 8), d_boff = carve((NB + 1) * 8), d_soff = carve((NB + 1) * 8), d_scr = carve(is_float ? NV * 8 : 0),
                 d_exp = carve(is_float ? NV * 2 : 0), d_len = carve(NB * 4), d_st = carve(NB), d_ooff = carve((NB + 1) * 8), d_slots = carve(slot_off[NB]);
    Scratch sc;
    if (sc.alloc(carve.o, stream) != cudaSuccess) {
        cudaGetLastError();
        return fail(BYDB_ENOMEM, "bydb_encode_pages: device allocation failed");
    }
    uint8_t *d = sc.base;
    cudaEvent_t ev0 = lease.slot->ev[0], ev1 = lease.slot->ev[1], ev2 = lease.slot->ev[2], ev3 = lease.slot->ev[3];
    CUDA_TRY(cudaMemcpyAsync(d + d_vals, in->values, NV * 8, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync(d + d_boff, block_off.data(), (NB + 1) * 8, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync(d + d_soff, slot_off.data(), (NB + 1) * 8, cudaMemcpyHostToDevice, stream));
    EncodeParams ep;
    memset(&ep, 0, sizeof ep);
    ep.values = d + d_vals;
    ep.block_off = reinterpret_cast<const uint64_t *>(d + d_boff);
    ep.n_blocks = static_cast<uint32_t>(NB);
    ep.is_float = is_float ? 1u : 0u;
    ep.scratch = reinterpret_cast<int64_t *>(d + d_scr);
    ep.exps = reinterpret_cast<int16_t *>(d + d_exp);
    ep.slots = d + d_slots;
    ep.slot_off = reinterpret_cast<const uint64_t *>(d + d_soff);
    ep.page_len = reinterpret_cast<uint32_t *>(d + d_len);
    ep.status = d + d_st;
    const int grid = ctx->sm_count * 4;
    CUDA_TRY(cudaEventRecord(ev0, stream));
    launch_encode_pages(ep, grid, stream);
    CUDA_TRY(cudaEventRecord(ev1, stream));
    std::vector<uint32_t> page_len(NB);
    CUDA_TRY(cudaMemcpyAsync(page_len.data(), d + d_len, NB * 4, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaMemcpyAsync(owner->needs_cpu.data(), d + d_st, NB, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    CUDA_TRY(cudaGetLastError());
    for (size_t b = 0; b < NB; ++b) {
        owner->page_off[b + 1] = owner->page_off[b] + page_len[b];
        out->n_cpu_blocks += owner->needs_cpu[b] ? 1u : 0u;
    }
    const size_t total = owner->page_off[NB];
    owner->bytes.assign(std::max<size_t>(total, 1), 0);
    out->bytes = owner->bytes.data();
    Scratch compact;
    CUDA_TRY(compact.alloc(std::max<size_t>(total, 256), stream));
    CUDA_TRY(cudaMemcpyAsync(d + d_ooff, owner->page_off.data(), (NB + 1) * 8, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaEventRecord(ev2, stream));
    launch_gather_pages(ep, reinterpret_cast<const uint64_t *>(d + d_ooff), compact.base, grid, stream);
    CUDA_TRY(cudaEventRecord(ev3, stream));
    if (total) CUDA_TRY(cudaMemcpyAsync(owner->bytes.data(), compact.base, total, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaStreamSynchronize(stream));
    CUDA_TRY(cudaGetLastError());
    float ms = 0, ms2 = 0;  // the two kernels only: the host's prefix sum of the page lengths lies between them
    cudaEventElapsedTime(&ms, ev0, ev1);
    cudaEventElapsedTime(&ms2, ev2, ev3);
    out->device_ms = ms + ms2;
    done = true;
    return 0;
    });
}

void bydb_encoded_pages_free(bydb_ctx *, bydb_encoded_pages *r) {
    if (!r) return;
    delete static_cast<EncodedOwner *>(r->owner);
    memset(r, 0, sizeof *r);
}

struct GatherSeg {
    const uint8_t *src;
    size_t dst;
    size_t len;
};
struct GatherImage {
    std::vector<DevBlock> blocks;
    std::vector<DevCol> cols;
    std::vector<GatherSeg> segs;  // ascending dst
    size_t off_cols = 0, off_files = 0, off_pages = 0, bytes = 0;
    uint64_t page_bytes = 0;
};

static int plan_gather(bydb_ctx *ctx, const std::vector<FileImage> &imgs, const bydb_query *q, const Plan &base, const PartDir &dir, GatherImage &g) {
    std::vector<uint16_t> need;
    for (const auto &f : base.fcols) need.push_back(ctx->names.find("f:" + f));
    for (uint32_t i = 0; i < q->n_preds; ++i) need.push_back(ctx->names.find(std::string("t:") + q->preds[i].family + "/" + q->preds[i].tag));
    std::vector<const FileImage *> file_of(dir.files.size(), nullptr);
    for (size_t i = 0; i < dir.files.size(); ++i)
        for (const auto &f : imgs)
            if (f.name == dir.files[i]) file_of[i] = &f;
    if (file_of.empty() || !file_of[0]) return fail(BYDB_ENOENT, "missing timestamps.bin");
    const uint64_t *sb = q->series_ids, *se = q->series_ids + q->n_series;
    struct Page {
        const uint8_t *src;
        uint32_t len;
    };
    std::vector<Page> pages;
    for (const DevBlock &b : dir.blocks) {
        const uint64_t *it = std::lower_bound(sb, se, b.sid);
        if (it == se || *it != b.sid || b.ts_max < q->tmin || b.ts_min > q->tmax) continue;  // plan_blocks' selection (part_iter.go:232-241)
        DevBlock nb = b;
        nb.col_begin = static_cast<uint32_t>(g.cols.size());
        pages.push_back({file_of[0]->data + b.ts_off, b.ts_size});
        uint16_t kept = 0;
        for (uint32_t c = 0; c < b.n_cols; ++c) {
            const DevCol &col = dir.cols[b.col_begin + c];
            if (col.name_id == 0 || std::find(need.begin(), need.end(), col.name_id) == need.end()) continue;
            if (col.file_id >= file_of.size() || !file_of[col.file_id]) return fail(BYDB_ENOENT, "missing file of a column page");
            DevCol nc = col;
            nc.file_id = 0;
            pages.push_back({file_of[col.file_id]->data + col.off, col.size});
            g.cols.push_back(nc);
            ++kept;
        }
        nb.n_cols = kept;
        g.blocks.push_back(nb);
    }
    // layout: directory first, then the pages (16 B aligned, >= 8 B apart: bit windows read a few bytes past a page)
    g.off_cols = align_up(g.blocks.size() * sizeof(DevBlock), 256);
    g.off_files = g.off_cols + align_up(g.cols.size() * sizeof(DevCol), 256);
    g.off_pages = g.off_files + 256;
    size_t cur = g.off_pages, pi = 0;
    g.segs.reserve(pages.size() + 3);
    if (!g.blocks.empty()) g.segs.push_back({reinterpret_cast<const uint8_t *>(g.blocks.data()), 0, g.blocks.size() * sizeof(DevBlock)});
    if (!g.cols.empty()) g.segs.push_back({reinterpret_cast<const uint8_t *>(g.cols.data()), g.off_cols, g.cols.size() * sizeof(DevCol)});
    g.segs.push_back({nullptr, g.off_files, 2 * sizeof(void *)});  // the file table: filled in once the arena address is known
    size_t ci = 0;
    for (DevBlock &nb : g.blocks) {
        nb.ts_off = cur;
        g.segs.push_back({pages[pi].src, cur, pages[pi].len});
        g.page_bytes += pages[pi].len;
        cur = align_up(cur + pages[pi].len + 8, 16);
        ++pi;
        for (uint16_t c = 0; c < nb.n_cols; ++c, ++ci, ++pi) {
            g.cols[ci].off = cur;
            g.segs.push_back({pages[pi].src, cur, pages[pi].len});
            g.page_bytes += pages[pi].len;
            cur = align_up(cur + pages[pi].len + 8, 16);
        }
    }
    g.bytes = align_up(cur + 256, 256);
    return 0;
}

// uploads the image through the staging ring onto `stream`; the copies of one chunk are spread over the worker pool
// the pinned staging ring of the gather path: made at the first pageable cold query -- or at bydb_comm_connect, because a
// page-locked allocation INSIDE a collective can stall peers that share the device (see ExecSlot::ensure_pinned)
static int ensure_stage_ring(bydb_ctx *ctx) {
    StageRing &ring = ctx->stage;
    for (int i = 0; i < StageRing::kBufs; ++i) {
        if (ring.buf[i]) continue;
        if (cudaMallocHost(reinterpret_cast<void **>(&ring.buf[i]), StageRing::kBytes) != cudaSuccess ||
            cudaEventCreateWithFlags(&ring.done[i], cudaEventDisableTiming) != cudaSuccess)
            return fail(BYDB_ENOMEM, "cannot allocate the pinned staging ring");
    }
    return 0;
}

static int upload_gather(bydb_ctx *ctx, GatherImage &g, uint8_t *d_arena, cudaStream_t stream) {
    StageRing &ring = ctx->stage;
    if (int rrc = ensure_stage_ring(ctx)) return rrc;
    const uint8_t *table[2] = {d_arena, d_arena};  // every page lives in the arena: "file" 0 (and a spare slot)
    size_t si = 0;
    for (size_t c0 = 0; c0 < g.bytes; c0 += StageRing::kBytes) {
        const size_t c1 = std::min(g.bytes, c0 + StageRing::kBytes);
        const int bi = ring.next;
        ring.next = (ring.next + 1) % StageRing::kBufs;
        if (ring.pending[bi]) {
            CUDA_TRY(cudaEventSynchronize(ring.done[bi]));
            ring.pending[bi] = false;
        }
        uint8_t *stage = ring.buf[bi];
        // segments that intersect [c0, c1); a segment cut by the chunk edge is copied in two parts
        while (si < g.segs.size() && g.segs[si].dst + g.segs[si].len <= c0) ++si;
        size_t sj = si;
        while (sj < g.segs.size() && g.segs[sj].dst < c1) ++sj;
        const size_t n = sj - si;
        const size_t tasks = std::max<size_t>(1, std::min<size_t>(32, n / 64));
        std::vector<std::future<void>> futs;
        for (size_t t = 0; t < tasks; ++t) {
            const size_t a = si + n * t / tasks, b = si + n * (t + 1) / tasks;
            auto task = std::make_shared<std::packaged_task<void()>>([&g, &table, stage, c0, c1, a, b] {
                for (size_t k = a; k < b; ++k) {
                    const GatherSeg &sg = g.segs[k];
                    const size_t lo = std::max(sg.dst, c0), hi = std::min(sg.dst + sg.len, c1);
                    if (lo >= hi) continue;
                    const uint8_t *src = sg.src ? sg.src : reinterpret_cast<const uint8_t *>(table);
                    memcpy(stage + (lo - c0), src + (lo - sg.dst), hi - lo);
                }
            });
            futs.push_back(task->get_future());
            if (t + 1 < tasks) ctx->pool.submit([task] { (*task)(); });
            else (*task)();  // the calling thread takes the last share itself
        }
        for (auto &f : futs) f.get();
        // the gaps between pages travel too (they are padding): one contiguous copy per chunk
        CUDA_TRY(cudaMemcpyAsync(d_arena + c0, stage, c1 - c0, cudaMemcpyHostToDevice, stream));
        CUDA_TRY(cudaEventRecord(ring.done[bi], stream));
        ring.pending[bi] = true;
    }
    return 0;
}

// Cold path, one zero-copy part: the block index is parsed in slices and the scan of slice k runs on the
// GPU (pulling its pages over PCIe) while the host parses slice k+1; the per-slice partial tables are
// combined on the device.  A series may straddle slices: partial tables merge exactly.
// gather = the images are in pageable memory: the touched pages of every slice are collected and staged (see above).
static int scan_agg_host_pipelined(bydb_ctx *ctx, const bydb_part_files *files, const bydb_query *q, bydb_result *out, bool gather = false) {
    constexpr int K = ExecSlot::kMaxBatches;  // most slices (scan launches) per call
    std::unique_lock<std::mutex> ring_lock(ctx->stage.mu, std::defer_lock);
    if (gather) ring_lock.lock();
    SlotLease lease(ctx);
    if (lease.init()) return fail(BYDB_EIO, "cannot create stream");
    ExecSlot &slot = *lease.slot;
    Plan base;
    if (int rc = query_shape(q, base)) return rc;
    const TableLayout &tl = base.tl;
    std::vector<FileImage> imgs;
    if (int frc = file_images(files, imgs)) return frc;
    size_t n_primary = 0;
    {
        std::string err;
        const int rc0 = count_primary_blocks(imgs, &n_primary, err);
        if (rc0) return fail(rc0, err);
    }
    Scratch tables;
    CUDA_TRY(tables.alloc(tl.total * K, slot.stream));
    if (slot.ensure_pinned(step_pinned_bytes(q, tl.G, tl.G, K))) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
    memset(&out->stats, 0, sizeof out->stats);
    // The block index is parsed in the background from the start, one task per group of primary blocks (they are
    // independent zstd frames).  The main thread takes the pieces in order: whatever is parsed by the time the GPU can
    // take more work becomes the next slice -- first slice = the first piece (shortest wait before the first launch),
    // later slices grow with what the parsers delivered meanwhile, the last allowed slice takes the rest.
    struct Parsed {
        PartDir dir;
        std::string err;
        int rc = 0;
    };
    // pieces of one or two primary blocks: the first piece (= the first slice the GPU can start on) is parsed quickly; with
    // fewer, larger pieces the GPU waits for the first big one before anything is launched
    const size_t T = std::max<size_t>(1, std::min<size_t>(n_primary, 128));
    const bool trace = getenv("BYDB_TRACE") != nullptr;  // host-side timeline of the cold path on stderr (read per call: a caller can trace one step)
    const auto t_begin = std::chrono::steady_clock::now();
    auto since = [&] { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_begin).count(); };
    std::vector<std::future<Parsed>> parses;
    for (size_t t = 0; t < T; ++t) {
        auto task = std::make_shared<std::packaged_task<Parsed()>>([ctx, &imgs, t, T] {
            Parsed r;
            r.rc = build_part_dir(imgs, ctx->names, r.dir, r.err, t, T);
            return r;
        });
        parses.push_back(task->get_future());
        ctx->pool.submit([task] { (*task)(); });
    }
    TransientParts tmp(ctx);
    std::vector<std::shared_ptr<GatherImage>> gathered;
    int rc = 0, n_slices = 0;
    size_t next = 0;
    while (next < T) {
        std::vector<PartDir> pieces;
        auto take = [&] {
            Parsed pr = parses[next++].get();
            if (pr.rc && !rc) rc = fail(pr.rc, "block index: " + pr.err);
            pieces.push_back(std::move(pr.dir));
        };
        take();
        if (rc || n_slices == K - 1) {
            while (next < T) take();  // the last slice takes the rest; after a failure every task is still joined
        } else {
            while (next < T && parses[next].wait_for(std::chrono::seconds(0)) == std::future_status::ready) take();
        }
        if (rc) break;
        PartDir merged;
        {
            std::string err;
            const int mrc = merge_part_dirs(pieces, merged, err);
            if (mrc) {
                rc = fail(mrc, err);
                continue;
            }
        }
        const int k = n_slices++;
        if (trace) fprintf(stderr, "[bydb cold] slice %d = pieces ..%zu of %zu, parsed at %.0f us (%zu blocks)\n", k, next, T, since(), merged.blocks.size());
        std::shared_ptr<Part> p;
        uint64_t h2d = 0;
        if (gather) {
            auto gi = std::make_shared<GatherImage>();
            rc = plan_gather(ctx, imgs, q, base, merged, *gi);
            if (rc) continue;
            if (gi->blocks.empty() && (next < T || n_slices > 1)) {
                --n_slices;  // nothing of this slice is selected (a query that selects nothing at all still runs one empty slice)
                continue;
            }
            p = std::make_shared<Part>();
            p->id = tmp.next_id();
            p->device = ctx->device;
            p->pool_stream = slot.stream;
            p->hbm_bytes = gi->bytes;
            rc = hbm_reserve(ctx, gi->bytes);
            if (rc) continue;
            if (cudaMallocAsync(reinterpret_cast<void **>(&p->d_arena), gi->bytes, slot.stream) != cudaSuccess) {
                p->d_arena = nullptr;
                hbm_release(ctx, gi->bytes);
                rc = fail(BYDB_ENOMEM, "device allocation failed for the gathered pages");
                continue;
            }
            tmp.parts.push_back(p);
            rc = upload_gather(ctx, *gi, p->d_arena, slot.stream);
            if (rc) continue;
            p->d_blocks = reinterpret_cast<const DevBlock *>(p->d_arena);
            p->d_cols = reinterpret_cast<const DevCol *>(p->d_arena + gi->off_cols);
            p->d_files = reinterpret_cast<const uint8_t *const *>(p->d_arena + gi->off_files);
            p->dir.blocks = std::move(gi->blocks);   // only the sizes are read from here on
            p->dir.files = {"arena"};
            p->dir.min_ts = merged.min_ts;
            p->dir.max_ts = merged.max_ts;
            h2d = gi->bytes;
            gathered.push_back(gi);                  // the directory vectors feed the staged copies: keep them until the end
        } else {
            AdmitOptions opt;
            opt.zero_copy = true;
            opt.parsed = &merged;
            rc = tmp.admit(files, &h2d, opt);
            if (rc) continue;
            p = tmp.parts.back();
        }
        out->stats.h2d_bytes += h2d;
        Plan plan = base;
        plan.parts = {p};
        plan.total_blocks = static_cast<uint32_t>(p->dir.blocks.size());
        rc = run_scan(ctx, q, plan, slot, slot.stream, tables.base + tl.total * static_cast<size_t>(k), tl, &out->stats, k);
        if (trace) fprintf(stderr, "[bydb cold] slice %d enqueued at %.0f us\n", k, since());
    }
    while (next < T) (void)parses[next++].get();
    if (!rc && n_slices > 0) {
        launch_combine_tables(tables.base, static_cast<uint32_t>(n_slices), tl, slot.stream);
        out->stats.kernel_launches += 1;
        // the pinned staging of the last slices may still be in flight: finalize copies into it only after the kernels
        rc = finalize_to_host(q, base, slot, slot.stream, tables.base, tl, out);
        if (rc) cudaStreamSynchronize(slot.stream);  // nothing of this call may be in flight when the slot and the parts go back
        if (trace) fprintf(stderr, "[bydb cold] finalized at %.0f us\n", since());
    } else {
        cudaStreamSynchronize(slot.stream);
    }
    for (int k = 0; k < static_cast<int>(tmp.parts.size()); ++k) {
        int rc2 = collect_scan(slot, &out->stats, k);
        if (!rc && rc2) {
            bydb_result_free(ctx, out);
            rc = rc2;
        }
    }
    if (!rc && !gather) out->stats.h2d_bytes += out->stats.page_bytes;  // pages were read in place over PCIe
    return rc;
}

int bydb_scan_agg_host(bydb_ctx *ctx, uint32_t n_parts, const bydb_part_files *parts, const bydb_query *q, bydb_result *out) {
    return guarded([&]() -> int {
    if (!ctx || !out) return fail(BYDB_EINVAL, "ctx/out is NULL");
    memset(out, 0, sizeof *out);
    int rc = validate_query(q, false);
    if (rc) return rc;
    if (n_parts == 0 || !parts || n_parts > kMaxParts) return fail(BYDB_EINVAL, "need 1..64 host parts");
    CUDA_TRY(cudaSetDevice(ctx->device));
    // The cold path first scans the pages as they are; only when a block turns out to hold fallback pages
    // (EncodeTypePlain numeric pages, zstd string blocks) are the parts unpacked on the device and scanned again.
    auto wants_unpack = [](int code) {
        return code == BYDB_ENOTSUP && (g_last_dev_err == kErrPlainPage || g_last_dev_err == kErrZstdDict || g_last_dev_err == kErrTagPlain);
    };
    g_last_dev_err = 0;
    if (n_parts == 1) {
        // pinned by the caller: pages pulled in place over PCIe; pageable: the touched pages gathered and staged
        rc = scan_agg_host_pipelined(ctx, &parts[0], q, out, (q->flags & BYDB_Q_HOST_ZERO_COPY) == 0);
        if (!wants_unpack(rc)) return rc;
    }
    for (int attempt = rc ? 1 : 0; attempt < 2; ++attempt) {
        TransientParts tmp(ctx);
        uint64_t h2d = 0;
        rc = 0;
        g_last_dev_err = 0;
        memset(out, 0, sizeof *out);
        AdmitOptions opt;
        opt.zero_copy = (q->flags & BYDB_Q_HOST_ZERO_COPY) != 0;
        opt.unpack = attempt == 1;
        for (uint32_t i = 0; i < n_parts && !rc; ++i) rc = tmp.admit(&parts[i], &h2d, opt);
        if (!rc) rc = scan_agg_impl(ctx, q, &tmp.parts, out, h2d);
        if (!rc && opt.zero_copy) out->stats.h2d_bytes += out->stats.page_bytes;  // pages were read in place over PCIe
        if (!wants_unpack(rc)) break;
    }
    return rc;
    });
}

void bydb_result_free(bydb_ctx *, bydb_result *r) {
    if (!r) return;
    delete static_cast<ResultOwner *>(r->owner);
    memset(r, 0, sizeof *r);
}

int bydb_partials_layout(const bydb_query *q, bydb_partials_layout_t *out) {
    return guarded([&]() -> int {
    if (!q || !out) return fail(BYDB_EINVAL, "NULL argument");
    int rc = validate_query(q, false);
    if (rc) return rc;
    Plan plan;
    rc = query_shape(q, plan);
    if (rc) return rc;
    const TableLayout &tl = plan.tl;
    out->total_bytes = tl.total;
    out->off_sum_f64 = tl.off_sum_f64;
    out->n_sum_f64 = tl.GF;
    out->off_max_f64 = tl.off_max_f64;
    out->n_max_f64 = 2 * tl.GF;
    out->off_sum_i64 = tl.off_sum_i64;
    out->n_sum_i64 = 2 * tl.GF + tl.G;
    out->off_max_i64 = tl.off_max_i64;
    out->n_max_i64 = 2 * tl.GF + tl.F;
    return 0;
    });
}

int bydb_scan_partials(bydb_ctx *ctx, const bydb_query *q, void *d_partials, uint64_t bytes, void *stream, bydb_stats *stats) {
    return guarded([&]() -> int {
    if (!ctx || !d_partials) return fail(BYDB_EINVAL, "ctx/d_partials is NULL");
    int rc = validate_query(q, true);
    if (rc) return rc;
    Plan plan;
    rc = make_plan(ctx, q, nullptr, plan);
    if (rc) return rc;
    const TableLayout &tl = plan.tl;
    if (bytes < tl.total) return fail(BYDB_EINVAL, "partial table buffer too small");
    CUDA_TRY(cudaSetDevice(ctx->device));
    SlotLease lease(ctx);
    if (lease.init()) return fail(BYDB_EIO, "cannot create stream");
    cudaStream_t s = static_cast<cudaStream_t>(stream);  // NULL = the legacy default stream, like every partial-table call
    bydb_stats local;
    memset(&local, 0, sizeof local);
    rc = run_scan(ctx, q, plan, *lease.slot, s, static_cast<uint8_t *>(d_partials), tl, &local);
    if (!rc && !stats) {
        // asynchronous form: nothing is read back here.  A device-side failure travels in the table (coltype words)
        // and surfaces in bydb_reduce_finalize on whichever rank finalises.
        CUDA_TRY(cudaEventRecord(lease.slot->busy, s));
        lease.slot->busy_pending = true;
        return 0;
    }
    if (!rc) {
        CUDA_TRY(cudaStreamSynchronize(s));
        CUDA_TRY(cudaGetLastError());
        rc = collect_scan(*lease.slot, &local);
    }
    if (stats) *stats = local;
    return rc;
    });
}

int bydb_partials_combine(bydb_ctx *ctx, const bydb_query *q, void *d_tables, uint32_t n_tables, uint64_t bytes_each, void *stream) {
    return guarded([&]() -> int {
    if (!ctx || !d_tables || n_tables == 0) return fail(BYDB_EINVAL, "NULL argument");
    int rc = validate_query(q, false);
    if (rc) return rc;
    Plan plan;
    rc = query_shape(q, plan);
    if (rc) return rc;
    const TableLayout &tl = plan.tl;
    if (bytes_each != tl.total) return fail(BYDB_EINVAL, "partial tables must be exactly bydb_partials_layout().total_bytes each");
    CUDA_TRY(cudaSetDevice(ctx->device));
    launch_combine_tables(static_cast<uint8_t *>(d_tables), n_tables, tl, static_cast<cudaStream_t>(stream));
    CUDA_TRY(cudaGetLastError());
    return 0;
    });
}

int bydb_reduce_finalize(bydb_ctx *ctx, const bydb_query *q, const void *d_partials, uint64_t bytes, void *stream, bydb_result *out) {
    return guarded([&]() -> int {
    if (!ctx || !d_partials || !out) return fail(BYDB_EINVAL, "NULL argument");
    memset(out, 0, sizeof *out);
    int rc = validate_query(q, false);
    if (rc) return rc;
    Plan plan;
    rc = query_shape(q, plan);
    if (rc) return rc;
    const TableLayout &tl = plan.tl;
    if (bytes < tl.total) return fail(BYDB_EINVAL, "partial table buffer too small");
    CUDA_TRY(cudaSetDevice(ctx->device));
    SlotLease lease(ctx);
    if (lease.init()) return fail(BYDB_EIO, "cannot create stream");
    cudaStream_t s = static_cast<cudaStream_t>(stream);  // NULL = the legacy default stream, like every partial-table call
    return finalize_to_host(q, plan, *lease.slot, s, static_cast<const uint8_t *>(d_partials), tl, out, true);
    });
}


int bydb_query_prepare(bydb_ctx *ctx, const bydb_query *q, bydb_prepared **out) {
    return guarded([&]() -> int {
    if (!ctx || !out) return fail(BYDB_EINVAL, "ctx/out is NULL");
    *out = nullptr;
    int rc = validate_query(q, true);
    if (rc) return rc;
    CUDA_TRY(cudaSetDevice(ctx->device));
    auto p = new bydb_prepared();
    p->parts.assign(q->parts, q->parts + q->n_parts);
    p->sids.assign(q->series_ids, q->series_ids + q->n_series);
    if (q->series_group) p->groups.assign(q->series_group, q->series_group + q->n_series);
    p->aggs.assign(q->aggs, q->aggs + q->n_aggs);
    p->agg_names.resize(q->n_aggs);
    for (uint32_t a = 0; a < q->n_aggs; ++a) p->agg_names[a] = q->aggs[a].field;
    for (uint32_t a = 0; a < q->n_aggs; ++a) p->aggs[a].field = p->agg_names[a].c_str();
    p->preds.assign(q->preds, q->preds + q->n_preds);
    p->pred_family.resize(q->n_preds);
    p->pred_tag.resize(q->n_preds);
    p->pred_lit.resize(q->n_preds);
    for (uint32_t i = 0; i < q->n_preds; ++i) {
        p->pred_family[i] = q->preds[i].family;
        p->pred_tag[i] = q->preds[i].tag;
        if (q->preds[i].lit && q->preds[i].lit_len) p->pred_lit[i].assign(q->preds[i].lit, q->preds[i].lit + q->preds[i].lit_len);
    }
    for (uint32_t i = 0; i < q->n_preds; ++i) {
        p->preds[i].family = p->pred_family[i].c_str();
        p->preds[i].tag = p->pred_tag[i].c_str();
        p->preds[i].lit = p->pred_lit[i].empty() ? nullptr : p->pred_lit[i].data();
    }
    p->q = *q;
    p->q.parts = p->parts.data();
    p->q.series_ids = p->sids.data();
    p->q.series_group = q->series_group ? p->groups.data() : nullptr;
    p->q.aggs = p->aggs.data();
    p->q.preds = p->preds.data();
    // a dedicated slot: stream, events, pinned staging
    p->slot.reset(new ExecSlot());
    bool ok = p->slot->create() == 0;  // with its pinned staging: nothing page-locked is allocated inside an execution
    if (ok) {
        // sized for this query now (see ExecSlot::ensure_pinned: a page-locked allocation inside a collective can stall the peers)
        // a query with too many fields is refused at its first execution, like bydb_scan_agg would
        Plan shape;
        (void)query_shape(q, shape);
        ok = p->slot->ensure_pinned(step_pinned_bytes(q, shape.tl.G, shape.tl.G)) == 0;
    }
    ok = ok && cudaEventCreate(&p->t0) == cudaSuccess && cudaEventCreate(&p->t1) == cudaSuccess;
    if (!ok) {
        prepared_destroy(p);
        return fail(BYDB_EIO, "cannot create the stream / events of a prepared query");
    }
    *out = p;
    return 0;
    });
}

void bydb_query_release(bydb_ctx *ctx, bydb_prepared *p) {
    if (ctx) cudaSetDevice(ctx->device);
    prepared_destroy(p);
}

int bydb_scan_agg_prepared(bydb_ctx *ctx, bydb_prepared *p, bydb_result *out) {
    return guarded([&]() -> int {
    if (!ctx || !p || !out) return fail(BYDB_EINVAL, "NULL argument");
    memset(out, 0, sizeof *out);
    std::lock_guard<std::mutex> lk(p->mu);
    g_last_dev_err = 0;
    CUDA_TRY(cudaSetDevice(ctx->device));
    // the first execution runs the ordinary path (it also performs the one-time kernel attribute setup); the second one
    // captures; from then on the graph is replayed
    const uint64_t run = p->runs++;
    if (run == 0 || !p->capturable) return scan_agg_impl(ctx, &p->q, nullptr, out, 0);
    if (!p->exec) {
        const int rc = prepared_capture(ctx, p);
        if (rc) return rc;
        if (!p->exec) return scan_agg_impl(ctx, &p->q, nullptr, out, 0);
    }
    if (!check_held_parts(ctx, p->parts, p->exec, p->held)) return fail(BYDB_ENOENT, "unknown part handle");
    if (!p->exec) {
        const int rc = prepared_capture(ctx, p);
        if (rc) return rc;
        if (!p->exec) return scan_agg_impl(ctx, &p->q, nullptr, out, 0);
    }
    const int rc = replay_graph(p->exec, *p->slot, p->t0, p->t1, p->captured, p->express, &out->stats);
    if (rc) return rc;
    return finalize_parse(p->slot->pinned + p->host_off, p->fl, false, out);
    });
}


struct PartialRowsOwner {
    std::vector<int32_t> group_id;
    std::vector<uint8_t> is_float;
    std::vector<int64_t> val_i64, cnt_i64;
    std::vector<double> val_f64, cnt_f64;
};

int bydb_partials_rows(bydb_ctx *ctx, const bydb_query *q, const void *d_partials, uint64_t bytes, void *stream, bydb_partial_rows *out) {
    return guarded([&]() -> int {
    if (!ctx || !d_partials || !out) return fail(BYDB_EINVAL, "NULL argument");
    memset(out, 0, sizeof *out);
    int rc = validate_query(q, false);
    if (rc) return rc;
    Plan plan;
    rc = query_shape(q, plan);
    if (rc) return rc;
    const TableLayout &tl = plan.tl;
    const std::vector<int> &agg_fcol = plan.agg_fcol;
    const size_t G = tl.G, F = tl.F, A = q->n_aggs;
    if (bytes < tl.total) return fail(BYDB_EINVAL, "partial table buffer too small");
    CUDA_TRY(cudaSetDevice(ctx->device));
    std::vector<uint8_t> h(tl.total);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    CUDA_TRY(cudaMemcpyAsync(h.data(), d_partials, tl.total, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    const TablePtrs t = tl.at(h.data());
    uint32_t dev_err = 0;
    for (size_t c = 0; c < F; ++c) dev_err = std::max(dev_err, static_cast<uint32_t>(t.coltype[c] >> 8));
    rc = table_status(dev_err);
    if (rc) return rc;
    auto owner = std::make_unique<PartialRowsOwner>();
    owner->is_float.resize(A);
    for (size_t a = 0; a < A; ++a) owner->is_float[a] = (t.coltype[agg_fcol[a]] & 0xff) == BYDB_VT_FLOAT64 ? 1 : 0;
    for (size_t g = 0; g < G; ++g) {
        if (t.rows[g] <= 0) continue;  // the group never appeared on this node
        owner->group_id.push_back(static_cast<int32_t>(g));
        for (size_t a = 0; a < A; ++a) {
            const size_t o = g * F + static_cast<size_t>(agg_fcol[a]);
            const bool isf = owner->is_float[a] != 0;
            const int64_t n = t.cnt[o];
            const bool met = met_column(isf, n, t.max_i64[o], t.max_f64[o]);  // else MIN / MAX keep the zero value
            int64_t vi = 0, ci = 0;
            double vf = 0.0, cf = 0.0;
            switch (q->aggs[a].func) {
                case BYDB_AGG_SUM: vi = t.sum_i64[o]; vf = t.sum_f64[o]; break;
                case BYDB_AGG_COUNT: vi = n; vf = static_cast<double>(n); break;
                case BYDB_AGG_MAX:
                    vi = n > 0 ? t.max_i64[o] : met ? INT64_MIN : 0;
                    vf = n > 0 ? t.max_f64[o] : met ? -1.7976931348623157e308 : 0.0;
                    break;
                case BYDB_AGG_MIN:
                    vi = n > 0 ? ~t.notmin_i64[o] : met ? INT64_MAX : 0;
                    vf = n > 0 ? -t.negmin_f64[o] : met ? 1.7976931348623157e308 : 0.0;
                    break;
                case BYDB_AGG_MEAN: vi = t.sum_i64[o]; vf = t.sum_f64[o]; ci = n; cf = static_cast<double>(n); break;
            }
            owner->val_i64.push_back(isf ? 0 : vi);
            owner->val_f64.push_back(isf ? vf : 0.0);
            owner->cnt_i64.push_back(isf ? 0 : ci);
            owner->cnt_f64.push_back(isf ? cf : 0.0);
        }
    }
    out->n_rows = static_cast<int32_t>(owner->group_id.size());
    out->n_aggs = static_cast<int32_t>(A);
    out->group_id = owner->group_id.data();
    out->is_float = owner->is_float.data();
    out->val_i64 = owner->val_i64.data();
    out->val_f64 = owner->val_f64.data();
    out->cnt_i64 = owner->cnt_i64.data();
    out->cnt_f64 = owner->cnt_f64.data();
    out->owner = owner.release();
    return 0;
    });
}

void bydb_partial_rows_free(bydb_ctx *, bydb_partial_rows *r) {
    if (!r) return;
    delete static_cast<PartialRowsOwner *>(r->owner);
    memset(r, 0, sizeof *r);
}

// ------------------------------------------------------------------------------------------------
// Multi-GPU reduce behind the C ABI: peer mailboxes over NVLink (see scan_kernels.cu, comm_*_kernel)
// ------------------------------------------------------------------------------------------------
struct CommBlob {  // what travels inside a bydb_comm_handle
    uint32_t magic, device;
    uint64_t pid, raw_ptr, slot_bytes, mailbox_bytes;
    cudaIpcMemHandle_t ipc;
    unsigned char uuid[16];  // the physical GPU (device ordinals differ between processes under CUDA_VISIBLE_DEVICES)
};
static_assert(sizeof(CommBlob) <= sizeof(bydb_comm_handle), "bydb_comm_handle too small");

int bydb_comm_export(bydb_ctx *ctx, uint64_t max_table_bytes, int32_t max_ranks, bydb_comm_handle *out) {
    return guarded([&]() -> int {
    if (!ctx || !out) return fail(BYDB_EINVAL, "ctx/out is NULL");
    if (max_ranks < 1 || max_ranks > kCommMaxRanks) return fail(BYDB_EINVAL, "max_ranks must be 1..64");
    if (max_table_bytes == 0 || max_table_bytes > (1ull << 32)) return fail(BYDB_EINVAL, "bad max_table_bytes");
    CUDA_TRY(cudaSetDevice(ctx->device));
    Comm &cm = ctx->comm;
    std::lock_guard<std::mutex> lk(cm.mu);
    if (cm.mine) return fail(BYDB_EINVAL, "bydb_comm_export was already called on this context");
    cm.slot_bytes = align_up(max_table_bytes, 256);
    cm.mailbox_bytes = kCommCtl + 2 * static_cast<size_t>(max_ranks) * cm.slot_bytes;
    if (int rc = hbm_reserve(ctx, cm.mailbox_bytes, "HBM budget exceeded (mailbox)")) return rc;
    if (cudaMalloc(reinterpret_cast<void **>(&cm.mine), cm.mailbox_bytes) != cudaSuccess) {
        cudaGetLastError();  // the failed allocation must not surface in a later call's error check
        cm.mine = nullptr;
        hbm_release(ctx, cm.mailbox_bytes);
        return fail(BYDB_ENOMEM, "device allocation failed for the mailbox");
    }
    CUDA_TRY(cudaMemset(cm.mine, 0, cm.mailbox_bytes));
    CommBlob b;
    memset(&b, 0, sizeof b);
    b.magic = 0xB1DBC011u;
    b.device = static_cast<uint32_t>(ctx->device);
    b.pid = static_cast<uint64_t>(getpid());
    b.raw_ptr = reinterpret_cast<uint64_t>(cm.mine);
    b.slot_bytes = cm.slot_bytes;
    b.mailbox_bytes = cm.mailbox_bytes;
    CUDA_TRY(cudaIpcGetMemHandle(&b.ipc, cm.mine));
    {
        cudaDeviceProp prop;
        CUDA_TRY(cudaGetDeviceProperties(&prop, ctx->device));
        static_assert(sizeof prop.uuid.bytes == sizeof b.uuid, "uuid size");
        memcpy(b.uuid, prop.uuid.bytes, sizeof b.uuid);
    }
    memset(out, 0, sizeof *out);
    memcpy(out, &b, sizeof b);
    return 0;
    });
}

int bydb_comm_connect(bydb_ctx *ctx, int32_t rank, int32_t nranks, const bydb_comm_handle *all) {
    return guarded([&]() -> int {
    if (!ctx || !all) return fail(BYDB_EINVAL, "ctx/handles is NULL");
    if (nranks < 1 || nranks > kCommMaxRanks || rank < 0 || rank >= nranks) return fail(BYDB_EINVAL, "bad rank / nranks");
    CUDA_TRY(cudaSetDevice(ctx->device));
    Comm &cm = ctx->comm;
    std::lock_guard<std::mutex> lk(cm.mu);
    if (!cm.mine) return fail(BYDB_EINVAL, "call bydb_comm_export first");
    if (cm.nranks) return fail(BYDB_EINVAL, "bydb_comm_connect was already called on this context");
    std::vector<uint8_t *> peer(static_cast<size_t>(nranks), nullptr);
    std::vector<bool> opened(static_cast<size_t>(nranks), false);
    std::vector<size_t> slots(static_cast<size_t>(nranks), 0);
    bool shares_device = false;  // another rank lives on this GPU (tests, a box with fewer GPUs than ranks)
    unsigned char my_uuid[16];
    {
        cudaDeviceProp prop;
        CUDA_TRY(cudaGetDeviceProperties(&prop, ctx->device));
        memcpy(my_uuid, prop.uuid.bytes, sizeof my_uuid);
    }
    for (int r = 0; r < nranks; ++r) {
        CommBlob b;
        memcpy(&b, &all[r], sizeof b);
        if (b.magic != 0xB1DBC011u) return fail(BYDB_EINVAL, "handle of rank " + std::to_string(r) + " is not a bydb_comm_handle");
        if (kCommCtl + 2 * static_cast<uint64_t>(nranks) * b.slot_bytes > b.mailbox_bytes)
            return fail(BYDB_EINVAL, "mailbox of rank " + std::to_string(r) + " was exported for fewer ranks");
        slots[r] = b.slot_bytes;
        if (r != rank && memcmp(b.uuid, my_uuid, sizeof my_uuid) == 0) shares_device = true;
        if (r == rank) {
            if (b.raw_ptr != reinterpret_cast<uint64_t>(cm.mine)) return fail(BYDB_EINVAL, "handles[rank] is not this context's own handle");
            peer[r] = cm.mine;
        } else if (b.pid == static_cast<uint64_t>(getpid())) {
            // same process (several contexts, one per GPU, or tests): the pointer is valid as it is once peer access is on
            if (static_cast<int>(b.device) != ctx->device) {
                int can = 0;
                cudaDeviceCanAccessPeer(&can, ctx->device, static_cast<int>(b.device));
                if (!can) return fail(BYDB_ENOTSUP, "no peer access between device " + std::to_string(ctx->device) + " and " + std::to_string(b.device));
                const cudaError_t e = cudaDeviceEnablePeerAccess(static_cast<int>(b.device), 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(BYDB_EIO, std::string("cudaDeviceEnablePeerAccess: ") + cudaGetErrorString(e));
                cudaGetLastError();
            }
            peer[r] = reinterpret_cast<uint8_t *>(b.raw_ptr);
        } else {
            void *p = nullptr;
            const cudaError_t e = cudaIpcOpenMemHandle(&p, b.ipc, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) {
                for (int k = 0; k < r; ++k)
                    if (opened[k]) cudaIpcCloseMemHandle(peer[k]);
                return fail(BYDB_EIO, std::string("cudaIpcOpenMemHandle (rank ") + std::to_string(r) + "): " + cudaGetErrorString(e));
            }
            peer[r] = static_cast<uint8_t *>(p);
            opened[r] = true;
        }
    }
    cm.peer = std::move(peer);
    cm.ipc_opened = std::move(opened);
    cm.peer_slot_bytes = std::move(slots);
    cm.rank = rank;
    cm.nranks = nranks;
    cm.epoch = 0;
    cm.last_use.assign(2 * static_cast<size_t>(nranks), 0);
    // ranks that share a device must not make page-locked allocations inside a collective (ExecSlot::ensure_pinned): the
    // staging ring of the pageable cold path is made now
    if (shares_device && ensure_stage_ring(ctx) != 0) g_last_error.clear();
    if (shares_device) {
        // host-polled waits (see Comm::shared_device): the polling stream and its pinned words are made now
        if (cudaStreamCreateWithFlags(&cm.poll_stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaMallocHost(reinterpret_cast<void **>(&cm.poll_buf), sizeof(unsigned long long) * kCommMaxRanks) != cudaSuccess)
            return fail(BYDB_EIO, "cannot create the polling stream of a shared-device collective");
        cm.shared_device = true;
    }
    return 0;
    });
}

// Host-side form of comm_wait_kernel for ranks that share a device (Comm::shared_device): polls n words until all have reached
// `epoch`; bounded like the kernel (60 s).  Returns 0 or kErrPeerTimeout.
static uint32_t comm_wait_host(Comm &cm, const unsigned long long *dev_words, uint32_t n, unsigned long long epoch) {
    const auto t0 = std::chrono::steady_clock::now();
    for (uint32_t spins = 0;; ++spins) {
        if (cudaMemcpyAsync(cm.poll_buf, dev_words, sizeof(unsigned long long) * n, cudaMemcpyDeviceToHost, cm.poll_stream) != cudaSuccess ||
            cudaStreamSynchronize(cm.poll_stream) != cudaSuccess) {
            cudaGetLastError();
            return kErrPeerTimeout;
        }
        bool all = true;
        for (uint32_t i = 0; i < n; ++i) all = all && cm.poll_buf[i] >= epoch;
        if (all) return 0;
        if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(60)) return kErrPeerTimeout;
        if (spins > 64) std::this_thread::sleep_for(std::chrono::microseconds(20));
        else std::this_thread::yield();
    }
}

// What one collective of epoch `epoch` uses of the root's mailbox (layout above struct Comm), and this rank's own error word.
struct MailboxView {
    uint64_t epoch;
    size_t parity, slot_bytes;            // slot parity of the epoch, slot size of the root's mailbox
    uint8_t *slots0, *my_slot;            // rank 0's and this rank's slot of that parity
    unsigned long long *flags, *status, *done;
    uint32_t *my_err;
    uint64_t *last_use;                   // Comm::last_use of this root and parity
    // Makes this collective the slots' latest use and returns the epoch of the previous one (0 = none): the root must have read
    // the slots of that one (its `done` word) before they are overwritten.
    uint64_t claim_slots() {
        const uint64_t prev = *last_use;
        *last_use = epoch;
        return prev;
    }
};
static MailboxView mailbox_view(Comm &cm, int32_t root, uint64_t epoch) {
    MailboxView v;
    v.epoch = epoch;
    v.parity = static_cast<size_t>(epoch & 1u);
    v.slot_bytes = cm.peer_slot_bytes[static_cast<size_t>(root)];
    uint8_t *root_mb = cm.peer[static_cast<size_t>(root)];
    v.slots0 = root_mb + kCommCtl + v.parity * static_cast<size_t>(cm.nranks) * v.slot_bytes;
    v.my_slot = v.slots0 + static_cast<size_t>(cm.rank) * v.slot_bytes;
    v.flags = reinterpret_cast<unsigned long long *>(root_mb);
    v.status = reinterpret_cast<unsigned long long *>(root_mb + kCommStatusOff);
    v.done = reinterpret_cast<unsigned long long *>(root_mb + kCommDoneOff);
    v.my_err = reinterpret_cast<uint32_t *>(cm.mine + kCommErrOff);
    v.last_use = &cm.last_use[2 * static_cast<size_t>(root) + v.parity];
    return v;
}

// the first rank whose status word of `epoch` (as read back from the root's mailbox) carries a failure, as that failure
static int peer_failure(const unsigned long long *status, int nranks, uint64_t epoch, const char *msg) {
    for (int r = 0; r < nranks; ++r) {
        const unsigned long long w = status[r];
        if ((w >> 32) == (epoch & 0xffffffffull) && static_cast<uint32_t>(w) != 0)
            return fail(-static_cast<int>(static_cast<uint32_t>(w)), "multi-GPU reduce: rank " + std::to_string(r) + msg);
    }
    return 0;
}

// One collective call of the peer-mailbox reduce, shared by bydb_scan_reduce and bydb_scan_reduce_keyed: the epoch and slot
// parity, the wait for the slots' previous use, this rank's status word and arrival flag, on the root the wait for every rank
// and the `done` word, and the outcome, most specific first.  What differs between the two forms comes in as hooks:
//   prepare(es, slot_bytes)     host-side work before the slots' previous use is awaited: validation, planning, sizing, the
//                               pinned staging (no page-locked allocation may follow: see ExecSlot::kInitialPinned)
//   contribute(es, my_slot)     this rank's share, on es.stream, into its slot of the root's mailbox
//   collect(es)                 once the stream is synchronised: this rank's own device-side errors and counters
//   reduce(es, slots0, slot_bytes, settle, finalized)
//                               root only, enqueued behind the wait for every rank: combine and finalise into the result
//                               (finalized = it holds memory).  settle() synchronises and returns the first failure of any
//                               rank; a reduce that must not read a failed rank's slot calls it first
//   discard()                   frees the result when a later check fails
// pre_rc: a failure that already happened on this rank (its transient parts could not be admitted) -- the rank still takes
// part in the collective and reports it.
struct CollectiveHooks {
    std::function<int(ExecSlot &, size_t)> prepare;
    std::function<int(ExecSlot &, uint8_t *)> contribute;
    std::function<int(ExecSlot &)> collect;
    std::function<int(ExecSlot &, uint8_t *, size_t, const std::function<int()> &, bool &)> reduce;
    std::function<void()> discard;
};

static int run_collective(bydb_ctx *ctx, int32_t root, int pre_rc, const CollectiveHooks &h) {
    const std::string pre_msg = pre_rc ? g_last_error : std::string();
    Comm &cm = ctx->comm;
    std::lock_guard<std::mutex> lk(cm.mu);
    if (cm.nranks == 0) return fail(BYDB_EINVAL, "bydb_comm_connect was not called on this context");
    if (root < 0 || root >= cm.nranks) return fail(BYDB_EINVAL, "bad root");
    CUDA_TRY(cudaSetDevice(ctx->device));
    SlotLease lease(ctx);
    if (lease.init()) return fail(BYDB_EIO, "cannot create stream");
    ExecSlot &es = *lease.slot;
    cudaStream_t s = es.stream;
    // From here on this rank ALWAYS raises its arrival flag (with a status word in front of it), whatever fails on the
    // host side: the other ranks' calls must neither hang nor fall out of step (every rank counts the same epochs).
    const uint64_t epoch = ++cm.epoch;
    MailboxView mb = mailbox_view(cm, root, epoch);
    int rc = pre_rc ? fail(pre_rc, pre_msg) : h.prepare(es, mb.slot_bytes);
    // the slots' previous use -- the last collective with THIS root and parity, the same epoch on every rank -- must have been
    // consumed by the root (its `done` word only ever grows) before they are overwritten
    const uint64_t prev_use = mb.claim_slots();
    uint32_t host_perr = 0;  // outcome of the host-polled waits (shared-device mode)
    if (prev_use) {
        if (cm.shared_device) host_perr = comm_wait_host(cm, mb.done, 1, prev_use);
        else launch_comm_wait(mb.done, 1, prev_use, mb.my_err, kErrPeerTimeout, s);
    }
    if (!rc) rc = h.contribute(es, mb.my_slot);
    const std::string my_msg = rc ? g_last_error : std::string();
    const unsigned long long st_word = (epoch << 32) | static_cast<unsigned long long>(static_cast<uint32_t>(-rc));
    cudaMemcpyAsync(mb.status + cm.rank, &st_word, sizeof st_word, cudaMemcpyHostToDevice, s);  // pageable source: staged before the call returns
    launch_comm_signal(mb.flags + cm.rank, epoch, s);
    unsigned long long peer_status[kCommMaxRanks] = {0};
    const char *peer_msg = " failed on its side of the collective";
    bool finalized = false;
    int frc = 0;
    if (cm.rank == root) {
        // reduce: wait for every rank's share, then the form's own combine and finalisation
        if (cm.shared_device) {
            const uint32_t e2 = comm_wait_host(cm, mb.flags, static_cast<uint32_t>(cm.nranks), epoch);  // own flag included: own share is complete
            host_perr = host_perr ? host_perr : e2;
        } else {
            launch_comm_wait(mb.flags, static_cast<uint32_t>(cm.nranks), epoch, mb.my_err, kErrPeerTimeout, s);
        }
        const std::function<int()> settle = [&]() -> int {
            cudaStreamSynchronize(s);
            uint32_t e = 0;
            if (cudaMemcpy(&e, mb.my_err, sizeof e, cudaMemcpyDeviceToHost) != cudaSuccess || e == 0) e = host_perr;
            if (e) return fail(dev_err_code(e), dev_err_text(e));
            cudaMemcpy(peer_status, mb.status, sizeof(unsigned long long) * static_cast<size_t>(cm.nranks), cudaMemcpyDeviceToHost);
            return peer_failure(peer_status, cm.nranks, epoch, peer_msg);
        };
        if (!rc) frc = h.reduce(es, mb.slots0, mb.slot_bytes, settle, finalized);
        cudaStreamSynchronize(s);
        cudaMemcpy(peer_status, mb.status, sizeof(unsigned long long) * static_cast<size_t>(cm.nranks), cudaMemcpyDeviceToHost);
        // the slots of this parity are free again: nothing reads them any more
        cudaMemcpyAsync(mb.done, &epoch, sizeof epoch, cudaMemcpyHostToDevice, s);
    }
    cudaStreamSynchronize(s);
    uint32_t perr = 0;
    if (cudaMemcpy(&perr, mb.my_err, sizeof perr, cudaMemcpyDeviceToHost) == cudaSuccess && perr != 0) cudaMemset(mb.my_err, 0, sizeof perr);
    if (!perr) perr = host_perr;
    // ---- outcome, most specific first: this rank's own host-side failure, its device-side errors, a peer's failure
    if (rc) {
        if (finalized) h.discard();
        return fail(rc, my_msg);
    }
    int crc = h.collect(es);
    if (!crc && perr) crc = fail(dev_err_code(perr), dev_err_text(perr));
    if (!crc && cm.rank == root) {
        crc = peer_failure(peer_status, cm.nranks, epoch, peer_msg);
        if (!crc) crc = frc;
    }
    if (crc && finalized) h.discard();
    return crc;
}

// given: the parts to scan instead of q->parts (the host-buffer form); pre_rc: see run_collective
static int scan_reduce_impl(bydb_ctx *ctx, const bydb_query *q, const std::vector<std::shared_ptr<Part>> *given, int pre_rc, uint64_t h2d_pre, int32_t root,
                            bydb_result *out) {
    Plan plan;
    const TableLayout &tl = plan.tl;
    memset(&out->stats, 0, sizeof out->stats);
    out->stats.h2d_bytes = h2d_pre;
    CollectiveHooks h;
    h.prepare = [&](ExecSlot &es, size_t slot) -> int {
        int rc = validate_query(q, given == nullptr);
        if (!rc) rc = make_plan(ctx, q, given, plan);
        if (rc) return rc;
        if (tl.total > slot) return fail(BYDB_EINVAL, "partial table larger than the mailbox slots (bydb_comm_export max_table_bytes)");
        if (es.ensure_pinned(step_pinned_bytes(q, tl.G, tl.G))) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
        return 0;
    };
    // map: this rank's group_reduce writes the table straight into the root's memory (P2P stores over NVLink)
    h.contribute = [&](ExecSlot &es, uint8_t *my_slot) { return run_scan(ctx, q, plan, es, es.stream, my_slot, tl, &out->stats); };
    h.collect = [&](ExecSlot &es) { return collect_scan(es, &out->stats); };
    // reduce: combine the slots in rank order (deterministic float sums), finalise; a failed rank's status travels in its table
    h.reduce = [&](ExecSlot &es, uint8_t *slots0, size_t slot, const std::function<int()> &, bool &finalized) -> int {
        launch_combine_tables(slots0, static_cast<uint32_t>(ctx->comm.nranks), tl, es.stream, slot);
        out->stats.kernel_launches += 3;
        const int frc = finalize_to_host(q, plan, es, es.stream, slots0, tl, out, true);  // synchronises
        finalized = frc == 0;
        return frc;
    };
    h.discard = [&] { bydb_result_free(ctx, out); };
    return run_collective(ctx, root, pre_rc, h);
}

// A hash of what every rank of a keyed collective must pass alike: the whole query but its parts, and the group key.
static uint64_t keyed_fingerprint(const bydb_query *q, const bydb_group_key *key, uint32_t cap) {
    uint64_t h = 0xcbf29ce484222325ull;  // FNV-1a
    auto mix = [&](const void *p, size_t n) {
        const uint8_t *b = static_cast<const uint8_t *>(p);
        for (size_t i = 0; i < n; ++i) h = (h ^ b[i]) * 0x100000001b3ull;
    };
    auto mix_u64 = [&](uint64_t v) { mix(&v, sizeof v); };
    auto mix_str = [&](const char *s) {
        const size_t n = s ? strlen(s) : 0;
        mix_u64(n);
        mix(s, n);
    };
    mix_u64(q->n_series);
    mix(q->series_ids, q->n_series * 8);
    mix_u64(q->series_group ? static_cast<uint64_t>(static_cast<uint32_t>(q->n_groups)) : ~0ull);
    if (q->series_group) mix(q->series_group, q->n_series * 4);
    mix_u64(static_cast<uint64_t>(q->tmin));
    mix_u64(static_cast<uint64_t>(q->tmax));
    mix_u64(q->n_preds);
    for (uint32_t i = 0; i < q->n_preds; ++i) {
        const bydb_pred &p = q->preds[i];
        mix_str(p.family);
        mix_str(p.tag);
        mix_u64(static_cast<uint64_t>(p.op) << 32 | static_cast<uint32_t>(p.value_type));
        if (p.value_type == BYDB_VT_INT64) {
            mix_u64(static_cast<uint64_t>(p.lit_i64));
        } else {
            mix_u64(p.lit_len);
            mix(p.lit, p.lit_len);
        }
    }
    mix_u64(q->n_aggs);
    for (uint32_t a = 0; a < q->n_aggs; ++a) {
        mix_str(q->aggs[a].field);
        mix_u64(static_cast<uint64_t>(q->aggs[a].func));
    }
    mix_u64(static_cast<uint64_t>(static_cast<uint32_t>(q->top_n)) << 32 | static_cast<uint32_t>(q->top_agg));
    mix_u64(static_cast<uint64_t>(static_cast<uint32_t>(q->top_desc)) << 32 | q->flags);
    mix_str(key->family);
    mix_str(key->tag);
    mix_u64(static_cast<uint64_t>(cap) << 32 | key->value_type);
    return h;
}

// the slot of a rank of a keyed collective that found V key values
static KeyedSlot keyed_slot(const Plan &plan, size_t V) { return KeyedSlot(plan.tl.G, plan.tl.F, plan.n_series, V); }

int bydb_keyed_reduce_slot_bytes(const bydb_query *q, const bydb_group_key *key, uint64_t *out) {
    return guarded([&]() -> int {
    if (!q || !out) return fail(BYDB_EINVAL, "NULL argument");
    int rc = validate_query(q, false);
    uint32_t cap = 0;
    if (!rc) rc = check_group_key(q, key, cap);
    if (rc) return rc;
    Plan plan;
    rc = query_shape(q, plan);
    if (rc) return rc;
    *out = keyed_slot(plan, cap).total;
    return 0;
    });
}

// The keyed collective: discovery and the per-value passes of bydb_scan_agg_keyed on every rank, written into its slot of the
// root's mailbox (layout KeyedSlot); on the root the union of the values, the cross-rank span check, the union table and first
// appearances (key_union / rank_span_check / combine_keyed / merge_first kernels), then bydb_scan_agg_keyed's ordering and
// finalisation.
int bydb_scan_reduce_keyed(bydb_ctx *ctx, const bydb_query *q, const bydb_group_key *key, int32_t root, bydb_keyed_result *out) {
    return guarded([&]() -> int {
    if (!ctx || !out) return fail(BYDB_EINVAL, "ctx/out is NULL");
    memset(out, 0, sizeof *out);
    g_last_dev_err = 0;
    auto owner = new KeyedOwner();
    out->owner = owner;
    KeyedUndo undo{ctx, out};
    set_key_table(out, owner, {});
    bydb_stats &stats = out->base.stats;
    Plan plan;
    uint32_t cap = 0;
    KeyValues values;
    std::vector<uint8_t> header;
    KeyedSlot ks(0, 0, 0, 0);
    uint64_t fp = 0;
    CollectiveHooks h;
    h.prepare = [&](ExecSlot &es, size_t slot) -> int {
        int rc = validate_query(q, true);
        if (!rc) rc = check_group_key(q, key, cap);
        if (!rc) rc = make_plan(ctx, q, nullptr, plan);
        if (rc) return rc;
        if (parts_overlap(plan.parts, q->tmin, q->tmax))
            return fail(BYDB_ENOTSUP, "group-key query over parts of one rank that overlap in time (version dedup) is not supported on the device path");
        rc = discover_keys(ctx, q, key, cap, plan, es, &stats, values);
        if (rc) return rc;
        const size_t V = values.size(), G = static_cast<size_t>(plan.n_groups), F = plan.fcols.size();
        if (G * cap > 0x7fffffffull / std::max<size_t>(F, 1)) return fail(BYDB_ENOMEM, "group-key query: too many composite groups");
        ks = keyed_slot(plan, V);
        if (ks.total > slot)
            return fail(BYDB_EINVAL, "keyed collective: this rank's " + std::to_string(V) + " key values need " + std::to_string(ks.total) +
                                         " bytes, more than the mailbox slots (bydb_comm_export max_table_bytes, see bydb_keyed_reduce_slot_bytes)");
        // sized for the union (at most cap values) now: the root's finalisation may not allocate page-locked memory later
        if (es.ensure_pinned(step_pinned_bytes(q, G, G * cap))) return fail(BYDB_ENOMEM, "cudaMallocHost failed");
        fp = keyed_fingerprint(q, key, cap);
        header.assign(ks.off_vals + V * kMaxLit, 0);
        const uint32_t v32 = static_cast<uint32_t>(V);
        memcpy(header.data(), &fp, 8);
        memcpy(header.data() + 8, &v32, 4);
        for (size_t v = 0; v < V; ++v) {
            const uint32_t len = static_cast<uint32_t>(values[v].size());
            memcpy(header.data() + ks.off_lens + 4 * v, &len, 4);
            if (len) memcpy(header.data() + ks.off_vals + v * kMaxLit, values[v].data(), len);
        }
        return 0;
    };
    h.contribute = [&](ExecSlot &es, uint8_t *my_slot) -> int {
        const size_t V = values.size();
        if (V) {
            int rc = run_keyed_passes(ctx, q, key, plan, es, values, TableLayout(V * plan.n_groups, plan.fcols.size()), my_slot + ks.off_table,
                                      reinterpret_cast<int64_t *>(my_slot + ks.off_coltype), reinterpret_cast<int64_t *>(my_slot + ks.off_kts),
                                      reinterpret_cast<uint32_t *>(my_slot + ks.off_krow), reinterpret_cast<int64_t *>(my_slot + ks.off_span), &stats);
            if (rc) return rc;
        }
        CUDA_TRY(cudaMemcpyAsync(my_slot, header.data(), header.size(), cudaMemcpyHostToDevice, es.stream));  // pageable: staged before it returns
        return 0;
    };
    h.collect = [&](ExecSlot &) { return 0; };  // every pass was collected as it ran
    h.reduce = [&](ExecSlot &es, uint8_t *slots0, size_t slot, const std::function<int()> &settle, bool &) -> int {
        int rc = settle();  // a failed rank's slot holds nothing to read
        if (rc) return rc;
        cudaStream_t s = es.stream;
        const uint32_t R = static_cast<uint32_t>(ctx->comm.nranks);
        for (uint32_t r = 0; r < R; ++r) {
            uint64_t theirs = 0;
            CUDA_TRY(cudaMemcpy(&theirs, slots0 + r * slot, 8, cudaMemcpyDeviceToHost));
            if (theirs != fp)
                return fail(BYDB_EINVAL, "keyed collective: rank " + std::to_string(r) +
                                             " passed another query or group key (only the parts may differ between ranks)");
        }
        // ---- union of the ranks' values, cross-rank span check
        const size_t NS = q->n_series, G = static_cast<size_t>(plan.n_groups), F = plan.fcols.size();
        Carve carve;
        const size_t u_ctl = carve(16), u_vals = carve(static_cast<size_t>(cap) * kMaxLit), u_lens = carve(static_cast<size_t>(cap) * 4),
                     u_inv = carve(static_cast<size_t>(R) * cap * 4);
        const size_t back_bytes = u_inv - u_ctl;  // ctl | vals | lens come back in one copy
        Scratch us;
        CUDA_TRY(us.alloc(carve.o, s));
        CUDA_TRY(cudaMemsetAsync(us.base + u_ctl, 0, 8, s));
        CUDA_TRY(cudaMemsetAsync(us.base + u_ctl + 8, 0xff, 4, s));
        KeyedUnionParams up;
        memset(&up, 0, sizeof up);
        up.slots = slots0;
        up.slot_stride = slot;
        up.G = static_cast<uint32_t>(G);
        up.F = static_cast<uint32_t>(F);
        up.NS = static_cast<uint32_t>(NS);
        up.cap = cap;
        up.n_ranks = R;
        up.tmin = q->tmin;
        up.tmax = q->tmax;
        up.vals = us.base + u_vals;
        up.lens = reinterpret_cast<uint32_t *>(us.base + u_lens);
        up.inv = reinterpret_cast<int32_t *>(us.base + u_inv);
        up.ctl = reinterpret_cast<uint32_t *>(us.base + u_ctl);
        launch_key_union(up, s);
        CUDA_TRY(cudaMemcpyAsync(es.pinned, us.base + u_ctl, back_bytes, cudaMemcpyDeviceToHost, s));
        CUDA_TRY(cudaStreamSynchronize(s));
        CUDA_TRY(cudaGetLastError());
        stats.kernel_launches += NS && R > 1 ? 2 : 1;
        stats.d2h_bytes += back_bytes;
        const uint32_t *ctl = reinterpret_cast<const uint32_t *>(es.pinned);
        if (ctl[1] == kErrKeyCap)
            return fail(BYDB_ENOMEM, "keyed collective: more distinct key values over all ranks than bydb_group_key.max_values (" + std::to_string(cap) + ")");
        if (ctl[1] == kErrRankOverlap) {
            const uint32_t i = ctl[2];
            return fail(BYDB_ENOTSUP, "keyed collective: series #" + std::to_string(i) + " (id " + std::to_string(i < NS ? q->series_ids[i] : 0) +
                                          ") lives on several ranks over time spans that intersect");
        }
        const size_t V = std::min<size_t>(ctl[0], cap);
        KeyValues uvals(V);
        const uint32_t *hl = reinterpret_cast<const uint32_t *>(es.pinned + (u_lens - u_ctl));
        for (size_t u = 0; u < V; ++u) {
            const uint8_t *b = es.pinned + (u_vals - u_ctl) + u * kMaxLit;
            uvals[u].assign(b, b + std::min<uint32_t>(hl[u], kMaxLit));
        }
        set_key_table(out, owner, uvals);
        if (V == 0) return 0;  // no rank selected a block: no rows
        // ---- the ranks' tables, column types and first appearances folded into the union arrays
        const TableLayout tlu(V * G, F);
        carve = Carve();
        const size_t c_table = carve(tlu.total), c_ct = carve(V * F * 8), c_kts = carve(V * NS * 8), c_krow = carve(V * NS * 4);
        Scratch uc;
        CUDA_TRY(uc.alloc(carve.o, s));
        up.n_values = static_cast<uint32_t>(V);
        up.table = reinterpret_cast<uint64_t *>(uc.base + c_table);
        up.coltype = reinterpret_cast<int64_t *>(uc.base + c_ct);
        up.Kts = reinterpret_cast<int64_t *>(uc.base + c_kts);
        up.Krow = reinterpret_cast<uint32_t *>(uc.base + c_krow);
        launch_combine_keyed(up, s);
        stats.kernel_launches += NS ? 2 : 1;
        return keyed_finish(q, plan, es, V, uc.base + c_table, tlu, up.coltype, up.Kts, up.Krow, out, owner);
    };
    h.discard = [] {};  // the result of a failed call is freed by `undo`
    const int rc = run_collective(ctx, root, 0, h);
    if (rc) return rc;
    undo.done = true;
    return 0;
    });
}

int bydb_scan_reduce(bydb_ctx *ctx, const bydb_query *q, int32_t root, bydb_result *out) {
    return guarded([&]() -> int {
    if (!ctx || !out) return fail(BYDB_EINVAL, "ctx/out is NULL");
    memset(out, 0, sizeof *out);
    return scan_reduce_impl(ctx, q, nullptr, 0, 0, root, out);
    });
}

// The collective as a prepared query: from its second execution on (per root and slot parity) the rank's whole step -- argument
// refresh, wait for the slots, staging copy, block selection, scan, reduce into the root's mailbox, status + arrival flag, and on
// the root the wait for all ranks, combine, finalisation, row selection, `done` word and read-back -- is ONE captured CUDA graph:
// one launch and one synchronisation per call.  Semantics are bydb_scan_reduce's; ranks may mix the two freely.
int bydb_scan_reduce_prepared(bydb_ctx *ctx, bydb_prepared *p, int32_t root, bydb_result *out) {
    return guarded([&]() -> int {
    if (!ctx || !p || !out) return fail(BYDB_EINVAL, "NULL argument");
    memset(out, 0, sizeof *out);
    std::lock_guard<std::mutex> lkp(p->mu);
    Comm &cm = ctx->comm;
    if (cm.nranks == 0) return fail(BYDB_EINVAL, "bydb_comm_connect was not called on this context");
    if (root < 0 || root >= cm.nranks) return fail(BYDB_EINVAL, "bad root");
    CUDA_TRY(cudaSetDevice(ctx->device));
    g_last_dev_err = 0;
    const uint64_t run = p->reduce_runs++;
    if (run == 0 || !p->reduce_capturable || cm.shared_device) return scan_reduce_impl(ctx, &p->q, nullptr, 0, 0, root, out);
    std::unique_lock<std::mutex> lk(cm.mu);
    const uint64_t epoch = cm.epoch + 1;
    MailboxView mb = mailbox_view(cm, root, epoch);  // its slots are claimed only when the graph replays
    CommArgs *d_args = reinterpret_cast<CommArgs *>(cm.mine + kCommArgsOff);
    ExecSlot &es = *p->slot;
    // pinned words of this prepared query that the graph's memcpy nodes read / write: the last two zero pages of its slot
    CommArgs *h_args = reinterpret_cast<CommArgs *>(es.page(7));
    uint8_t *h_back = reinterpret_cast<uint8_t *>(es.page(6));  // [0,4) this rank's wait-kernel error word, [8, 8 + 8 * nranks) the status words (root)
    if (static_cast<size_t>(cm.nranks) * 8 + 8 > kZeroPageBytes) {  // more ranks than the pinned read-back page holds status words for
        lk.unlock();
        return scan_reduce_impl(ctx, &p->q, nullptr, 0, 0, root, out);
    }
    auto &rg = p->reduce_graphs[root * 2 + static_cast<int>(mb.parity)];
    // a graph reads its parts through the pointers captured with it (same rule as bydb_scan_agg_prepared)
    if (rg.exec) (void)check_held_parts(ctx, p->parts, rg.exec, rg.held);  // a missing part fails in make_plan below
    if (!rg.exec) {
        Plan plan;
        int rc = make_plan(ctx, &p->q, nullptr, plan);
        if (rc) {
            lk.unlock();
            return scan_reduce_impl(ctx, &p->q, nullptr, 0, 0, root, out);  // takes part in the collective and reports the failure
        }
        const TableLayout &tl = plan.tl;
        p->host_off = stage_layout(p->q.n_series, tl.G).stride;
        // the version-dedup precheck synchronises: such queries keep the plain path
        if (parts_overlap(plan.parts, p->q.tmin, p->q.tmax) || tl.total > mb.slot_bytes || es.ensure_pinned(step_pinned_bytes(&p->q, tl.G, tl.G))) {
            p->reduce_capturable = false;
            lk.unlock();
            return scan_reduce_impl(ctx, &p->q, nullptr, 0, 0, root, out);
        }
        memset(&rg.captured, 0, sizeof rg.captured);
        cudaStream_t s = es.stream;
        cudaGetLastError();  // a stale error of an earlier call must not be blamed on the capture
        cudaError_t e = cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
        const char *bad_step = nullptr;  // first step of the capture the runtime objected to (BYDB_TRACE prints it)
        if (e == cudaSuccess) {
            Scratch fin;
            auto step = [&](const char *name, bool good) {
                const cudaError_t le = cudaGetLastError();
                if ((!good || le != cudaSuccess) && !bad_step) {
                    bad_step = name;
                    if (le != cudaSuccess) e = le;
                }
            };
            step("args copy", cudaMemcpyAsync(d_args, h_args, sizeof(CommArgs), cudaMemcpyHostToDevice, s) == cudaSuccess);
            launch_comm_wait_args(mb.done, 1, d_args, 1, mb.my_err, kErrPeerTimeout, s);
            step("wait for the slots", true);
            step("scan", run_scan(ctx, &p->q, plan, es, s, mb.my_slot, tl, &rg.captured) == 0);
            rg.express = es.express[0];
            launch_comm_signal_args(mb.flags + cm.rank, mb.status + cm.rank, d_args, s);
            step("signal", true);
            if (cm.rank == root) {
                launch_comm_wait_args(mb.flags, static_cast<uint32_t>(cm.nranks), d_args, 0, mb.my_err, kErrPeerTimeout, s);
                step("wait for the ranks", true);
                launch_combine_tables(mb.slots0, static_cast<uint32_t>(cm.nranks), tl, s, mb.slot_bytes);
                step("combine", true);
                uint32_t fin_launches = 0;
                step("finalize", finalize_enqueue(&p->q, plan, es, s, mb.slots0, tl, p->host_off, fin, rg.fl, fin_launches) == 0);
                launch_comm_done_args(mb.done, d_args, s);
                step("done word", true);
                step("status read-back",
                     cudaMemcpyAsync(h_back + 8, mb.status, sizeof(unsigned long long) * static_cast<size_t>(cm.nranks), cudaMemcpyDeviceToHost, s) == cudaSuccess);
                rg.captured.kernel_launches += 3 + fin_launches;
            }
            step("error read-back", cudaMemcpyAsync(h_back, mb.my_err, sizeof(uint32_t), cudaMemcpyDeviceToHost, s) == cudaSuccess);
            rg.captured.kernel_launches += 2;
        }
        cudaGraph_t graph = nullptr;
        if (e == cudaSuccess || bad_step) {
            const cudaError_t ee = cudaStreamEndCapture(s, &graph);  // always leave capture mode
            if (!bad_step && ee != cudaSuccess) {
                bad_step = "end capture";
                e = ee;
            }
        }
        if (!bad_step && graph) {
            e = cudaGraphInstantiate(&rg.exec, graph, 0);
            if (e != cudaSuccess) bad_step = "instantiate";
        }
        if (graph) cudaGraphDestroy(graph);
        if (bad_step || !rg.exec) {
            static const bool trace = getenv("BYDB_TRACE") != nullptr;
            if (trace) fprintf(stderr, "[bydb] prepared collective: capture failed at '%s' (%s); keeping the plain path\n", bad_step ? bad_step : "?", cudaGetErrorString(e));
            cudaGetLastError();
            if (rg.exec) cudaGraphExecDestroy(rg.exec);
            rg.exec = nullptr;
            p->reduce_capturable = false;  // the plain path from here on
            lk.unlock();
            return scan_reduce_impl(ctx, &p->q, nullptr, 0, 0, root, out);
        }
        rg.held = plan.parts;
    }
    // ---- replay
    cm.epoch = epoch;
    h_args->epoch = epoch;
    h_args->prev_use = mb.claim_slots();
    memset(h_back, 0, kZeroPageBytes);
    memset(es.page(0), 0, kZeroPageBytes);
    const int rc = replay_graph(rg.exec, es, p->t0, p->t1, rg.captured, rg.express, &out->stats);
    const uint32_t perr = *reinterpret_cast<const uint32_t *>(h_back);
    if (perr != 0) cudaMemset(mb.my_err, 0, sizeof perr);
    if (rc) return rc;
    if (perr != 0) return fail(dev_err_code(perr), dev_err_text(perr));
    if (cm.rank != root) return 0;
    const int prc = peer_failure(reinterpret_cast<const unsigned long long *>(h_back + 8), cm.nranks, epoch, " failed before its scan");
    if (prc) return prc;
    return finalize_parse(es.pinned + p->host_off, rg.fl, true, out);
    });
}

// The collective with HOST file images on every rank (the end-to-end form of a cold distributed query): each rank's parts
// are admitted for the duration of the call (BYDB_Q_HOST_ZERO_COPY: directory upload only, pages pulled over PCIe by the
// scan), scanned into the root's mailbox and dropped.  q->parts / q->n_parts are ignored.
int bydb_scan_reduce_host(bydb_ctx *ctx, uint32_t n_parts, const bydb_part_files *parts, const bydb_query *q, int32_t root, bydb_result *out) {
    return guarded([&]() -> int {
    if (!ctx || !out) return fail(BYDB_EINVAL, "ctx/out is NULL");
    memset(out, 0, sizeof *out);
    CUDA_TRY(cudaSetDevice(ctx->device));
    g_last_dev_err = 0;
    TransientParts tmp(ctx);
    uint64_t h2d = 0;
    int rc = validate_query(q, false);
    if (!rc && (n_parts == 0 || !parts || n_parts > kMaxParts)) rc = fail(BYDB_EINVAL, "need 1..64 host parts");
    AdmitOptions opt;
    opt.zero_copy = !rc && (q->flags & BYDB_Q_HOST_ZERO_COPY) != 0;
    opt.unpack = !opt.zero_copy;  // fallback pages are unpacked up front here: a collective cannot be re-run by one rank alone
    for (uint32_t i = 0; i < n_parts && !rc; ++i) rc = tmp.admit(&parts[i], &h2d, opt);
    rc = scan_reduce_impl(ctx, q, &tmp.parts, rc, h2d, root, out);
    if (!rc && opt.zero_copy) out->stats.h2d_bytes += out->stats.page_bytes;  // pages were read in place over PCIe
    return rc;
    });
}

}  // extern "C"
