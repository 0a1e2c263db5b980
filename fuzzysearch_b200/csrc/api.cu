// api.cu -- host side of libfuzzb200.so: the C-ABI declared in include/fuzzb200.h.
//
// No CPU search path exists in this file: every search launches the sm_90a kernels of kernels.cuh
// and fails with FZB_E_CUDA when no device is usable.  The only host-side algorithm is the
// O(N log N) consolidation of the (small) match list, which the reference also performs after its
// search (common.py:185-189).
#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cmath>
#include <cstring>
#include <dlfcn.h>
#include <sched.h>
#include <unistd.h>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <thread>
#include <new>
#include <string>
#include <type_traits>
#include <vector>

#include "kernels.cuh"
#include "ham_kernels.cuh"
#include "lp_kernels.cuh"
#include "post_kernels.cuh"
#include "p2p_kernels.cuh"
#include "batch_kernels.cuh"
#include "ham_batch_kernels.cuh"
#include "generic_batch_kernels.cuh"
#include "best_kernels.cuh"
#include "nearest_kernels.cuh"
#include "sym_kernels.cuh"
#include "align_kernels.cuh"
#include <unordered_map>
#include "debug_kernels.cuh"

using namespace fzb;

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_err;

static int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}

#define CK(call)                                                                          \
    do {                                                                                  \
        cudaError_t e_ = (call);                                                          \
        if (e_ != cudaSuccess)                                                            \
            return fail(FZB_E_CUDA, "%s failed: %s", #call, cudaGetErrorString(e_));      \
    } while (0)

#define TRY(call)                                                                         \
    do {                                                                                  \
        const int rc_ = (call);                                                           \
        if (rc_) return rc_;                                                              \
    } while (0)

// ------------------------------------------------------------------------------------------------
// owned allocations
// ------------------------------------------------------------------------------------------------
enum class Mem { Device, Pinned, Mapped };  // cudaMalloc; cudaHostAlloc, page-locked; ... and mapped for the device

// One device or pinned host allocation of size() elements of T, freed (cudaFree / cudaFreeHost) when the object dies
// or takes another allocation.  alloc() allocates into a temporary and replaces the current allocation only on
// success: a failed allocation or growth leaves the object, and whatever holds it, as it was.
template <class T, Mem kMem>
class Buf {
  public:
    Buf() = default;
    Buf(Buf &&o) noexcept : p_(o.p_), n_(o.n_) {
        o.p_ = nullptr;
        o.n_ = 0;
    }
    Buf &operator=(Buf o) noexcept {  // (`o` takes the previous allocation with it)
        std::swap(p_, o.p_);
        std::swap(n_, o.n_);
        return *this;
    }
    ~Buf() {
        if (p_) (void)(kMem == Mem::Device ? cudaFree(p_) : cudaFreeHost(p_));
    }
    T *get() const { return p_; }
    uint64_t size() const { return n_; }
    explicit operator bool() const { return p_ != nullptr; }
    T &operator[](uint64_t i) const {
        static_assert(kMem != Mem::Device, "device memory is not addressable from the host");
        return p_[i];
    }
    // n elements; `bytes` instead of n * sizeof(T) when the allocation also holds a trailing array of another type
    int alloc(uint64_t n, uint64_t bytes = 0) {
        Buf b;
        if (!bytes) bytes = n * sizeof(T);
        const unsigned flags = kMem == Mem::Mapped ? cudaHostAllocMapped | cudaHostAllocPortable : cudaHostAllocDefault;
        const cudaError_t e = kMem == Mem::Device ? cudaMalloc(&b.p_, bytes) : cudaHostAlloc(&b.p_, bytes, flags);
        if (e != cudaSuccess)
            return fail(FZB_E_CUDA, "%s(%llu bytes) failed: %s", kMem == Mem::Device ? "cudaMalloc" : "cudaHostAlloc",
                        (unsigned long long)bytes, cudaGetErrorString(e));
        b.n_ = n;
        *this = std::move(b);
        return FZB_OK;
    }

  private:
    T *p_ = nullptr;
    uint64_t n_ = 0;
};
template <class T> using DevBuf = Buf<T, Mem::Device>;
template <class T> using PinnedBuf = Buf<T, Mem::Pinned>;
template <class T> using MappedBuf = Buf<T, Mem::Mapped>;

// The buffer groups a handle allocates on first use, each built whole or not at all (ensure_group).
struct BatchBufs {  // the tables of the shared batch passes (batch_kernels.cuh, ham_batch_kernels.cuh)
    DevBuf<uint32_t> d_mbits;  // first + second level key tables
    DevBuf<uint2> d_gtab;
    DevBuf<uint32_t> d_postings, d_pinfo;
    DevBuf<BatchPat> d_bpats;
    DevBuf<unsigned long long> d_mset;  // (pattern, granule) set of the q-sample pass: all-zero between passes
    DevBuf<WorkItem> d_mwork;
};
struct LpBatchBufs {  // the LP batch pass
    DevBuf<ulonglong2> d_lmlut;           // per-byte pattern-set vectors [256], then the match masks u32 [64][256]
    DevBuf<unsigned long long> d_lmlist;  // survivor list (after the sort: grouped by pattern)
    DevBuf<unsigned long long> d_lmkept;  // the survivors of the exact per-pattern window test
    DevBuf<uint32_t> d_lmhist;            // per-pattern counts [64] + kept total [1] | cursors [64]
};
struct GenericBatchBufs {  // the generic batch passes (generic_batch_kernels.cuh)
    DevBuf<uint32_t> d_glim;  // per pattern of a pass: max_subs | max_ins << 8 | max_dels << 16
};
struct PeerBufs {  // the peer-memory reduction (p2p_kernels.cuh)
    DevBuf<uint8_t> d_p2p;  // my receive area: [2 parities][world] slots + flags
    DevBuf<MergeScratch> d_ms;
    DevBuf<unsigned long long> d_mscore;
    DevBuf<uint32_t> d_mpos;
    MappedBuf<int64_t> h_grows;  // global final rows of the last global search (16 bytes each)
    MappedBuf<uint32_t> h_ghdr;  // status, count, epoch
};
struct RecBufs {  // a record set (fzb_haystack_set_records, DESIGN.md section 5.10)
    DevBuf<uint64_t> d_off;    // the count + 1 record offsets
    DevBuf<uint32_t> d_first;  // per 64-byte granule: the record holding its first position (k_rec_first)
    uint64_t longest = 0;      // positions of the longest record, its separator included
};
struct BestBufs {  // fzb_best_per_record (best_kernels.cuh)
    DevBuf<uint64_t> d_words;  // best[records], then top2[records]
    DevBuf<uint32_t> d_ids;    // the pattern ordinals of the pass being reduced
};
// The sink of the batches fzb_best_per_record runs (DESIGN.md section 5.13): they reduce the raw records of every pass
// and of every one-by-one search into these words instead of returning lists.
struct BestState {
    uint64_t *best, *top2;    // one word per record each
    const uint32_t *ordinal;  // pattern i of the batch being run is pattern ordinal[i] of the call
};
struct NearBufs {  // the nearest calls, single and batch (nearest_kernels.cuh)
    DevBuf<uint32_t> d_lanes;  // batches: m | ordinal << 16 per lane of every group
    DevBuf<uint8_t> d_pats;    // batches: kNearBatchMaxM bytes per lane
    DevBuf<uint64_t> d_words;  // the answer: the whole-sequence result (2 words), one word per record or per pattern,
                               // or best[records] then top2[records]
    DevBuf<uint64_t> d_scan;   // the symbols read, the partials of kNearMaxGrid CTAs, then a long pattern's record words
    uint64_t *steps() const { return d_scan.get(); }
    uint64_t *partials() const { return d_scan.get() + 1; }
    uint64_t *rec_words() const { return d_scan.get() + 1 + 2 * (uint64_t)kNearMaxGrid; }
};
struct GatherBufs {  // the staged NCCL all-gather
    uint32_t cap = 0;  // rows per rank
    DevBuf<int64_t> d_send, d_recv;
    PinnedBuf<int64_t> h_send, h_recv;
};

// Gives `slot` its group unless it has one.  `init` allocates and sets up the whole group in a local, which `slot`
// takes only when all of it succeeded: a failure leaves the slot empty, never holding part of a group.
template <class G, class F>
static int ensure_group(std::unique_ptr<G> &slot, F init) {
    if (slot) return FZB_OK;
    std::unique_ptr<G> g(new (std::nothrow) G());
    if (!g) return fail(FZB_E_CUDA, "out of host memory");
    TRY(init(*g));
    slot = std::move(g);
    return FZB_OK;
}

extern "C" int fzb_version(void) { return FZB_VERSION; }

extern "C" int fzb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

extern "C" const char *fzb_last_error(void) { return g_err.c_str(); }

// ------------------------------------------------------------------------------------------------
// NCCL, resolved at run time (the process usually has torch's libnccl.so.2 loaded already)
// ------------------------------------------------------------------------------------------------
struct NcclId {
    char b[FZB_NCCL_ID_BYTES];
};
struct NcclApi {
    int (*GetUniqueId)(NcclId *id) = nullptr;
    int (*CommInitRank)(void **comm, int nranks, NcclId id, int rank) = nullptr;  // ncclUniqueId is passed by value
    int (*AllGather)(const void *send, void *recv, size_t count, int dtype, void *comm, cudaStream_t s) = nullptr;
    int (*CommDestroy)(void *comm) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    bool ok = false;
};
static NcclApi g_nccl;
static std::string g_nccl_path;  // optional explicit library path (fzb_nccl_set_library)

extern "C" void fzb_nccl_set_library(const char *path) { g_nccl_path = path ? path : ""; }

static int nccl_load() {
    static std::once_flag once;
    std::call_once(once, [] {
        void *lib = nullptr;
        if (!g_nccl_path.empty()) lib = dlopen(g_nccl_path.c_str(), RTLD_NOW | RTLD_GLOBAL);
        if (!lib) lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!lib) return;
        *(void **)&g_nccl.GetUniqueId = dlsym(lib, "ncclGetUniqueId");
        *(void **)&g_nccl.CommInitRank = dlsym(lib, "ncclCommInitRank");
        *(void **)&g_nccl.AllGather = dlsym(lib, "ncclAllGather");
        *(void **)&g_nccl.CommDestroy = dlsym(lib, "ncclCommDestroy");
        *(void **)&g_nccl.GetErrorString = dlsym(lib, "ncclGetErrorString");
        g_nccl.ok = g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.AllGather && g_nccl.CommDestroy;
    });
    return g_nccl.ok ? FZB_OK : fail(FZB_E_CUDA, "libnccl.so.2 not available: %s", dlerror() ? dlerror() : "missing symbols");
}

static void nccl_comm_destroy(void *comm) {
    if (g_nccl.ok && comm) g_nccl.CommDestroy(comm);
}

#define NCCLCK(call)                                                                                      \
    do {                                                                                                  \
        int r_ = (call);                                                                                  \
        if (r_ != 0)                                                                                      \
            return fail(FZB_E_CUDA, "%s failed: %s", #call, g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "?"); \
    } while (0)

// ------------------------------------------------------------------------------------------------
// handles
// ------------------------------------------------------------------------------------------------
struct fzb_haystack {
    std::recursive_mutex mu;  // one search / upload at a time per handle (HandleLock); recursive: has_near_match and
                              // the windowed exact search call the search entry points on their own handle
    int device = 0;
    // Every buffer below is freed with the handle (fzb_haystack_destroy makes its device current first).
    uint8_t *d = nullptr;       // H[0] == global position buf_lo: owned_buf's bytes, an adopted buffer or a view
    DevBuf<uint8_t> owned_buf;  // the handle's own sequence buffer (size(): its capacity); empty when adopted
    uint64_t buf_len = 0, buf_lo = 0, global_len = 0, own_lo = 0, own_hi = 0;
    uint64_t padded_len = 0;
    cudaEvent_t ev_stop = nullptr;
    cudaStream_t stream = nullptr;
    DevBuf<uint32_t> d_bitmap;
    DevBuf<RawRec> d_out;  // size() raw records, then their size() packed keys (alloc_out)
    DevBuf<uint32_t> d_counters;
    // k_post writes these straight into MAPPED pinned host memory (no copy operations per search)
    MappedBuf<uint32_t> h_counters;  // CNT_COUNT counters
    MappedBuf<int64_t> h_fin;        // final rows (kPostMax x kFinCols)
    DevBuf<int64_t> d_fin;           // device copy of the final rows (input of the multi-GPU reduction)
    DevBuf<uint64_t> d_sorted;       // k_post scratch: the sorted canonical keys
    fzb_result *pending = nullptr;   // the last result, while its raw records still sit in d_out only
    bool ev1_recorded = false;
    bool filter_attrs_set = false;
    int scan_per_sm = 0;      // resident k_filter_sampled CTAs per SM (asked once, after set_filter_attrs)
    double coll_prob = -1.0;  // sum_c p_c^2 of the byte distribution (sampled lazily; < 0 = unknown)
    // multi-GPU reduction (FZB_F_GLOBAL): peer-memory world (p2p_kernels.cuh) + NCCL for bootstrap / staged fallback
    bool p2p = false;               // every rank of the world can store into every other rank's receive area
    bool local_world = false;       // the world lives in this process (fzb_comm_init_local): no NCCL
    std::unique_ptr<PeerBufs> peer;  // allocated when the handle joins a world (p2p_alloc)
    uint8_t *peer_base[kMaxWorld] = {};
    bool peer_opened[kMaxWorld] = {};
    uint32_t p2p_cap = 4096;        // group rows per slot
    uint64_t slot_bytes = 0, flags_off = 0;
    uint32_t epoch = 0;             // number of FZB_F_GLOBAL searches issued on this handle
    bool counters_clean = false;    // the device counters are all zero (the last search's final kernel left them so)
    uint32_t seq = 0;               // number of search attempts enqueued: the last kernel of each writes it to mapped
                                    // memory as its final store and the host polls for it (wait_done)
    void *comm = nullptr;  // ncclComm_t
    int rank = 0, world = 1;
    uint32_t gather_cap = 4096;     // rows per rank in one all-gather slot
    std::unique_ptr<GatherBufs> gather;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
    int sm_count = 132;
    DevBuf<uint64_t> d_hits;        // dense route: list of confirmed n-gram hits (allocated on first use)
    DevBuf<uint32_t> d_glist;       // compacted list of marked granules
    uint32_t glist_cap = 0;         // (d_glist has max(glist_cap, 1) entries)
    DevBuf<uint32_t> d_scratch;     // candidate lists of the LP / generic kernels
    DevBuf<unsigned long long> d_lplist;  // streaming LP route: starts that survived the scan (allocated on first use)
    // single-pass multi-pattern batches (batch_kernels.cuh), allocated on first use
    std::unique_ptr<BatchBufs> batch;
    DevBuf<unsigned long long> d_mhits;  // dense batch pass: (pattern, n-gram, position) hits
    std::unique_ptr<LpBatchBufs> lpb;
    std::unique_ptr<GenericBatchBufs> gbatch;
    std::unique_ptr<RecBufs> recs;  // the record set, if any (cleared by every upload)
    std::unique_ptr<BestBufs> bestb;
    std::unique_ptr<NearBufs> nearb;
};

struct fzb_result {
    std::vector<RawRec> raw;      // filled lazily from the owner's mapped staging buffer (fetch_raw)
    uint32_t raw_n = 0;           // number of raw records
    fzb_haystack *owner = nullptr;  // non-null while raw records / global rows still sit in the owner's mapped buffers
    bool raw_in_stage = false;
    void fetch_raw();
    void discard_attempt();
    std::vector<RawRec> fin;
    std::vector<int64_t> hulls;  // (hull_start, hull_end) of the group behind each final match
    bool unconsolidated = false;  // exact / Hamming routes: FINAL is the whole raw list in (start, end, dist) order
    bool have_fin = false;        // fin / hulls are filled
    bool device_post = false;  // the final list came from the device (k_post)
    bool raw_ordered = false;  // raw is already in its reference order
    bool has_global = false;   // FZB_F_GLOBAL: gfin is the global consolidated list of all shards
    bool global_on_device = false;  // ... produced by k_merge; its rows sit in owner->peer->h_grows until fetched
    bool fused_issued = false;      // a k_push / k_merge pair ran for this search
    uint32_t fused_status = 0;      // MS_* of that merge
    uint32_t gcount = 0;
    std::vector<RawRec> gfin;
    int raw_order = 0;         // 0 generation (ngram, idx) / 1 canonical / 2 generic n-grams (5 fields)
    void order_raw();
    fzb_stats stats{};
};

static uint64_t round_up(uint64_t x, uint64_t a) { return (x + a - 1) / a * a; }

static RawRec make_rec(int64_t start, int64_t end, int64_t dist) {  // a match without an anchor
    RawRec r;
    r.start = start;
    r.end = end;
    r.dist = (int32_t)dist;
    r.idx = -1;
    r.ngram = -1;
    return r;
}

// Every entry point that touches a handle's device state (buffer, counters, output area, stream order) holds the
// handle's mutex for the whole call: two threads sharing one resident sequence take turns, like callers of the
// reference under the GIL.  (Results are separate objects; their lazy raw fetch is guarded by g_pending_mutex.)
struct HandleLock {
    std::recursive_mutex *m;
    explicit HandleLock(fzb_haystack *h) : m(h ? &h->mu : nullptr) {
        if (m) m->lock();
    }
    ~HandleLock() {
        if (m) m->unlock();
    }
    HandleLock(const HandleLock &) = delete;
    HandleLock &operator=(const HandleLock &) = delete;
};

// The raw records of the LAST search of a handle stay in its DEVICE output buffer (and the global rows of a
// multi-GPU search in its mapped host buffer) until somebody asks for them (fzb_result_copy), the next search
// on the handle is about to overwrite the buffers, or the handle / the result dies: find_near_matches() only
// needs the consolidated list, and shipping 200 KB of raw records over PCIe behind every search is 1-2 % of a
// 4 GiB scan.  One process-wide mutex guards the result <-> handle link.
static std::mutex g_pending_mutex;

void fzb_result::fetch_raw() {
    std::lock_guard<std::mutex> lock(g_pending_mutex);
    if (!owner) return;
    if (raw_in_stage) {  // the records are still in the owner's device buffer: one D2H copy, now
        raw.resize(raw_n);
        if (raw_n) {
            cudaSetDevice(owner->device);
            if (cudaMemcpyAsync(raw.data(), owner->d_out.get(), (size_t)raw_n * sizeof(RawRec), cudaMemcpyDeviceToHost,
                                owner->stream) != cudaSuccess ||
                cudaStreamSynchronize(owner->stream) != cudaSuccess) {
                cudaGetLastError();
                raw.clear();  // (the handle's context is gone: nothing left to fetch)
                raw_n = 0;
            }
        }
        raw_in_stage = false;
    }
    if (global_on_device) {  // rows: start, (end - start) << 32 | dist
        gfin.resize(gcount);
        for (uint32_t i = 0; i < gcount; i++) {
            const int64_t s0 = owner->peer->h_grows[2 * (size_t)i], v = owner->peer->h_grows[2 * (size_t)i + 1];
            gfin[i] = make_rec(s0, s0 + (v >> 32), v & 0xFFFFFFFF);
        }
        global_on_device = false;
    }
    owner->pending = nullptr;
    owner = nullptr;
}

void fzb_result::discard_attempt() {  // a search attempt that has to be redone: unlink and drop its matches
    fetch_raw();
    raw.clear();
    raw_n = 0;
    fin.clear();
}

static void detach_pending(fzb_haystack *h) {  // before h->d_out / h->peer->h_grows are overwritten or freed
    fzb_result *r;
    {
        std::lock_guard<std::mutex> lock(g_pending_mutex);
        r = h->pending;
    }
    if (r) r->fetch_raw();
}

// d_out: `cap` raw records, then their `cap` packed canonical keys (k_post)
static int alloc_out(fzb_haystack *h, uint64_t cap) { return h->d_out.alloc(cap, cap * (sizeof(RawRec) + sizeof(uint64_t))); }

static int haystack_common_init(fzb_haystack *h) {
    CK(cudaSetDevice(h->device));
    CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    for (auto &e : h->ev) CK(cudaEventCreate(&e));
    CK(cudaEventCreate(&h->ev_stop));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, h->device));
    h->sm_count = prop.multiProcessorCount;
    uint64_t granules = (h->padded_len >> kGranuleShift) + 2;
    TRY(h->d_bitmap.alloc(round_up((granules + 31) / 32, 32)));
    TRY(h->d_counters.alloc(CNT_COUNT));
    TRY(h->h_counters.alloc(CNT_COUNT));
    memset(h->h_counters.get(), 0, CNT_COUNT * sizeof(uint32_t));  // the sequence word the host polls must not hold a stale value
    TRY(h->h_fin.alloc((uint64_t)kPostMax * kFinCols));
    TRY(h->d_fin.alloc((uint64_t)kPostMax * kFinCols));
    TRY(h->d_sorted.alloc(kPostMax));
    CK(cudaFuncSetAttribute(k_post, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPostSmem));
    CK(cudaMemset(h->d_bitmap.get(), 0, h->d_bitmap.size() * sizeof(uint32_t)));  // stays all-zero between searches
    h->glist_cap = (uint32_t)std::min<uint64_t>(granules, 1u << 20);
    TRY(h->d_glist.alloc(std::max<uint32_t>(h->glist_cap, 1)));
    return alloc_out(h, 1u << 16);
}

static int check_shard(uint64_t buf_len, uint64_t buf_lo, uint64_t global_len, uint64_t own_lo,
                       uint64_t own_hi) {
    // k_post's canonical keys and k_merge's winner scores hold a position in 46 bits; the LP route's empty match
    // (N, N, m) is one of them, so N itself must fit
    if (global_len >= (1ull << 46)) return fail(FZB_E_INVALID, "global_len must be below 2^46");
    if (buf_lo > global_len || buf_len > global_len - buf_lo || own_lo > own_hi || own_hi > global_len ||
        (own_lo < own_hi && (own_lo < buf_lo || own_hi > buf_lo + buf_len)))
        return fail(FZB_E_INVALID, "inconsistent shard geometry");
    if (buf_lo % 16 != 0) return fail(FZB_E_INVALID, "buf_lo must be a multiple of 16");
    // the batch passes pack buffer-relative positions into 40 bits (MdenseParams::hits, LpMultiParams::list)
    if (buf_len >= (1ull << 40)) return fail(FZB_E_INVALID, "buf_len must be below 2^40");
    return FZB_OK;
}

static int alloc_buffer(fzb_haystack *h) {
    CK(cudaSetDevice(h->device));
    TRY(h->owned_buf.alloc(h->padded_len));
    h->d = h->owned_buf.get();
    CK(cudaMemset(h->d + h->buf_len, 0, h->padded_len - h->buf_len));
    return FZB_OK;
}

static void close_peers(fzb_haystack *h);
static int upload_bytes(fzb_haystack *h, uint64_t dst_off, const uint8_t *host, uint64_t n);

extern "C" void fzb_haystack_destroy(fzb_haystack *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    detach_pending(h);
    if (h->comm) nccl_comm_destroy(h->comm);
    close_peers(h);
    for (auto &e : h->ev)
        if (e) cudaEventDestroy(e);
    if (h->ev_stop) cudaEventDestroy(h->ev_stop);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;  // (frees its buffers, on the device made current above)
}

// The constructors' common part.  `arg_error`: the caller's own argument check failed (reported after the `out`
// check).  `dev_ptr` non-null adopts that caller-owned buffer, otherwise the handle allocates its own and uploads
// `host` into it, if given.
static int haystack_new(const char *arg_error, const uint8_t *host, const void *dev_ptr, uint64_t buf_len,
                        uint64_t buf_lo, uint64_t global_len, uint64_t own_lo, uint64_t own_hi, int device,
                        fzb_haystack **out) {
    if (!out) return fail(FZB_E_INVALID, "out is NULL");
    *out = nullptr;
    if (arg_error) return fail(FZB_E_INVALID, "%s", arg_error);
    int rc = check_shard(buf_len, buf_lo, global_len, own_lo, own_hi);
    if (rc) return rc;
    if (fzb_device_count() <= device || device < 0)
        return fail(FZB_E_CUDA, "CUDA device %d not available (%d devices)", device, fzb_device_count());
    fzb_haystack *h = new (std::nothrow) fzb_haystack();
    if (!h) return fail(FZB_E_CUDA, "out of host memory");
    h->device = device;
    h->d = (uint8_t *)dev_ptr;
    h->buf_len = buf_len;
    h->buf_lo = buf_lo;
    h->global_len = global_len;
    h->own_lo = own_lo;
    h->own_hi = own_hi;
    h->padded_len = round_up(buf_len, 128) + 128;
    rc = dev_ptr ? FZB_OK : alloc_buffer(h);
    if (rc == FZB_OK) rc = haystack_common_init(h);
    if (rc == FZB_OK && host) rc = upload_bytes(h, 0, host, buf_len);
    if (rc) {
        fzb_haystack_destroy(h);
        return rc;
    }
    *out = h;
    return FZB_OK;
}

extern "C" int fzb_haystack_create_shard(const uint8_t *host, uint64_t buf_len, uint64_t buf_lo,
                                         uint64_t global_len, uint64_t own_lo, uint64_t own_hi,
                                         int device, fzb_haystack **out) {
    return haystack_new(!host && buf_len ? "host buffer is NULL" : nullptr, host, nullptr, buf_len, buf_lo,
                        global_len, own_lo, own_hi, device, out);
}

extern "C" int fzb_haystack_create(const uint8_t *host, uint64_t n, int device, fzb_haystack **out) {
    return fzb_haystack_create_shard(host, n, 0, n, 0, n, device, out);
}

extern "C" int fzb_haystack_adopt_device(const void *dev_ptr, uint64_t buf_len, uint64_t buf_lo,
                                         uint64_t global_len, uint64_t own_lo, uint64_t own_hi,
                                         int device, fzb_haystack **out) {
    return haystack_new(!dev_ptr || ((uintptr_t)dev_ptr & 15) ? "dev_ptr must be 16-byte aligned" : nullptr, nullptr,
                        dev_ptr, buf_len, buf_lo, global_len, own_lo, own_hi, device, out);
}

extern "C" int fzb_haystack_alloc(uint64_t buf_len, uint64_t buf_lo, uint64_t global_len, uint64_t own_lo,
                                  uint64_t own_hi, int device, fzb_haystack **out, void **dev_ptr) {
    const int rc = haystack_new(nullptr, nullptr, nullptr, buf_len, buf_lo, global_len, own_lo, own_hi, device, out);
    if (rc == FZB_OK && dev_ptr) *dev_ptr = (*out)->d;
    return rc;
}

extern "C" void fzb_synth_host(uint8_t *dst, uint64_t global_offset, uint64_t n, const uint8_t *alphabet,
                               uint32_t alphabet_len, uint64_t seed) {
    uint64_t i = 0;
    while (i < n) {
        uint64_t g = global_offset + i;
        uint32_t w = synth_word(seed, g / 4, alphabet, alphabet_len);
        for (uint64_t b = g % 4; b < 4 && i < n; b++, i++) dst[i] = (uint8_t)(w >> (8 * b));
    }
}

extern "C" int fzb_haystack_fill_synthetic(fzb_haystack *h, const uint8_t *alphabet, uint32_t alphabet_len,
                                           uint64_t seed) {
    HandleLock handle_lock(h);
    if (!h || !alphabet || alphabet_len == 0 || alphabet_len > 256) return fail(FZB_E_INVALID, "bad arguments");
    if (!h->owned_buf) return fail(FZB_E_INVALID, "cannot fill an adopted buffer");
    CK(cudaSetDevice(h->device));
    DevBuf<uint8_t> d_alpha;
    TRY(d_alpha.alloc(256));
    CK(cudaMemcpyAsync(d_alpha.get(), alphabet, alphabet_len, cudaMemcpyHostToDevice, h->stream));
    int64_t nwords = (int64_t)(round_up(h->buf_len, 4) / 4);
    k_fill_synth<<<h->sm_count * 8, 256, 0, h->stream>>>(h->d, (int64_t)h->buf_lo, nwords, seed, d_alpha.get(),
                                                        alphabet_len);
    CK(cudaGetLastError());
    // bytes past buf_len must stay zero (the last word may have spilled over)
    if (h->buf_len % 4)
        CK(cudaMemsetAsync(h->d + h->buf_len, 0, 4 - h->buf_len % 4, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    h->coll_prob = -1.0;
    return FZB_OK;
}

extern "C" int fzb_haystack_write(fzb_haystack *h, uint64_t global_offset, const uint8_t *src, uint64_t n) {
    HandleLock handle_lock(h);
    if (!h || (!src && n)) return fail(FZB_E_INVALID, "bad arguments");
    if (global_offset < h->buf_lo || global_offset + n > h->buf_lo + h->buf_len)
        return fail(FZB_E_INVALID, "write outside the buffer");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(h->d + (global_offset - h->buf_lo), src, n, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return FZB_OK;
}

extern "C" int fzb_haystack_read(fzb_haystack *h, uint64_t global_offset, uint8_t *dst, uint64_t n) {
    HandleLock handle_lock(h);
    if (!h || (!dst && n)) return fail(FZB_E_INVALID, "bad arguments");
    if (global_offset < h->buf_lo || global_offset + n > h->buf_lo + h->buf_len)
        return fail(FZB_E_INVALID, "read outside the buffer");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(dst, h->d + (global_offset - h->buf_lo), n, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return FZB_OK;
}

extern "C" uint64_t fzb_haystack_len(const fzb_haystack *h) {
    // under the handle's lock like every other call: a windowed exact search / has_near_match on another thread
    // swaps the geometry (global_len included) for the duration of its view
    HandleLock handle_lock(const_cast<fzb_haystack *>(h));
    return h ? h->global_len : 0;
}

// ------------------------------------------------------------------------------------------------
// Upload of PAGEABLE host memory (what a Python bytes object is).  cudaMemcpy from pageable memory stages through
// the driver's own bounce buffer, well below PCIe speed; page-locking the caller's buffer in place
// (cudaHostRegister) costs more than the copy.  Instead: a ring of three 64 MiB pinned buffers; a small pool of
// host threads copies slice i+1 of the caller's buffer into one of them while the DMA engine moves slice i
// to the device -- the pipeline runs at min(host memcpy bandwidth of the pool, PCIe).
// ------------------------------------------------------------------------------------------------
class CopyPool {
  public:
    static CopyPool &get() {
        static CopyPool *pool = new CopyPool();  // leaked on purpose: no joins at process exit
        return *pool;
    }
    void copy(uint8_t *dst, const uint8_t *src, size_t n) {  // parallel memcpy; returns when all of it is done
        if (n < (8u << 20) || threads_.empty()) {
            memcpy(dst, src, n);
            return;
        }
        {
            std::lock_guard<std::mutex> lock(m_);
            dst_ = dst;
            src_ = src;
            n_ = n;
            next_.store(0);
            pending_ = (int)threads_.size();
            gen_++;
        }
        cv_.notify_all();
        work();  // the caller copies too
        std::unique_lock<std::mutex> lock(m_);
        done_.wait(lock, [&] { return pending_ == 0; });
    }

  private:
    static constexpr size_t kSlice = 2u << 20;
    CopyPool() {
        unsigned want = 16;  // enough to stay ahead of PCIe even when the source pages sit on a remote NUMA node
        if (const char *e = getenv("FZB_UPLOAD_THREADS")) want = (unsigned)std::max(0, atoi(e));
        unsigned hw = std::thread::hardware_concurrency();
        cpu_set_t set;
        if (sched_getaffinity(0, sizeof set, &set) == 0) hw = (unsigned)CPU_COUNT(&set);
        want = std::min(want, hw > 1 ? hw - 1 : 0u);
        for (unsigned i = 0; i < want; i++) {
            threads_.emplace_back([this] { loop(); });
            threads_.back().detach();
        }
    }
    void work() {
        for (;;) {
            const size_t off = next_.fetch_add(kSlice);
            if (off >= n_) return;
            memcpy(dst_ + off, src_ + off, std::min(kSlice, n_ - off));
        }
    }
    void loop() {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lock(m_);
                cv_.wait(lock, [&] { return gen_ != seen; });
                seen = gen_;
            }
            work();
            std::lock_guard<std::mutex> lock(m_);
            if (--pending_ == 0) done_.notify_all();
        }
    }
    std::vector<std::thread> threads_;
    std::mutex m_;
    std::condition_variable cv_, done_;
    uint8_t *dst_ = nullptr;
    const uint8_t *src_ = nullptr;
    size_t n_ = 0;
    std::atomic<size_t> next_{0};
    int pending_ = 0;
    uint64_t gen_ = 0;
};

constexpr int kStageBufs = 3;
constexpr size_t kStageBytes = 64u << 20;
static std::mutex g_stage_mutex;  // one staged upload at a time per process (the ring is shared by all handles)
static uint8_t *g_stage[kStageBufs];

static bool is_pinned_host(const void *p) {
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return attr.type == cudaMemoryTypeHost;
}

// host -> h->d + dst_off, n bytes, on h->stream; returns when the caller may reuse `host`
static int upload_bytes(fzb_haystack *h, uint64_t dst_off, const uint8_t *host, uint64_t n) {
    if (n == 0) return FZB_OK;
    if (n < (16u << 20) || is_pinned_host(host)) {
        CK(cudaMemcpyAsync(h->d + dst_off, host, n, cudaMemcpyHostToDevice, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        return FZB_OK;
    }
    std::lock_guard<std::mutex> lock(g_stage_mutex);
    for (auto &b : g_stage)
        if (!b) CK(cudaHostAlloc(&b, kStageBytes, cudaHostAllocPortable));
    cudaEvent_t ev[kStageBufs];
    for (auto &e : ev) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    int rc = FZB_OK;
    uint64_t off = 0;
    for (int i = 0; off < n && rc == FZB_OK; i++, off += kStageBytes) {
        const int b = i % kStageBufs;
        const size_t len = (size_t)std::min<uint64_t>(kStageBytes, n - off);
        cudaError_t e = i >= kStageBufs ? cudaEventSynchronize(ev[b]) : cudaSuccess;  // the DMA out of this buffer is done
        if (e == cudaSuccess) {
            CopyPool::get().copy(g_stage[b], host + off, len);
            e = cudaMemcpyAsync(h->d + dst_off + off, g_stage[b], len, cudaMemcpyHostToDevice, h->stream);
        }
        if (e == cudaSuccess) e = cudaEventRecord(ev[b], h->stream);
        if (e != cudaSuccess) rc = fail(FZB_E_CUDA, "staged upload failed: %s", cudaGetErrorString(e));
    }
    cudaError_t e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess && rc == FZB_OK) rc = fail(FZB_E_CUDA, "staged upload failed: %s", cudaGetErrorString(e));
    for (auto &x : ev) cudaEventDestroy(x);
    return rc;
}

// The handle holds a whole sequence, not a shard of a longer one.
static bool is_whole_sequence(const fzb_haystack *h) {
    return h->buf_lo == 0 && h->global_len == h->buf_len && h->own_lo == 0 && h->own_hi == h->buf_len;
}

extern "C" int fzb_haystack_upload(fzb_haystack *h, const uint8_t *host, uint64_t n) {
    HandleLock handle_lock(h);
    if (!h || (!host && n)) return fail(FZB_E_INVALID, "bad arguments");
    if (!h->owned_buf) return fail(FZB_E_INVALID, "upload needs an owned handle");
    if (round_up(n, 128) + 128 > h->owned_buf.size()) return fail(FZB_E_INVALID, "upload larger than the handle's capacity");
    CK(cudaSetDevice(h->device));
    h->recs.reset();
    if (!is_whole_sequence(h)) {  // a shard keeps its geometry: the new bytes replace the same window of the global sequence
        if (n != h->buf_len) return fail(FZB_E_INVALID, "a shard upload must supply exactly buf_len bytes");
    } else {
        h->buf_len = h->global_len = h->own_hi = n;
        h->own_lo = 0;
    }
    h->padded_len = round_up(n, 128) + 128;
    h->coll_prob = -1.0;
    CK(cudaMemsetAsync(h->d + n, 0, h->padded_len - n, h->stream));
    return upload_bytes(h, 0, host, n);  // the caller may reuse `host` as soon as we return
}

// Wide-symbol sequences (sym_kernels.cuh): the code units travel to a device scratch chunk by chunk and
// k_reduce_symbols writes one byte per symbol into the handle's buffer.
extern "C" int fzb_haystack_upload_symbols(fzb_haystack *h, const void *host, uint64_t n, uint32_t width,
                                           const uint32_t *alphabet, uint32_t n_alpha) {
    HandleLock handle_lock(h);
    if (!h || (!host && n) || (!alphabet && n_alpha)) return fail(FZB_E_INVALID, "bad arguments");
    if (width != 2 && width != 4) return fail(FZB_E_INVALID, "symbol width must be 2 or 4 bytes");
    if (n_alpha > (uint32_t)kMaxPattern) return fail(FZB_E_UNSUPPORTED, "more than %d distinct pattern symbols", kMaxPattern);
    for (uint32_t i = 1; i < n_alpha; i++)
        if (alphabet[i - 1] >= alphabet[i]) return fail(FZB_E_INVALID, "the alphabet must be strictly ascending");
    if (!h->owned_buf) return fail(FZB_E_INVALID, "upload needs an owned handle");
    if (round_up(n, 128) + 128 > h->owned_buf.size()) return fail(FZB_E_INVALID, "upload larger than the handle's capacity");
    if (!is_whole_sequence(h)) return fail(FZB_E_INVALID, "symbol uploads replace a whole (unsharded) sequence");
    CK(cudaSetDevice(h->device));
    h->recs.reset();
    h->buf_len = h->global_len = h->own_hi = n;
    h->padded_len = round_up(n, 128) + 128;
    h->coll_prob = -1.0;
    CK(cudaMemsetAsync(h->d + n, 0, h->padded_len - n, h->stream));
    if (n == 0) {
        CK(cudaStreamSynchronize(h->stream));
        return FZB_OK;
    }
    constexpr uint64_t kChunk = 16u << 20;  // symbols per chunk (a multiple of 4: the kernel stores 32-bit words)
    const uint64_t chunk = std::min<uint64_t>(kChunk, round_up(n, 4));
    // every operation below is on h->stream: a chunk's copy is ordered behind the reduction of the previous chunk, so
    // one scratch buffer is enough.  (On an error return, freeing the buffers waits for the work queued on them.)
    DevBuf<uint32_t> d_alpha;
    DevBuf<uint8_t> d_tmp;
    TRY(d_alpha.alloc(256));
    if (n_alpha) CK(cudaMemcpyAsync(d_alpha.get(), alphabet, n_alpha * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
    TRY(d_tmp.alloc(chunk * width));
    const uint8_t *src = static_cast<const uint8_t *>(host);
    for (uint64_t off = 0; off < n; off += chunk) {
        const uint64_t cnt = std::min<uint64_t>(chunk, n - off);
        CK(cudaMemcpyAsync(d_tmp.get(), src + off * width, cnt * width, cudaMemcpyHostToDevice, h->stream));
        const int grid = (int)std::min<uint64_t>((uint64_t)h->sm_count * 8, (cnt / 4 + kSymThreads - 1) / kSymThreads + 1);
        if (width == 4)
            k_reduce_symbols<uint32_t><<<grid, kSymThreads, 0, h->stream>>>(reinterpret_cast<const uint32_t *>(d_tmp.get()),
                                                                            cnt, d_alpha.get(), n_alpha, h->d + off);
        else
            k_reduce_symbols<uint16_t><<<grid, kSymThreads, 0, h->stream>>>(reinterpret_cast<const uint16_t *>(d_tmp.get()),
                                                                            cnt, d_alpha.get(), n_alpha, h->d + off);
        CK(cudaGetLastError());
    }
    CK(cudaStreamSynchronize(h->stream));
    return FZB_OK;
}

// Record sets (DESIGN.md section 5.10): the offsets and the per-granule lookup table of the exact stages, built whole
// in a new group that replaces the handle's only on success.
extern "C" int fzb_haystack_set_records(fzb_haystack *h, const uint64_t *offsets, uint64_t count) {
    HandleLock handle_lock(h);
    if (!h) return fail(FZB_E_INVALID, "haystack handle is NULL");
    if (!is_whole_sequence(h)) return fail(FZB_E_INVALID, "record sets need a whole (unsharded) sequence");
    if (count == 0) {
        h->recs.reset();
        return FZB_OK;
    }
    if (!offsets) return fail(FZB_E_INVALID, "offsets is NULL");
    if (count >= (1ull << 32)) return fail(FZB_E_INVALID, "a record set holds fewer than 2^32 records");
    if (offsets[0] != 0 || offsets[count] != h->global_len)
        return fail(FZB_E_INVALID, "record offsets must run from 0 to the sequence length");
    for (uint64_t i = 0; i < count; i++)
        if (offsets[i + 1] <= offsets[i]) return fail(FZB_E_INVALID, "record offsets must be strictly increasing");
    CK(cudaSetDevice(h->device));
    const uint64_t ngran = (h->global_len + kGranule - 1) >> kGranuleShift;
    std::unique_ptr<RecBufs> recs;
    TRY(ensure_group(recs, [&](RecBufs &b) -> int {
        TRY(b.d_off.alloc(count + 1));
        TRY(b.d_first.alloc(ngran));
        CK(cudaMemcpyAsync(b.d_off.get(), offsets, (count + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
        const int grid = (int)std::min<uint64_t>((uint64_t)h->sm_count * 8, (ngran + 255) / 256);
        k_rec_first<<<grid, 256, 0, h->stream>>>(b.d_off.get(), count, b.d_first.get(), ngran);
        CK(cudaGetLastError());
        CK(cudaStreamSynchronize(h->stream));
        for (uint64_t i = 0; i < count; i++) b.longest = std::max(b.longest, offsets[i + 1] - offsets[i]);
        return FZB_OK;
    }));
    h->recs = std::move(recs);
    return FZB_OK;
}

// The record set the exact stages of a search on `h` take (null pointers without one) and its compile-time switch:
// with_recs(h, f) returns f(std::true_type) on a handle with a record set, f(std::false_type) otherwise.
static RecSet rec_set(const fzb_haystack *h) {
    return h->recs ? RecSet{h->recs->d_off.get(), h->recs->d_first.get()} : RecSet{nullptr, nullptr};
}

template <class F>
static auto with_recs(const fzb_haystack *h, F f) {
    return h->recs ? f(std::true_type{}) : f(std::false_type{});
}

// The entry points outside a record set's scope (batches, has_near_match, windows, FZB_F_GLOBAL) refuse to run on one.
static int refuse_records(const fzb_haystack *h, const char *what) {
    return h && h->recs ? fail(FZB_E_UNSUPPORTED, "%s does not support record sets", what) : FZB_OK;
}

// The batches take a record set only when the caller asks for per-record results (FZB_F_PER_RECORD), so that a handle
// passed by accident does not silently change what a batch means; the flag without a record set is an error.
static int check_batch_records(const fzb_haystack *h, uint32_t flags) {
    if (!(flags & FZB_F_PER_RECORD)) return refuse_records(h, "a batch search without FZB_F_PER_RECORD");
    return h->recs ? FZB_OK : fail(FZB_E_INVALID, "FZB_F_PER_RECORD needs a handle with a record set");
}

extern "C" void *fzb_host_alloc(uint64_t n) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, n ? n : 1, cudaHostAllocDefault) != cudaSuccess) {
        cudaGetLastError();
        fail(FZB_E_CUDA, "cudaHostAlloc(%llu) failed", (unsigned long long)n);
        return nullptr;
    }
    return p;
}

extern "C" void fzb_host_free(void *p) { cudaFreeHost(p); }  // (a no-op for NULL)

extern "C" int fzb_timer_start(fzb_haystack *h) {
    if (!h) return fail(FZB_E_INVALID, "NULL handle");
    CK(cudaSetDevice(h->device));
    CK(cudaEventRecord(h->ev[3], h->stream));
    return FZB_OK;
}

extern "C" int fzb_timer_stop(fzb_haystack *h, double *ms) {
    if (!h || !ms) return fail(FZB_E_INVALID, "NULL argument");
    CK(cudaSetDevice(h->device));
    CK(cudaEventRecord(h->ev_stop, h->stream));
    CK(cudaEventSynchronize(h->ev_stop));
    float f = 0.f;
    CK(cudaEventElapsedTime(&f, h->ev[3], h->ev_stop));
    *ms = f;
    return FZB_OK;
}

extern "C" int fzb_nccl_unique_id(uint8_t id[FZB_NCCL_ID_BYTES]) {
    if (!id) return fail(FZB_E_INVALID, "NULL argument");
    int rc = nccl_load();
    if (rc) return rc;
    NcclId nid;
    NCCLCK(g_nccl.GetUniqueId(&nid));
    memcpy(id, nid.b, FZB_NCCL_ID_BYTES);
    return FZB_OK;
}

// The staging buffers of the all-gather, grown to `cap` rows per rank: the new ones are allocated before the old ones
// are released, so a failure leaves the handle with its previous buffers.
static int ensure_gather_buffers(fzb_haystack *h, uint32_t cap) {
    if (h->gather && cap <= h->gather->cap) return FZB_OK;
    const uint64_t slot = (uint64_t)(cap + 1) * kFinCols;
    std::unique_ptr<GatherBufs> grown;
    TRY(ensure_group(grown, [&](GatherBufs &g) -> int {
        TRY(g.d_send.alloc(slot));
        TRY(g.d_recv.alloc(slot * h->world));
        TRY(g.h_send.alloc(slot));
        TRY(g.h_recv.alloc(slot * h->world));
        g.cap = cap;
        return FZB_OK;
    }));
    h->gather = std::move(grown);
    return FZB_OK;
}

// Receive area + scratch of the peer-memory reduction (p2p_kernels.cuh).
static int p2p_alloc(fzb_haystack *h) {
    if (h->world > kMaxWorld) return fail(FZB_E_UNSUPPORTED, "world sizes above %d are not supported", kMaxWorld);
    CK(cudaSetDevice(h->device));
    h->slot_bytes = ((uint64_t)kHdrWords + (uint64_t)h->p2p_cap * kFinCols) * 8;
    h->flags_off = round_up(2 * (uint64_t)h->world * h->slot_bytes, 256);
    const size_t bytes = h->flags_off + 2 * kMaxWorld * sizeof(uint32_t) + 256;
    const uint64_t rows = (uint64_t)h->world * h->p2p_cap;
    return ensure_group(h->peer, [&](PeerBufs &pb) -> int {
        TRY(pb.d_p2p.alloc(bytes));
        CK(cudaMemset(pb.d_p2p.get(), 0, bytes));
        TRY(pb.d_ms.alloc(1));
        CK(cudaMemset(pb.d_ms.get(), 0, sizeof(MergeScratch)));
        TRY(pb.d_mscore.alloc(rows));
        TRY(pb.d_mpos.alloc(rows));
        TRY(pb.h_grows.alloc(rows * 2));
        TRY(pb.h_ghdr.alloc(16));
        memset(pb.h_ghdr.get(), 0, 16 * sizeof(uint32_t));
        return FZB_OK;
    });
}

static void close_peers(fzb_haystack *h) {
    for (int r = 0; r < kMaxWorld; r++) {
        if (h->peer_opened[r] && h->peer_base[r]) cudaIpcCloseMemHandle(h->peer_base[r]);
        h->peer_opened[r] = false;
        h->peer_base[r] = nullptr;
    }
}

static void p2p_free(fzb_haystack *h) {
    detach_pending(h);  // the last result's global rows may still sit in h_grows
    close_peers(h);
    h->peer.reset();
    h->p2p = false;
}

// Leaves the handle's current world (communicator, peer memory) and makes it rank `rank` of a new one.
static void reset_world(fzb_haystack *h, int rank, int world_size, bool local_world) {
    if (h->comm) nccl_comm_destroy(h->comm);
    h->comm = nullptr;
    p2p_free(h);
    h->rank = rank;
    h->world = world_size;
    h->epoch = 0;
    h->local_world = local_world;
}

extern "C" int fzb_haystack_comm_init(fzb_haystack *h, const uint8_t id[FZB_NCCL_ID_BYTES], int rank,
                                      int world_size) {
    if (!h || !id || world_size < 1 || rank < 0 || rank >= world_size) return fail(FZB_E_INVALID, "bad arguments");
    int rc = nccl_load();
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    reset_world(h, rank, world_size, false);
    NcclId nid;
    memcpy(nid.b, id, FZB_NCCL_ID_BYTES);
    NCCLCK(g_nccl.CommInitRank(&h->comm, world_size, nid, rank));
    TRY(ensure_gather_buffers(h, h->gather_cap));
    // Peer-memory world: every rank exports its receive area through CUDA IPC; the handles travel over the
    // fresh NCCL communicator (bootstrap only).  Any failure on any rank (no IPC in this container, no peer
    // access between two GPUs) leaves p2p = false on ALL ranks and FZB_F_GLOBAL searches use the staged path.
    struct Hello {
        cudaIpcMemHandle_t handle;
        int32_t ok, device;
        long long pid;
    };
    static_assert(sizeof(Hello) <= 128, "hello record");
    const size_t rec = 128;
    Hello me{};
    me.ok = world_size <= kMaxWorld && p2p_alloc(h) == FZB_OK &&
            cudaIpcGetMemHandle(&me.handle, h->peer->d_p2p.get()) == cudaSuccess;
    cudaGetLastError();
    me.device = h->device;
    me.pid = (long long)getpid();
    std::vector<uint8_t> all(rec * world_size);
    GatherBufs &g = *h->gather;
    auto exchange = [&](const void *mine) -> int {  // all-gather one 128-byte record per rank
        memset(g.h_send.get(), 0, rec);
        memcpy(g.h_send.get(), mine, sizeof(Hello));
        CK(cudaMemcpyAsync(g.d_send.get(), g.h_send.get(), rec, cudaMemcpyHostToDevice, h->stream));
        NCCLCK(g_nccl.AllGather(g.d_send.get(), g.d_recv.get(), rec, /*ncclInt8*/ 0, h->comm, h->stream));
        CK(cudaMemcpyAsync(g.h_recv.get(), g.d_recv.get(), rec * world_size, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        memcpy(all.data(), g.h_recv.get(), rec * world_size);
        return FZB_OK;
    };
    rc = exchange(&me);
    if (rc) return rc;
    bool ok = true;
    for (int r = 0; r < world_size; r++) ok = ok && reinterpret_cast<Hello *>(all.data() + rec * r)->ok;
    if (ok) {
        for (int r = 0; r < world_size && ok; r++) {
            const Hello *peer = reinterpret_cast<const Hello *>(all.data() + rec * r);
            if (r == rank) {
                h->peer_base[r] = h->peer->d_p2p.get();
            } else {
                void *ptr = nullptr;
                if (cudaIpcOpenMemHandle(&ptr, peer->handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                    cudaGetLastError();
                    ok = false;
                } else {
                    h->peer_base[r] = (uint8_t *)ptr;
                    h->peer_opened[r] = true;
                }
            }
        }
    }
    Hello second{};
    second.ok = ok;
    rc = exchange(&second);  // everybody must have opened everybody
    if (rc) return rc;
    for (int r = 0; r < world_size; r++) ok = ok && reinterpret_cast<Hello *>(all.data() + rec * r)->ok;
    h->p2p = ok;
    if (!ok) close_peers(h);
    return FZB_OK;
}

extern "C" int fzb_comm_init_local(fzb_haystack **handles, int world_size) {
    if (!handles || world_size < 1 || world_size > kMaxWorld) return fail(FZB_E_INVALID, "bad arguments");
    for (int r = 0; r < world_size; r++)
        if (!handles[r]) return fail(FZB_E_INVALID, "NULL handle");
    for (int r = 0; r < world_size; r++) {
        fzb_haystack *h = handles[r];
        reset_world(h, r, world_size, true);
        TRY(p2p_alloc(h));
    }
    for (int r = 0; r < world_size; r++) {
        fzb_haystack *h = handles[r];
        CK(cudaSetDevice(h->device));
        for (int q = 0; q < world_size; q++) {
            h->peer_base[q] = handles[q]->peer->d_p2p.get();
            if (handles[q]->device != h->device) {
                int can = 0;
                CK(cudaDeviceCanAccessPeer(&can, h->device, handles[q]->device));
                if (!can) return fail(FZB_E_UNSUPPORTED, "no peer access between devices %d and %d", h->device, handles[q]->device);
                cudaError_t e = cudaDeviceEnablePeerAccess(handles[q]->device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
                    return fail(FZB_E_CUDA, "cudaDeviceEnablePeerAccess failed: %s", cudaGetErrorString(e));
                cudaGetLastError();
            }
        }
        h->p2p = true;
    }
    return FZB_OK;
}

// The same peer-memory world WITHOUT NCCL: the caller all-gathers the 64-byte CUDA IPC handles itself (any transport;
// fuzzysearch_b200.sharding does it over its TCP rendezvous).  Also works for several processes sharing ONE GPU,
// which NCCL refuses.  Such a world has no staged fallback: a shard that overflows a slot makes the search fail on
// every rank (FZB_E_UNSUPPORTED) instead of silently returning a partial list.
extern "C" int fzb_p2p_export(fzb_haystack *h, int rank, int world_size, uint8_t handle[FZB_IPC_HANDLE_BYTES]) {
    if (!h || !handle || world_size < 1 || world_size > kMaxWorld || rank < 0 || rank >= world_size)
        return fail(FZB_E_INVALID, "bad arguments");
    static_assert(sizeof(cudaIpcMemHandle_t) == FZB_IPC_HANDLE_BYTES, "IPC handle size");
    CK(cudaSetDevice(h->device));
    reset_world(h, rank, world_size, false);
    TRY(p2p_alloc(h));
    cudaIpcMemHandle_t mine;
    CK(cudaIpcGetMemHandle(&mine, h->peer->d_p2p.get()));
    memcpy(handle, &mine, sizeof mine);
    return FZB_OK;
}

extern "C" int fzb_p2p_connect(fzb_haystack *h, const uint8_t *handles) {
    if (!h || !handles || !h->peer) return fail(FZB_E_INVALID, "fzb_p2p_export first");
    CK(cudaSetDevice(h->device));
    for (int r = 0; r < h->world; r++) {
        if (r == h->rank) {
            h->peer_base[r] = h->peer->d_p2p.get();
            continue;
        }
        cudaIpcMemHandle_t peer;
        memcpy(&peer, handles + (size_t)r * FZB_IPC_HANDLE_BYTES, sizeof peer);
        void *ptr = nullptr;
        const cudaError_t e = cudaIpcOpenMemHandle(&ptr, peer, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) {
            cudaGetLastError();
            close_peers(h);
            return fail(FZB_E_CUDA, "cudaIpcOpenMemHandle(rank %d) failed: %s", r, cudaGetErrorString(e));
        }
        h->peer_base[r] = (uint8_t *)ptr;
        h->peer_opened[r] = true;
    }
    h->p2p = true;
    h->local_world = true;  // (no NCCL communicator behind this world: no staged fallback)
    return FZB_OK;
}

extern "C" void fzb_p2p_disable(fzb_haystack *h) {
    if (h) p2p_free(h);
}

extern "C" int fzb_haystack_p2p_enabled(const fzb_haystack *h) { return h && h->p2p ? 1 : 0; }

// ------------------------------------------------------------------------------------------------
// consolidation (common.py:145-189).  Groups are the connected components of interval overlap
// (SURVEY F11): sort by (start,end), sweep with the running hull end; a match joins the current
// group iff start < hull_end (this also reproduces the reference for empty matches, which never
// overlap anything they merely touch).  Winner = min (dist, -(end-start)), ties -> smallest
// (start,end).  Output sorted by (start,end,dist).
//
// The sweep runs over GROUPS: a winner (start, end, dist) and the hull [hull_start, hull_end) of its members.  A raw
// match is a group of its own, whose hull is the match.  Groups of different shards that overlap belong to one
// global group (a group's hull is covered by its members, so hulls overlap iff members do), and the winner of a
// union is the better of the two winners -- so the global consolidate_overlapping_matches (common.py:185-189) is
// the same sweep run over the per-shard groups instead of the raw matches.
// ------------------------------------------------------------------------------------------------
struct GroupRow {
    int64_t s, e, d, hs, he;
};

static bool group_less(const GroupRow &a, const GroupRow &b) {
    if (a.hs != b.hs) return a.hs < b.hs;
    if (a.he != b.he) return a.he < b.he;
    if (a.s != b.s) return a.s < b.s;
    if (a.e != b.e) return a.e < b.e;
    return a.d < b.d;
}

// `g` sorted by group_less.  Winners come out in group order, which is already (start, end, dist) order: groups
// are disjoint and ordered, and an empty group at x sorts before a group starting at x.
static void sweep_groups(const std::vector<GroupRow> &g, std::vector<RawRec> &out, std::vector<int64_t> *hulls = nullptr) {
    auto better = [](const GroupRow &a, const GroupRow &b) {  // a strictly better than b
        if (a.d != b.d) return a.d < b.d;
        int64_t la = a.e - a.s, lb = b.e - b.s;
        if (la != lb) return la > lb;
        if (a.s != b.s) return a.s < b.s;
        return a.e < b.e;
    };
    out.clear();
    if (hulls) hulls->clear();
    for (size_t i = 0, j; i < g.size(); i = j) {
        GroupRow best = g[i];
        int64_t hull_end = g[i].he;
        for (j = i + 1; j < g.size() && g[j].hs < hull_end; j++) {
            if (better(g[j], best)) best = g[j];
            hull_end = std::max(hull_end, g[j].he);
        }
        out.push_back(make_rec(best.s, best.e, best.d));
        if (hulls) {
            hulls->push_back(g[i].hs);
            hulls->push_back(hull_end);
        }
    }
}

static GroupRow match_row(int64_t start, int64_t end, int64_t dist) { return GroupRow{start, end, dist, start, end}; }

static void consolidate_recs(const std::vector<RawRec> &v, std::vector<RawRec> &out,
                             std::vector<int64_t> *hulls = nullptr) {
    std::vector<GroupRow> g;
    g.reserve(v.size());
    for (const RawRec &r : v) g.push_back(match_row(r.start, r.end, r.dist));
    std::sort(g.begin(), g.end(), group_less);
    sweep_groups(g, out, hulls);
}

static std::vector<GroupRow> match_rows(const int64_t *start, const int64_t *end, const int32_t *dist, uint64_t n) {
    std::vector<GroupRow> g(n);
    for (uint64_t i = 0; i < n; i++) g[i] = match_row(start[i], end[i], dist[i]);
    std::sort(g.begin(), g.end(), group_less);
    return g;
}

// Group rows (kFinCols columns) that arrive as one run of counts[r] rows per shard, in shard order, sorted for the
// sweep.  Every run is sorted by hull start and runs only interleave within a halo of their seams, so instead of
// sorting, each seam is fixed with an inplace_merge of the few out-of-order rows around it.
static std::vector<GroupRow> read_group_runs(const int64_t *rows, const std::vector<uint64_t> &counts) {
    uint64_t n = 0;
    for (uint64_t c : counts) n += c;
    std::vector<GroupRow> g;
    g.reserve(n);
    for (uint64_t c : counts) {
        const size_t seam = g.size();
        for (uint64_t i = 0; i < c; i++, rows += kFinCols) g.push_back(GroupRow{rows[0], rows[1], rows[2], rows[3], rows[4]});
        if (!std::is_sorted(g.begin() + seam, g.end(), group_less)) std::sort(g.begin() + seam, g.end(), group_less);  // defensive
        if (seam > 0 && seam < g.size() && group_less(g[seam], g[seam - 1])) {
            auto lo = std::upper_bound(g.begin(), g.begin() + seam, g[seam], group_less);
            auto hi = std::lower_bound(g.begin() + seam, g.end(), g[seam - 1], group_less);
            std::inplace_merge(lo, g.begin() + seam, hi, group_less);
        }
    }
    if (!std::is_sorted(g.begin(), g.end(), group_less)) std::sort(g.begin(), g.end(), group_less);  // shards smaller than a halo
    return g;
}

// The first n final matches and their hulls as group rows (start, end, dist, hull_start, hull_end).
static void write_group_rows(const std::vector<RawRec> &fin, const std::vector<int64_t> &hulls, size_t n, int64_t *rows) {
    for (size_t i = 0; i < n; i++, rows += kFinCols) {
        rows[0] = fin[i].start;
        rows[1] = fin[i].end;
        rows[2] = fin[i].dist;
        rows[3] = hulls[2 * i];
        rows[4] = hulls[2 * i + 1];
    }
}

extern "C" int64_t fzb_consolidate(const int64_t *start, const int64_t *end, const int32_t *dist, uint64_t n,
                                   int64_t *out_start, int64_t *out_end, int32_t *out_dist) {
    if (n && (!start || !end || !dist)) return fail(FZB_E_INVALID, "NULL input");
    std::vector<RawRec> o;
    sweep_groups(match_rows(start, end, dist, n), o);
    for (size_t i = 0; i < o.size(); i++) {
        if (out_start) out_start[i] = o[i].start;
        if (out_end) out_end[i] = o[i].end;
        if (out_dist) out_dist[i] = o[i].dist;
    }
    return (int64_t)o.size();
}

extern "C" int64_t fzb_consolidate_groups(const int64_t *start, const int64_t *end, const int32_t *dist, uint64_t n,
                                          int64_t *out_rows) {
    if (n && (!start || !end || !dist || !out_rows)) return fail(FZB_E_INVALID, "NULL input");
    std::vector<RawRec> o;
    std::vector<int64_t> hulls;
    sweep_groups(match_rows(start, end, dist, n), o, &hulls);
    write_group_rows(o, hulls, o.size(), out_rows);
    return (int64_t)o.size();
}

extern "C" int64_t fzb_result_group_rows(const fzb_result *r, int64_t *rows, uint64_t max_rows) {
    if (!r || (!rows && max_rows)) return fail(FZB_E_INVALID, "NULL argument");
    if (!r->have_fin || r->hulls.size() != r->fin.size() * 2)
        return fail(FZB_E_INVALID, "result was produced with FZB_F_NO_FINAL");
    write_group_rows(r->fin, r->hulls, std::min<size_t>(r->fin.size(), max_rows), rows);
    return (int64_t)r->fin.size();
}

extern "C" int fzb_result_hulls(const fzb_result *r, int64_t *hull_start, int64_t *hull_end) {
    if (!r) return fail(FZB_E_INVALID, "result is NULL");
    // (unconsolidated routes: every match is its own group, hull == the match)
    if (!r->have_fin || r->hulls.size() != r->fin.size() * 2)
        return fail(FZB_E_INVALID, "result was produced with FZB_F_NO_FINAL");
    for (size_t i = 0; i < r->fin.size(); i++) {
        if (hull_start) hull_start[i] = r->hulls[2 * i];
        if (hull_end) hull_end[i] = r->hulls[2 * i + 1];
    }
    return FZB_OK;
}

// Merge per-shard consolidated lists (group rows).  Where the shards' runs begin is not known here: the input is
// treated as a single run, sorted if needed.
extern "C" int64_t fzb_merge_groups(const int64_t *rows, uint64_t n, int64_t *out_start, int64_t *out_end,
                                    int32_t *out_dist) {
    if (n && !rows) return fail(FZB_E_INVALID, "NULL input");
    std::vector<RawRec> o;
    sweep_groups(read_group_runs(rows, {n}), o);
    for (size_t i = 0; i < o.size(); i++) {
        if (out_start) out_start[i] = o[i].start;
        if (out_end) out_end[i] = o[i].end;
        if (out_dist) out_dist[i] = o[i].dist;
    }
    return (int64_t)o.size();
}

// The staged (host-buffer) all-gather of group rows: used when the fused one behind the kernels could
// not be trusted on every rank (a rank overflowed a buffer and retried, or its list was too long for
// the on-device consolidation).  Collective: every rank calls it the same number of times.
static int allgather_groups_staged(fzb_haystack *h, const std::vector<int64_t> &rows, std::vector<int64_t> &all,
                                   std::vector<uint64_t> &counts) {
    const uint64_t n = rows.size() / kFinCols;
    for (;;) {
        const uint32_t cap = h->gather_cap;
        TRY(ensure_gather_buffers(h, cap));
        GatherBufs &g = *h->gather;
        const size_t slot_rows = (size_t)cap + 1, slot = slot_rows * kFinCols * sizeof(int64_t);
        g.h_send[0] = (int64_t)n;
        g.h_send[1] = n <= cap;
        g.h_send[2] = g.h_send[3] = g.h_send[4] = 0;
        if (n <= cap && n) memcpy(g.h_send.get() + kFinCols, rows.data(), n * kFinCols * sizeof(int64_t));
        CK(cudaMemcpyAsync(g.d_send.get(), g.h_send.get(), (1 + (n <= cap ? n : 0)) * kFinCols * sizeof(int64_t),
                           cudaMemcpyHostToDevice, h->stream));
        NCCLCK(g_nccl.AllGather(g.d_send.get(), g.d_recv.get(), slot, /*ncclInt8*/ 0, h->comm, h->stream));
        CK(cudaMemcpyAsync(g.h_recv.get(), g.d_recv.get(), slot * h->world, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        uint64_t top = 0;
        for (int r = 0; r < h->world; r++) top = std::max<uint64_t>(top, (uint64_t)g.h_recv[(size_t)r * slot_rows * kFinCols]);
        if (top <= cap) {
            all.clear();
            counts.clear();
            for (int r = 0; r < h->world; r++) {
                const int64_t *base = g.h_recv.get() + (size_t)r * slot_rows * kFinCols;
                all.insert(all.end(), base + kFinCols, base + kFinCols + (size_t)base[0] * kFinCols);
                counts.push_back((uint64_t)base[0]);
            }
            return FZB_OK;
        }
        while (h->gather_cap < top) h->gather_cap *= 2;  // every rank sees the same `top`
    }
}

// ------------------------------------------------------------------------------------------------
// search plumbing
// ------------------------------------------------------------------------------------------------
static void fill_params(const fzb_haystack *h, const uint8_t *pattern, uint32_t m, ScanParams &p) {
    memset(&p, 0, sizeof p);
    p.H = h->d;
    p.buf_lo = (int64_t)h->buf_lo;
    p.buf_len = (int64_t)h->buf_len;
    p.N = (int64_t)h->global_len;
    p.own_lo = (int64_t)h->own_lo;
    p.own_hi = (int64_t)h->own_hi;
    p.bitmap = h->d_bitmap.get();
    p.glist = h->d_glist.get();
    p.glist_cap = h->glist_cap;
    p.counters = h->d_counters.get();
    p.m = (int)m;
    memcpy(p.P, pattern, m);
}

static int check_halo(const fzb_haystack *h, uint64_t halo) {
    uint64_t need_lo = h->own_lo > halo ? h->own_lo - halo : 0;
    uint64_t need_hi = std::min(h->global_len, h->own_hi + halo);
    if (h->own_lo == h->own_hi) return FZB_OK;
    if (h->buf_lo > need_lo || h->buf_lo + h->buf_len < need_hi)
        return fail(FZB_E_INVALID, "shard halo too small: need %llu bytes each side",
                    (unsigned long long)halo);
    return FZB_OK;
}

static int check_pattern(const fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t flags) {
    if (!h) return fail(FZB_E_INVALID, "haystack handle is NULL");
    if (flags & FZB_F_GLOBAL) TRY(refuse_records(h, "FZB_F_GLOBAL"));
    if ((flags & FZB_F_GLOBAL) && !h->comm && !h->local_world)
        return fail(FZB_E_INVALID, "FZB_F_GLOBAL needs fzb_haystack_comm_init / fzb_comm_init_local on this handle");
    if (!pattern || m == 0) return fail(FZB_E_INVALID, "Given subsequence is empty!");
    if (m > FZB_MAX_PATTERN) return fail(FZB_E_UNSUPPORTED, "pattern longer than %d bytes", FZB_MAX_PATTERN);
    return FZB_OK;
}

// How one pattern is searched: the route that runs, the total limit k it runs with (after every clamp and lowering)
// and, on the generic routes, the per-operation limits clamped to k.  The plan_* functions are the one statement of
// the route rules and of the refusals of the single searches; the single searches, the batches and
// fzb_best_per_record all run from plans.  Routes: Exact is search_lev_ngrams at k = 0 with the sorted raw list for
// final list, LevNgrams search_lev_ngrams (also the generic search's k = 0 route), LevLp search_lev_lp, Hamming
// search_hamming, GenericNgrams and GenericLp the two routes of search_generic.
enum class Route : uint8_t { Exact, LevNgrams, LevLp, Hamming, GenericNgrams, GenericLp };

struct Plan {
    Route route;
    uint32_t m, k, subs, ins, dels;
    uint32_t L() const { return m / (k + 1); }  // the n-gram length of the n-gram routes
    bool generic() const { return route == Route::GenericNgrams || route == Route::GenericLp; }
};

// The n-gram routes take n-grams of at least 3 symbols (levenshtein.py:9-38, generic_search.py:25-54), or k == 0;
// FZB_F_FORCE_LP, then FZB_F_FORCE_NGRAMS, override.
static bool ngram_route(uint32_t m, uint32_t k, uint32_t flags) {
    if (flags & FZB_F_FORCE_LP) return false;
    return (flags & FZB_F_FORCE_NGRAMS) || k == 0 || m / ((uint64_t)k + 1) >= 3;
}

static int check_ngram_length(const Plan &pl) {
    return pl.L() == 0 ? fail(FZB_E_NGRAM_ZERO, "the subsequence length must be greater than max_l_dist") : FZB_OK;
}

static int plan_exact(const fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t flags, Plan &pl) {
    // check_pattern in the words of the exact search (search_exact.py), which has only this one complaint
    const int rc = check_pattern(h, pattern, m, flags);
    if (rc) return rc == FZB_E_INVALID && h ? fail(FZB_E_INVALID, "subsequence must not be empty") : rc;
    pl = Plan{Route::Exact, m, 0, 0, 0, 0};
    return check_halo(h, m);
}

static int plan_levenshtein(const fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t k, uint32_t flags,
                            Plan &pl) {
    TRY(check_pattern(h, pattern, m, flags));
    // every k >= len(pattern) takes the same branch (levenshtein.py:62-65): (i, i, m) for all i
    pl = Plan{Route::LevLp, m, std::min(k, m), 0, 0, 0};
    if (ngram_route(m, pl.k, flags)) {
        pl.route = Route::LevNgrams;
        TRY(check_ngram_length(pl));
    }
    return check_halo(h, (uint64_t)m + pl.k);
}

static int plan_hamming(const fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t k, uint32_t flags,
                        Plan &pl) {
    TRY(check_pattern(h, pattern, m, flags));
    pl = Plan{Route::Hamming, m, std::min(k, m), 0, 0, 0};
    return check_halo(h, m);
}

static int plan_generic(const fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t max_subs,
                        uint32_t max_ins, uint32_t max_dels, uint32_t max_l, uint32_t flags, Plan &pl) {
    TRY(check_pattern(h, pattern, m, flags));
    // find_near_matches_generic (generic_search.py:25-54)
    if (max_l == 0 && !(flags & (FZB_F_FORCE_LP | FZB_F_FORCE_NGRAMS))) {
        pl = Plan{Route::LevNgrams, m, 0, 0, 0, 0};
        return check_halo(h, m);
    }
    pl = Plan{Route::GenericNgrams, m, max_l, 0, 0, 0};
    if (!ngram_route(m, max_l, flags)) {
        // LP route: every substitution and every deletion consumes a pattern character (so does the "insertion +
        // deletion" pair the reference books when the substitutions are used up, generic_search.py:111-128), hence a
        // live candidate at pattern index j has spent l <= j + n_ins < m + max_ins: a total limit above m + max_ins
        // never binds -- not in `l_dist < max_l_dist` (:101-102), not in the deletion loop's bound (:141), not in the
        // final loop (:172-177) -- and can be lowered to it without changing the raw stream.  (Not so on the n-gram
        // route, where max_l_dist also sets the n-gram length and the windows.)  E.g. max_substitutions=100,
        // max_insertions=1, max_deletions=1 on 20 symbols: 102 -> 21.
        pl.route = Route::GenericLp;
        pl.k = (uint32_t)std::min<uint64_t>(max_l, (uint64_t)m + std::min(max_ins, max_l));
    }
    // the packed candidate of sim_generic keeps 6 bits per counter
    if (pl.k > 63) return fail(FZB_E_UNSUPPORTED, "max_l_dist > 63 is not supported by the generic search");
    // no counter can exceed k (every operation that increments one costs >= 1), so clamping the per-operation limits
    // to k changes nothing (LevenshteinSearchParams does the same, common.py:108-116)
    pl.subs = std::min(max_subs, pl.k);
    pl.ins = std::min(max_ins, pl.k);
    pl.dels = std::min(max_dels, pl.k);
    TRY(check_halo(h, (uint64_t)m + pl.k));
    return pl.route == Route::GenericNgrams ? check_ngram_length(pl) : FZB_OK;
}

// choose_search_class (__init__.py:60-83) on normalised limits
static int plan_by_class(const fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t max_subs,
                         uint32_t max_ins, uint32_t max_dels, uint32_t max_l, uint32_t flags, Plan &pl) {
    if (max_l == 0) return plan_exact(h, pattern, m, flags, pl);
    if (max_ins == 0 && max_dels == 0) return plan_hamming(h, pattern, m, std::min(max_l, max_subs), flags, pl);
    if (max_l <= std::min(max_subs, std::min(max_ins, max_dels)))
        return plan_levenshtein(h, pattern, m, max_l, flags, pl);
    return plan_generic(h, pattern, m, max_subs, max_ins, max_dels, max_l, flags, pl);
}

constexpr uint64_t kMaxRawRecs = 1ull << 27;  // raw records of one search (or one shared batch pass)

// Grows d_out to hold `need` records.  The new buffer is allocated before the old one is released, so a failure leaves
// the handle with its previous buffer and size; the price is a transient peak of 1.5x the new size during the growth
// (at the 2^27-record limit, 40 B per record: 5.4 GB + 2.7 GB).
static int ensure_out_cap(fzb_haystack *h, uint64_t need) {
    if (need <= h->d_out.size()) return FZB_OK;
    uint64_t cap = h->d_out.size();
    while (cap < need) cap *= 2;
    if (cap > kMaxRawRecs) return fail(FZB_E_UNSUPPORTED, "more than 2^27 raw matches in one search");
    return alloc_out(h, cap);
}

// Runs one search attempt after another until the output buffer was large enough.  `enqueue` must
// put EVERY kernel of the search on h->stream (filter included: the verify kernels clear the dirty
// bitmap as they consume it, so a retry has to re-mark it) and may record h->ev[1] after its scan
// kernel.  One attempt = one stream synchronisation and NO copy operation: k_post, enqueued behind the
// emitting kernels, writes the counters, the raw records and the final rows into mapped pinned host
// memory, which the host reads as soon as the stream has drained.

// Completion of a search attempt: its last kernel stores h->seq into mapped pinned memory after everything else
// (fenced at system scope); polling that word returns a few microseconds earlier than cudaStreamSynchronize and
// does not depend on the process's device scheduling flags (another library in the process -- e.g. a framework
// that asked for blocking synchronisation -- would otherwise add its wake-up latency to every search).  Falls back to
// the stream synchronisation if the word does not arrive (a failed launch), which also surfaces the error.
static int wait_done(fzb_haystack *h, const volatile uint32_t *word) {
    const uint32_t want = h->seq;
    for (uint64_t spins = 0; *word != want; spins++) {
#if defined(__x86_64__) || defined(__i386__)
        __builtin_ia32_pause();
#endif
        if ((spins & 0xFFF) == 0xFFF) {
            const cudaError_t e = cudaStreamQuery(h->stream);
            if (e == cudaSuccess) break;  // stream drained: the word is there (or the kernel never ran: error below)
            if (e != cudaErrorNotReady) return fail(FZB_E_CUDA, "search failed: %s", cudaGetErrorString(e));
        }
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    if (*word != want) {
        CK(cudaStreamSynchronize(h->stream));
        CK(cudaGetLastError());
        if (*word != want) return fail(FZB_E_CUDA, "search kernels did not complete");
    }
    return FZB_OK;
}

// What k_post should do behind the emitting kernels.
struct PostPlan {
    int mode = 1;         // 0 raw stream only; 1 consolidate_overlapping_matches; 2 final = sorted raw list
    bool global = false;  // FZB_F_GLOBAL: reduce the groups of every shard behind the kernels
};

static void finalize_on_host(fzb_result *res, int mode);

template <class F>
static int run_emitting(fzb_haystack *h, fzb_result *res, F enqueue, PostPlan post = PostPlan()) {
    detach_pending(h);  // k_post is about to overwrite the staging buffer an earlier result may still point at
    for (int attempt = 0; attempt < 8; attempt++) {
        if (!h->counters_clean) CK(cudaMemsetAsync(h->d_counters.get(), 0, CNT_COUNT * sizeof(uint32_t), h->stream));
        h->counters_clean = false;
        CK(cudaEventRecord(h->ev[0], h->stream));
        h->ev1_recorded = false;
        int rc = enqueue();
        if (rc) return rc;
        CK(cudaGetLastError());
        h->seq++;
        PostArgs pa{reinterpret_cast<const uint64_t *>(h->d_out.get() + h->d_out.size()), (uint32_t)h->d_out.size(), post.mode,
                    h->d_sorted.get(), h->d_fin.get(), h->h_fin.get(), h->h_counters.get(), h->d_counters.get(), h->seq, 0};
        // fused multi-GPU reduction over peer memory (below): k_push reads the counters after k_post, and clears them
        pa.clear = !(post.global && attempt == 0 && h->p2p && !res->fused_issued);
        k_post<<<h->sm_count, kPostThreads, kPostSmem, h->stream>>>(pa);
        CK(cudaGetLastError());
        res->stats.n_launches++;
        // fused multi-GPU reduction over peer memory: exactly one push + merge per search, in the FIRST attempt
        // (a rank that has to retry locally has pushed a header with valid = 0: every rank sees it and all of them
        // take the staged path together)
        const bool fused = post.global && attempt == 0 && h->p2p && !res->fused_issued;
        if (fused) {
            h->epoch++;
            WorldArgs w{};
            w.world = h->world;
            w.rank = h->rank;
            w.epoch = h->epoch;
            w.cap = h->p2p_cap;
            w.slot_bytes = h->slot_bytes;
            w.flags_off = h->flags_off;
            for (int r = 0; r < h->world; r++) w.peer[r] = h->peer_base[r];
            PeerBufs &pb = *h->peer;
            k_push<<<kPushCtas, kPushThreads, 0, h->stream>>>(w, h->d_fin.get(), h->d_counters.get(), post.mode, pb.d_ms.get());
            MergeOut mo{pb.d_mscore.get(), pb.d_mpos.get(), pb.h_grows.get(), pb.h_ghdr.get(), h->seq};
            k_merge<<<h->world, kPostThreads, 0, h->stream>>>(w, pb.d_ms.get(), mo);
            CK(cudaGetLastError());
            res->stats.n_launches += 2;
        }
        CK(cudaEventRecord(h->ev[2], h->stream));
        rc = wait_done(h, fused ? h->peer->h_ghdr.get() + 7 : h->h_counters.get() + CNT_SEQ);
        if (rc) return rc;
        const uint32_t n = h->h_counters[CNT_OUT];
        res->stats.n_candidates = h->h_counters[CNT_CAND];
        if (fused) {
            res->fused_issued = true;
            res->fused_status = h->peer->h_ghdr[0];
            res->gcount = h->peer->h_ghdr[1];
            if (h->peer->h_ghdr[2] != h->epoch && res->fused_status == MS_OK) res->fused_status = MS_TIMEOUT;
        }
        if (n > h->d_out.size()) {  // output buffer too small: grow and redo the whole attempt
            TRY(ensure_out_cap(h, n));
            continue;
        }
        const bool posted = h->h_counters[CNT_POST_DONE] != 0;
        // k_post (or k_push behind it, if the shard was valid) zeroed the device counters on its way out
        h->counters_clean = posted && (!fused || (res->fused_status == MS_OK));
        res->raw.clear();
        res->raw_n = n;
        res->raw_ordered = false;
        if (posted || (res->fused_issued && res->fused_status == MS_OK)) {
            // the raw records are in h->d_out, the global rows in h->peer->h_grows: copied out lazily (fetch_raw)
            std::lock_guard<std::mutex> lock(g_pending_mutex);
            res->raw_in_stage = posted;
            res->owner = h;
            h->pending = res;
        }
        if (!posted && n) {  // list too long for k_post: fetch it, the host orders and consolidates
            res->raw.resize(n);
            CK(cudaMemcpyAsync(res->raw.data(), h->d_out.get(), (size_t)n * sizeof(RawRec), cudaMemcpyDeviceToHost, h->stream));
            CK(cudaStreamSynchronize(h->stream));
        }
        res->fin.clear();
        res->hulls.clear();
        res->have_fin = false;
        res->device_post = false;
        if (post.mode != 0) {
            if (posted) {
                const uint32_t nf = h->h_counters[CNT_NFINAL];
                res->fin.resize(nf);
                res->hulls.resize((size_t)nf * 2);
                for (uint32_t i = 0; i < nf; i++) {
                    res->fin[i] = make_rec(h->h_fin[kFinCols * i], h->h_fin[kFinCols * i + 1], h->h_fin[kFinCols * i + 2]);
                    res->hulls[2 * i] = h->h_fin[kFinCols * i + 3];
                    res->hulls[2 * i + 1] = h->h_fin[kFinCols * i + 4];
                }
                res->device_post = true;
            } else {
                finalize_on_host(res, post.mode);
            }
            res->have_fin = true;
        }
        float ms = 0.f;
        while (cudaEventQuery(h->ev[2]) == cudaErrorNotReady) {  // a microsecond behind the polled word
        }
        cudaEventElapsedTime(&ms, h->ev[0], h->ev[2]);
        res->stats.gpu_ms = ms;
        res->stats.filter_ms = ms;
        if (h->ev1_recorded) {
            cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]);
            res->stats.filter_ms = ms;
        }
        return FZB_OK;
    }
    return fail(FZB_E_CUDA, "output buffer kept overflowing");
}

static void sort_generation_order(std::vector<RawRec> &v) {
    std::sort(v.begin(), v.end(), [](const RawRec &a, const RawRec &b) {
        if (a.ngram != b.ngram) return a.ngram < b.ngram;
        return a.idx < b.idx;
    });
}

static void sort_canonical(std::vector<RawRec> &v) {
    std::sort(v.begin(), v.end(), [](const RawRec &a, const RawRec &b) {
        if (a.start != b.start) return a.start < b.start;
        if (a.end != b.end) return a.end < b.end;
        return a.dist < b.dist;
    });
}

void fzb_result::order_raw() {
    fetch_raw();
    if (raw_ordered) return;
    if (raw_order == 0)
        sort_generation_order(raw);
    else if (raw_order == 1)
        sort_canonical(raw);
    else
        std::sort(raw.begin(), raw.end(), [](const RawRec &a, const RawRec &b) {
            if (a.ngram != b.ngram) return a.ngram < b.ngram;
            if (a.idx != b.idx) return a.idx < b.idx;
            if (a.start != b.start) return a.start < b.start;
            if (a.end != b.end) return a.end < b.end;
            return a.dist < b.dist;
        });
    raw_ordered = true;
}

// Host twin of k_post for lists it does not take (more than kPostMax records).
static void finalize_on_host(fzb_result *res, int mode) {
    if (mode == 1) {
        consolidate_recs(res->raw, res->fin, &res->hulls);
        return;
    }
    res->fin = res->raw;
    sort_canonical(res->fin);
    res->hulls.resize(res->fin.size() * 2);
    for (size_t i = 0; i < res->fin.size(); i++) {
        res->fin[i].idx = -1;
        res->fin[i].ngram = -1;
        res->hulls[2 * i] = res->fin[i].start;
        res->hulls[2 * i + 1] = res->fin[i].end;
    }
}

static int set_filter_attrs(size_t smem) {
    // per device: the attribute belongs to the function on the current device
    CK(cudaFuncSetAttribute(k_filter_sampled, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(k_filter_dense<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDenseSmem));
    CK(cudaFuncSetAttribute(k_filter_dense<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDenseSmem));
    CK(cudaFuncSetAttribute(k_filter_dense<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDenseSmem));
    CK(cudaFuncSetAttribute(k_filter_dense<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDenseSmem));
    CK(cudaFuncSetAttribute(k_filter_dense2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDense2Smem));
    return FZB_OK;
}

constexpr int kVerifyCtasPerSm = 8;  // k_verify_lev is latency bound (one DRAM round trip + a dependent chain per granule)

// The q-sample lemma of k_filter_sampled needs floor((m-k-3)/4) >= k+1 aligned words per occurrence.
static bool sampled_filter_applies(uint32_t m, uint32_t k, uint32_t flags) {
    if (flags & FZB_F_FORCE_DENSE) return false;
    if (m < 4 || m < k + 3) return false;
    return (m - k - 3) / 4 >= k + 1;
}

// Byte statistics of the haystack from 16 sampled 4 KiB blocks (once per handle content): the
// collision probability sum_c p_c^2 tells how selective a q-gram test is (1/4 on DNA, ~1/95 on text).
static int sample_collision_prob(fzb_haystack *h) {
    if (h->coll_prob >= 0.0) return FZB_OK;
    const uint64_t blk = 4096, nblk = 16;
    std::vector<uint8_t> buf;
    uint64_t hist[256] = {0}, total = 0;
    if (h->buf_len <= blk * nblk) {
        buf.resize(h->buf_len);
        if (h->buf_len) CK(cudaMemcpy(buf.data(), h->d, h->buf_len, cudaMemcpyDeviceToHost));
    } else {
        buf.resize(blk * nblk);
        for (uint64_t i = 0; i < nblk; i++) {
            const uint64_t off = ((h->buf_len - blk) / (nblk - 1) * i) & ~(uint64_t)15;
            CK(cudaMemcpyAsync(buf.data() + i * blk, h->d + off, blk, cudaMemcpyDeviceToHost, h->stream));
        }
        CK(cudaStreamSynchronize(h->stream));
    }
    for (uint8_t c : buf) hist[c]++;
    total = buf.size();
    double s = 0.0;
    if (total)
        for (int c = 0; c < 256; c++) s += ((double)hist[c] / total) * ((double)hist[c] / total);
    h->coll_prob = total ? s : 1.0;
    return FZB_OK;
}

// The sampled filter is sound whenever the lemma holds, but only SELECTIVE if an aligned word rarely
// equals a pattern 4-gram; otherwise (small alphabets) the dense filter, which finds the n-gram hits
// themselves, marks far fewer granules.  Expected marked-granule fractions decide.
static bool sampled_is_selective(fzb_haystack *h, uint32_t m, uint32_t k, int L, int n_ngrams) {
    if (sample_collision_prob(h) != FZB_OK) return true;
    const double c = h->coll_prob;
    const double span = (2.0 * m + 2.0 * k - L - 3.0) / kGranule + 1.0;       // granules marked per word hit
    const double sampled = std::min(1.0, (m - 3.0) * c * c * c * c * (kGranule / 4.0) * span);
    const double dense = std::min(1.0, n_ngrams * std::pow(c, std::min(L, 8)) * kGranule);
    return sampled <= 0.02 || sampled <= dense;
}

// The filter of an n-gram-route search of plan `pl`: the sampled one, or (false) the dense one.
static bool sampled_filter(fzb_haystack *h, const Plan &pl, uint32_t flags) {
    return sampled_filter_applies(pl.m, pl.k, flags) &&
           ((flags & FZB_F_FORCE_SAMPLED) || sampled_is_selective(h, pl.m, pl.k, (int)pl.L(), (int)(pl.m / pl.L())));
}

// Enqueue the one pass over the haystack that marks candidate granules; records ev[1] behind it.
static int enqueue_filter(fzb_haystack *h, const ScanParams &p, bool sampled, fzb_result *res) {
    const int64_t nvec = (int64_t)(round_up(h->buf_len, 16) / 16);
    int64_t ntiles = (nvec + kTileVecs - 1) / kTileVecs;
    // dense route on a low-entropy haystack (about six effective symbols or fewer): index the table with 2-bit codes
    bool two_bit = false;
    if (!sampled && h->buf_len > 0 && sample_collision_prob(h) == FZB_OK) two_bit = h->coll_prob >= 0.15;
    if (ntiles > 0) {
        int per_sm = 4;
        if (sampled) {  // the sampled scan strides over its own (larger) tiles
            ntiles = (nvec + kScanVecs - 1) / kScanVecs;
            if (h->scan_per_sm == 0) {
                CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_filter_sampled, kScanThreads, kScanSmem));
                h->scan_per_sm = std::max(per_sm, 1);
            }
            per_sm = h->scan_per_sm;
        } else if (two_bit) {
            CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_filter_dense2, kFilterThreads, kDense2Smem));
            per_sm = std::max(per_sm, 1);
        } else if (!sampled) {  // persistent grid = exactly the resident CTAs of the chosen instantiation
            const void *fn = p.q < 4    ? (const void *)k_filter_dense<0>
                             : p.q == 4 ? (const void *)k_filter_dense<1>
                             : p.q < 8  ? (const void *)k_filter_dense<2>
                                        : (const void *)k_filter_dense<3>;
            CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kFilterThreads, kDenseSmem));
            per_sm = std::max(per_sm, 1);
        }
        int grid = (int)std::min<int64_t>(ntiles, (int64_t)h->sm_count * per_sm);
        if (sampled)
            k_filter_sampled<<<grid, kScanThreads, kScanSmem, h->stream>>>(p, nvec, ntiles);
        else if (two_bit)
            k_filter_dense2<<<grid, kFilterThreads, kDense2Smem, h->stream>>>(p, nvec, ntiles);
        else if (p.q < 4)
            k_filter_dense<0><<<grid, kFilterThreads, kDenseSmem, h->stream>>>(p, nvec, ntiles);
        else if (p.q == 4)
            k_filter_dense<1><<<grid, kFilterThreads, kDenseSmem, h->stream>>>(p, nvec, ntiles);
        else if (p.q < 8)
            k_filter_dense<2><<<grid, kFilterThreads, kDenseSmem, h->stream>>>(p, nvec, ntiles);
        else
            k_filter_dense<3><<<grid, kFilterThreads, kDenseSmem, h->stream>>>(p, nvec, ntiles);
        CK(cudaGetLastError());
        res->stats.n_launches++;
    }
    CK(cudaEventRecord(h->ev[1], h->stream));
    h->ev1_recorded = true;
    return FZB_OK;
}

// n-gram Levenshtein search (also serves exact search as k == 0, L == m)
static int search_lev_ngrams(fzb_haystack *h, const uint8_t *pattern, const Plan &pl, uint32_t flags,
                             fzb_result *res, int post_mode) {
    const uint32_t m = pl.m, k = pl.k;
    ScanParams p;
    fill_params(h, pattern, m, p);
    p.k = (int)k;
    p.L = (int)pl.L();
    p.n_ngrams = (int)m / p.L;  // range(0, m-L+1, L)
    int rc;
    CK(cudaSetDevice(h->device));
    const bool sampled = sampled_filter(h, pl, flags);
    p.q = sampled ? 4 : std::min(p.L, 8);
    res->stats.route = k == 0 ? 0 : (sampled ? 1 : 2);
    res->stats.bytes_scanned = h->buf_len;
    CK(cudaSetDevice(h->device));
    if (!h->filter_attrs_set) {
        rc = set_filter_attrs(kScanSmem);
        if (rc) return rc;
        h->filter_attrs_set = true;
    }
    // dense route: confirmed n-gram hits go to a list and are verified one lane per hit (the window of a
    // hit must fit a lane's shared-memory slot); the list overflowing triggers one retry in granule mode
    const int vm = verify_mode((int)m, p.L);
    bool use_hits = !sampled && k > 0 && (m + 2 * k + 8 <= (uint32_t)kHitSlotBytes);
    if (use_hits && !h->d_hits)
        TRY(h->d_hits.alloc(std::min<uint64_t>(std::max<uint64_t>(1u << 20, h->owned_buf.size() / 256), 1u << 28)));
    bool fuse_gather = post_mode != 0 && (flags & FZB_F_GLOBAL) != 0;
    bool bitmap_mode = false;
    if (flags & FZB_F_TINY_LIST) p.glist_cap = std::min(h->glist_cap, 8u);
    const RecSet rs = rec_set(h);
    auto enqueue = [&]() -> int {
        int r2 = enqueue_filter(h, p, sampled, res);
        if (r2) return r2;
        if (use_hits) {
            with_recs(h, [&](auto rec) {
                constexpr bool R = decltype(rec)::value;
                if (vm == 0)
                    k_verify_hits<0, R><<<h->sm_count * 8, kHitThreads, 0, h->stream>>>(p, h->d_out.get(), h->d_out.size(),
                                                                                         h->d_counters.get(), rs);
                else if (vm == 1)
                    k_verify_hits<1, R><<<h->sm_count * 8, kHitThreads, 0, h->stream>>>(p, h->d_out.get(), h->d_out.size(),
                                                                                         h->d_counters.get(), rs);
                else
                    k_verify_hits<2, R><<<h->sm_count * 8, kHitThreads, 0, h->stream>>>(p, h->d_out.get(), h->d_out.size(),
                                                                                         h->d_counters.get(), rs);
            });
            res->stats.n_launches++;
            return FZB_OK;
        }
        {   // one verify launch: the granule work list -- or, second attempt after the list overflowed, the whole bitmap
            const int scan_mode = bitmap_mode ? 1 : 0;
            const int grid = h->sm_count * kVerifyCtasPerSm;
            with_recs(h, [&](auto rec) {
                constexpr bool R = decltype(rec)::value;
                if (vm == 0)
                    k_verify_lev<0, R><<<grid, kVerifyThreads, 0, h->stream>>>(p, h->d_bitmap.size(), h->d_glist.get(),
                                                                               p.glist_cap, scan_mode, h->d_out.get(),
                                                                               h->d_out.size(), h->d_counters.get(), rs);
                else if (vm == 1)
                    k_verify_lev<1, R><<<grid, kVerifyThreads, 0, h->stream>>>(p, h->d_bitmap.size(), h->d_glist.get(),
                                                                               p.glist_cap, scan_mode, h->d_out.get(),
                                                                               h->d_out.size(), h->d_counters.get(), rs);
                else
                    k_verify_lev<2, R><<<grid, kVerifyThreads, 0, h->stream>>>(p, h->d_bitmap.size(), h->d_glist.get(),
                                                                               p.glist_cap, scan_mode, h->d_out.get(),
                                                                               h->d_out.size(), h->d_counters.get(), rs);
            });
        }
        res->stats.n_launches += 1;
        return FZB_OK;
    };
    for (;;) {
        p.hits = use_hits ? h->d_hits.get() : nullptr;
        const uint32_t hits_cap = (uint32_t)h->d_hits.size();
        p.hits_cap = use_hits ? ((flags & FZB_F_TINY_LIST) ? std::min(hits_cap, 8u) : hits_cap) : 0;
        // (the raw stream's order (n-gram, hit index) is restored lazily)
        rc = run_emitting(h, res, enqueue, PostPlan{post_mode, fuse_gather});
        if (rc) return rc;
        if (!use_hits && !bitmap_mode && h->h_counters[CNT_GRAN] > p.glist_cap) {
            // more marked granules than the work list holds: the verify kernel raised CNT_OVERFLOW and did nothing (so a
            // fused reduction, if any, went out invalid); redo the search with the list switched off, sweeping the bitmap
            bitmap_mode = true;
            fuse_gather = false;
            p.glist_cap = 0;
        } else if (use_hits && h->h_counters[CNT_HITS] > p.hits_cap) {
            // the fused all-gather (if any) went out with valid = 0 (k_verify_hits raised CNT_OVERFLOW), so every
            // rank will take finish_global's staged round; the retry itself must not issue another collective
            fuse_gather = false;
            use_hits = false;
        } else {
            break;
        }
        res->discard_attempt();
    }
    res->raw_order = 0;
    return FZB_OK;
}

// ------------------------------------------------------------------------------------------------
// LP / generic routes (lp_kernels.cuh)
// ------------------------------------------------------------------------------------------------
// Grows the candidate lists to `words`: the new slab is allocated before the old one is released, so a failure leaves
// the handle with its previous slab.
static int ensure_scratch(fzb_haystack *h, uint64_t words) {
    return words <= h->d_scratch.size() ? FZB_OK : h->d_scratch.alloc(words);
}

// FZB_F_TINY_LIST (testing) caps the survivor list of the streaming LP search (and of the batch LP pass) at this many
// entries for that call only, so that tests reach its overflow fallback
constexpr uint32_t kTinyLpListCap = 1024;

// Per-thread candidate capacities of the LP-style searches: 256, 2 048, then kLpMaxCap entries per list.  The slab
// is threads x 2 lists x cap x 4 B: 17.7 GB at 16 384 with 132 SMs (4 CTAs of 256 threads each), 141 GB at the next
// step, so a start with more live candidates than kLpMaxCap fails the search.
constexpr int kLpMaxCap = 16384;

// Runs an LP-style search with growing per-thread candidate capacity until no list overflowed.
// `enqueue(grid, cap)` must put every kernel of one attempt on the stream.
template <class F>
static int run_lp(fzb_haystack *h, fzb_result *res, F enqueue, PostPlan post = PostPlan()) {
    const int grid = h->sm_count * 4;
    const uint64_t threads = (uint64_t)grid * kLpThreads;
    for (int cap = 256; cap <= kLpMaxCap; cap *= 8) {
        TRY(ensure_scratch(h, threads * 2 * (uint64_t)cap));
        TRY(run_emitting(h, res, [&]() -> int { return enqueue(grid, cap); }, post));
        if (!h->h_counters[CNT_OVERFLOW]) return FZB_OK;
    }
    return fail(FZB_E_UNSUPPORTED, "candidate explosion: more than 16384 live candidates for one start");
}

static int search_lev_lp(fzb_haystack *h, const uint8_t *pattern, const Plan &pl, uint32_t flags, fzb_result *res,
                         int post_mode) {
    const uint32_t m = pl.m, k = pl.k;
    ScanParams p;
    fill_params(h, pattern, m, p);
    p.k = (int)k;
    int rc;
    CK(cudaSetDevice(h->device));
    res->stats.route = 3;
    res->stats.bytes_scanned = h->buf_len;
    // streaming form (k_lp_scan + k_lp_verify) when the look-ahead masks cover the window; the list of surviving
    // starts overflowing (low-entropy data: most starts survive) falls back to the tile kernel
    bool streaming = k < m && m + k <= (uint32_t)kLpsMaxWin && !(flags & FZB_F_FORCE_DENSE) && h->buf_len > 0;
    if (streaming && !h->d_lplist)
        TRY(h->d_lplist.alloc(std::min<uint64_t>(std::max<uint64_t>(1u << 20, h->owned_buf.size() / 64), 1u << 26)));
    const PostPlan plan{post_mode, post_mode != 0 && (flags & FZB_F_GLOBAL) != 0};
    const RecSet rs = rec_set(h);
    if (streaming) {
        const uint32_t list_cap = (flags & FZB_F_TINY_LIST) ? std::min<uint32_t>(h->d_lplist.size(), kTinyLpListCap)
                                                            : (uint32_t)h->d_lplist.size();
        rc = run_lp(h, res, [&](int grid, int cap) -> int {
            k_lp_scan<<<h->sm_count * 4, kLpsThreads, 0, h->stream>>>(p, h->d_lplist.get(), list_cap);
            CK(cudaEventRecord(h->ev[1], h->stream));
            h->ev1_recorded = true;
            with_recs(h, [&](auto rec) {
                constexpr bool R = decltype(rec)::value;
                k_lp_verify<R><<<grid, kLpThreads, 0, h->stream>>>(p, h->d_lplist.get(), list_cap, h->d_scratch.get(), cap,
                                                                   h->d_out.get(), h->d_out.size(), h->d_counters.get(), rs);
            });
            res->stats.n_launches += 2;
            return FZB_OK;
        }, plan);
        if (rc) return rc;
        if (h->h_counters[CNT_LPWORK] == 0) {
            res->raw_order = 1;
            return FZB_OK;
        }
        res->discard_attempt();  // list overflow: nothing was verified (and the fused reduction saw an invalid shard)
    }
    rc = run_lp(h, res, [&](int grid, int cap) -> int {
        with_recs(h, [&](auto rec) {
            constexpr bool R = decltype(rec)::value;
            k_lev_lp<R><<<grid, kLpThreads, 0, h->stream>>>(p, h->d_scratch.get(), cap, h->d_out.get(), h->d_out.size(),
                                                            h->d_counters.get(), rs);
        });
        res->stats.n_launches++;
        return FZB_OK;
    }, plan);
    if (rc) return rc;
    res->raw_order = 1;
    return FZB_OK;
}

static int search_generic(fzb_haystack *h, const uint8_t *pattern, const Plan &pl, uint32_t flags, fzb_result *res,
                          int post_mode) {
    ScanParams p;
    fill_params(h, pattern, pl.m, p);
    p.k = (int)pl.k;
    p.max_subs = (int)pl.subs;
    p.max_ins = (int)pl.ins;
    p.max_dels = (int)pl.dels;
    int rc;
    CK(cudaSetDevice(h->device));
    res->stats.bytes_scanned = h->buf_len;
    const RecSet rs = rec_set(h);
    if (pl.route == Route::GenericLp) {
        res->stats.route = 6;
        rc = run_lp(h, res, [&](int grid, int cap) -> int {
            with_recs(h, [&](auto rec) {
                constexpr bool R = decltype(rec)::value;
                k_generic_lp<R><<<grid, kLpThreads, 0, h->stream>>>(p, h->d_scratch.get(), cap, h->d_out.get(),
                                                                    h->d_out.size(), h->d_counters.get(), rs);
            });
            res->stats.n_launches++;
            return FZB_OK;
        }, PostPlan{post_mode, post_mode != 0 && (flags & FZB_F_GLOBAL) != 0});
        if (rc) return rc;
        res->raw_order = 1;
        return FZB_OK;
    }
    p.L = (int)pl.L();
    p.n_ngrams = (int)pl.m / p.L;
    const bool sampled = sampled_filter(h, pl, flags);
    p.q = sampled ? 4 : std::min(p.L, 8);
    res->stats.route = 5;
    rc = set_filter_attrs(kScanSmem);
    if (rc) return rc;
    rc = run_lp(h, res, [&](int grid, int cap) -> int {
        int r2 = enqueue_filter(h, p, sampled, res);
        if (r2) return r2;
        with_recs(h, [&](auto rec) {
            constexpr bool R = decltype(rec)::value;
            k_verify_generic<R><<<grid, kLpThreads, 0, h->stream>>>(p, h->d_bitmap.size(), h->d_scratch.get(), cap,
                                                                    h->d_out.get(), h->d_out.size(), h->d_counters.get(), rs);
        });
        res->stats.n_launches++;
        return FZB_OK;
    }, PostPlan{post_mode, post_mode != 0 && (flags & FZB_F_GLOBAL) != 0});
    if (rc) return rc;
    res->raw_order = 2;  // n-gram major, hit index, then the window's matches in canonical order
    return FZB_OK;
}

// FZB_F_GLOBAL epilogue of every search entry point: turn the per-shard groups into the global final list.
// Fast path: k_push / k_merge already did it on the device (run_emitting).  Otherwise (no peer-memory world, a
// shard whose list overflowed a buffer, pathological chaining across seams) every rank arrives here and the
// rows go through the staged NCCL all-gather and the host merge.
static int finish_global(fzb_haystack *h, fzb_result *res) {
    if (h->world < 1 || (!h->comm && !h->local_world))
        return fail(FZB_E_INVALID, "FZB_F_GLOBAL needs fzb_haystack_comm_init / fzb_comm_init_local");
    if (res->fused_issued) {
        if (res->fused_status == MS_OK) {
            res->has_global = true;
            res->global_on_device = true;
            return FZB_OK;
        }
        if (res->fused_status == MS_TIMEOUT)
            return fail(FZB_E_CUDA, "multi-GPU reduction timed out waiting for a peer (rank %d of %d)", h->rank, h->world);
    }
    if (h->local_world && res->fused_issued && res->fused_status == MS_OVERFLOW)
        return fail(FZB_E_UNSUPPORTED, "NCCL-free world: more than %u groups continue across shard seams; the staged "
                    "fallback needs an NCCL communicator (fzb_haystack_comm_init)", kMaxNonHeads);
    if (h->local_world)
        return fail(FZB_E_UNSUPPORTED, "NCCL-free world: a shard produced more than %u groups (or more than %d raw "
                    "matches); the staged fallback needs an NCCL communicator (fzb_haystack_comm_init)", h->p2p_cap, kPostMax);
    std::vector<int64_t> all;
    std::vector<uint64_t> counts;
    std::vector<int64_t> rows(res->fin.size() * kFinCols);
    write_group_rows(res->fin, res->hulls, res->fin.size(), rows.data());
    int rc = allgather_groups_staged(h, rows, all, counts);
    if (rc) return rc;
    if (res->unconsolidated) {  // unconsolidated routes (exact, Hamming): the global list is the sorted union
        res->gfin.resize(all.size() / kFinCols);
        for (size_t i = 0; i < res->gfin.size(); i++)
            res->gfin[i] = make_rec(all[kFinCols * i], all[kFinCols * i + 1], all[kFinCols * i + 2]);
        sort_canonical(res->gfin);
    } else {
        sweep_groups(read_group_runs(all.data(), counts), res->gfin);
    }
    res->gcount = (uint32_t)res->gfin.size();
    res->has_global = true;
    return FZB_OK;
}

static int make_result(fzb_result **out, fzb_result **res) {
    if (!out) return fail(FZB_E_INVALID, "out is NULL");
    *out = nullptr;
    *res = new (std::nothrow) fzb_result();
    if (!*res) return fail(FZB_E_CUDA, "out of host memory");
    return FZB_OK;
}

static int search_hamming(fzb_haystack *h, const uint8_t *pattern, const Plan &pl, uint32_t flags, fzb_result *res);

// The route of plan `pl`, then the reduction to the global list under FZB_F_GLOBAL.  The final list of the exact and
// the Hamming search is their sorted raw list whatever the flags (ExactSearch.consolidate_matches is the base no-op,
// common.py:198-205); the others honour FZB_F_NO_FINAL (LevenshteinSearch.consolidate_matches,
// levenshtein.py:158-160, also applies when k == 0).
static int run_route(fzb_haystack *h, const uint8_t *pattern, const Plan &pl, uint32_t flags, fzb_result *res) {
    res->unconsolidated = pl.route == Route::Exact || pl.route == Route::Hamming;
    const int post_mode = res->unconsolidated ? 2 : (flags & FZB_F_NO_FINAL) ? 0 : 1;
    int rc = pl.route == Route::Hamming ? search_hamming(h, pattern, pl, flags, res)
             : pl.route == Route::LevLp ? search_lev_lp(h, pattern, pl, flags, res, post_mode)
             : pl.generic()             ? search_generic(h, pattern, pl, flags, res, post_mode)
                                        : search_lev_ngrams(h, pattern, pl, flags, res, post_mode);
    if (rc == FZB_OK && post_mode && (flags & FZB_F_GLOBAL)) rc = finish_global(h, res);
    return rc;
}

// The frame of the single searches: handle lock, result, `plan(pl)`, its route, and the result destroyed on any error.
template <class P>
static int run_search(fzb_haystack *h, const uint8_t *pattern, uint32_t flags, fzb_result **out, P plan) {
    HandleLock handle_lock(h);
    fzb_result *res;
    int rc = make_result(out, &res);
    if (rc) return rc;
    Plan pl;
    rc = plan(pl);
    if (rc == FZB_OK) rc = run_route(h, pattern, pl, flags, res);
    if (rc) {
        fzb_result_destroy(res);
        return rc;
    }
    *out = res;
    return FZB_OK;
}

extern "C" int fzb_search_levenshtein(fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t k,
                                      uint32_t flags, fzb_result **out) {
    return run_search(h, pattern, flags, out, [&](Plan &pl) { return plan_levenshtein(h, pattern, m, k, flags, pl); });
}

// ------------------------------------------------------------------------------------------------
// Batches: one scan for all the patterns the q-sample lemma covers (batch_kernels.cuh)
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kGtabSlots = 1u << 17;     // gram table (open addressing, <= 50 % full)
constexpr uint32_t kMaxBatchGrams = 60000;    // distinct grams of one pass
constexpr uint32_t kMaxBatchPostings = 1u << 20;
constexpr uint32_t kMaxBatchPats = 4096;      // patterns of one pass
// FZB_F_TINY_LIST (testing) shrinks, for that call only, the q-sample work list and the dense pass's hit list to
// kTinyBatchCap, the batch LP survivor list to kTinyLpListCap, and scans the LP starts in chunks of kTinyLpChunk (not
// a multiple of a tile or of 128: every chunk seam falls inside a tile), so that tests reach the overflow fallbacks
// and the chunk seams
constexpr uint32_t kTinyBatchCap = 8;
constexpr uint64_t kTinyLpChunk = 3000;

static int ensure_batch_buffers(fzb_haystack *h) {
    CK(cudaSetDevice(h->device));
    return ensure_group(h->batch, [](BatchBufs &b) -> int {
        TRY(b.d_mbits.alloc(kMultiTblWords + kMulti2Words));  // first + second level tables
        TRY(b.d_gtab.alloc(kGtabSlots));
        TRY(b.d_postings.alloc(kMaxBatchPostings));
        TRY(b.d_pinfo.alloc(kMaxBatchPats));
        TRY(b.d_bpats.alloc(kMaxBatchPats));
        TRY(b.d_mset.alloc(1u << 22));
        CK(cudaMemset(b.d_mset.get(), 0, b.d_mset.size() * sizeof(unsigned long long)));
        TRY(b.d_mwork.alloc(1u << 21));
        CK(cudaFuncSetAttribute(k_filter_multi, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMultiSmem));
        return FZB_OK;
    });
}

static int read_counters(fzb_haystack *h, uint32_t cnts[CNT_COUNT]) {
    CK(cudaMemcpyAsync(cnts, h->d_counters.get(), CNT_COUNT * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return FZB_OK;
}

static void add_stats(fzb_stats *sum, const fzb_stats &s) {
    sum->gpu_ms += s.gpu_ms;
    sum->filter_ms += s.filter_ms;
    sum->bytes_scanned += s.bytes_scanned;
    sum->n_candidates += s.n_candidates;
    sum->n_launches += s.n_launches;
}

// Splits the raw records of a pass over the patterns ids[] (`ngram` = pattern ordinal << 8 | n-gram) into the results
// out[ids[i]], consolidates each list (unconsolidated: FINAL is the raw list in canonical order, as the Hamming
// search returns it), and adds the pass to `sum`.  Every result carries the pass's route, the first one its other
// stats (the haystack is read once for the whole pass).
static int split_batch(const std::vector<RawRec> &raw, const std::vector<uint32_t> &ids, const fzb_stats &pass,
                       int raw_order, bool unconsolidated, fzb_result **out, fzb_stats *sum) {
    const uint32_t cnt = (uint32_t)ids.size();
    std::vector<uint32_t> per(cnt, 0);
    for (const RawRec &r : raw) per[(uint32_t)r.ngram >> 8]++;
    for (uint32_t i = 0; i < cnt; i++) {
        fzb_result *res = new (std::nothrow) fzb_result();
        if (!res) return fail(FZB_E_CUDA, "out of host memory");
        res->raw.reserve(per[i]);
        if (i == 0) res->stats = pass;
        res->stats.route = pass.route;
        res->raw_order = raw_order;
        out[ids[i]] = res;
    }
    for (const RawRec &r : raw) {
        RawRec q = r;
        q.ngram = r.ngram & 0xFF;
        out[ids[(uint32_t)r.ngram >> 8]]->raw.push_back(q);
    }
    // consolidate the lists in parallel (LP patterns on text have tens of thousands of raw matches each)
    const unsigned nthreads = std::min<unsigned>({8u, std::max(1u, std::thread::hardware_concurrency()), cnt});
    std::atomic<uint32_t> next{0};
    auto work = [&]() {
        for (uint32_t i = next.fetch_add(1); i < cnt; i = next.fetch_add(1)) {
            fzb_result *res = out[ids[i]];
            res->raw_n = (uint32_t)res->raw.size();
            res->unconsolidated = unconsolidated;
            if (unconsolidated)
                finalize_on_host(res, 2);
            else
                consolidate_recs(res->raw, res->fin, &res->hulls);
            res->have_fin = true;
        }
    };
    std::vector<std::thread> pool;
    for (unsigned t = 1; t < nthreads; t++) pool.emplace_back(work);
    work();
    for (auto &t : pool) t.join();
    add_stats(sum, pass);
    return FZB_OK;
}

// The n raw records in h->d_out reduced into the words of `best`: those of a shared pass whose pattern j is pattern
// d_ids[j] of the fzb_best_per_record call, or (d_ids == nullptr) those of a single search of pattern `id`.
static int best_accumulate(fzb_haystack *h, const BestState &best, uint32_t n, const uint32_t *d_ids, uint32_t id) {
    if (n == 0) return FZB_OK;
    const int grid = (int)std::min<uint32_t>((n + kBestThreads - 1) / kBestThreads, (uint32_t)h->sm_count * 8);
    if (d_ids)
        k_best_accumulate<true><<<grid, kBestThreads, 0, h->stream>>>(h->d_out.get(), n, rec_set(h), d_ids, id,
                                                                     best.best, best.top2);
    else
        k_best_accumulate<false><<<grid, kBestThreads, 0, h->stream>>>(h->d_out.get(), n, rec_set(h), d_ids, id,
                                                                      best.best, best.top2);
    CK(cudaGetLastError());
    return FZB_OK;
}

// One batch call: a batch entry point's, or one class of fzb_best_per_record's.  It holds the patterns and their
// plans, what the flags let the passes do, the running sum of the stats and the sink the passes and the one-by-one
// searches end in: the per-pattern results out[count], or (best != nullptr) the words of fzb_best_per_record, into
// which every record is reduced (DESIGN.md section 5.13).
struct BatchCall {
    fzb_haystack *h;
    const uint8_t *patterns;
    const uint32_t *offsets;
    uint32_t count, flags;
    std::vector<Plan> plans;  // plans[i]: how pattern i is searched, in a pass or on its own
    fzb_result **out;        // list sink: out[i] is pattern i's result once a pass or its own search settled it
    const BestState *best;   // reduction sink
    std::vector<uint8_t> done;  // reduction sink: pattern i is settled
    // FZB_F_TINY_LIST (testing) shrinks the capacities of the shared passes; the passes take no other flag than that
    // and FZB_F_PER_RECORD (forced routes, raw-only, the multi-GPU reduction: one by one)
    bool tiny, share;
    fzb_stats sum{};

    BatchCall(fzb_haystack *h_, const uint8_t *p, const uint32_t *o, uint32_t n, uint32_t f, fzb_result **out_,
              const BestState *best_)
        : h(h_), patterns(p), offsets(o), count(n), flags(f), out(out_), best(best_), done(best_ ? n : 0, 0),
          tiny((f & FZB_F_TINY_LIST) != 0), share((f & ~(FZB_F_TINY_LIST | FZB_F_PER_RECORD)) == 0 && h_->buf_len > 0) {}

    uint32_t len(uint32_t i) const { return offsets[i + 1] - offsets[i]; }
    bool settled(uint32_t i) const { return best ? done[i] != 0 : out[i] != nullptr; }

    // The refusals of the batch entry points, behind every result cleared; then every pattern planned by
    // `plan(i, pattern, m, pl)`, the class's plan function, whose first refusal fails the call before any work.
    template <class P>
    int begin(P plan) {
        for (uint32_t i = 0; i < count; i++) out[i] = nullptr;
        TRY(check_batch_records(h, flags));
        for (uint32_t i = 0; i < count; i++)
            if (offsets[i + 1] < offsets[i]) return fail(FZB_E_INVALID, "offsets must be non-decreasing");
        plans.resize(count);
        for (uint32_t i = 0; i < count; i++) TRY(plan(i, patterns + offsets[i], len(i), plans[i]));
        return FZB_OK;
    }

    // The outcome `rc` of a shared pass over the patterns ids[]: an error drops every result; an overflow (+1) drops
    // the pass's results, leaving its patterns to the one-by-one searches.
    int settle(int rc, const std::vector<uint32_t> &ids) {
        auto drop = [&](uint32_t j) {
            if (!out) return;  // (the reduction sink keeps no results)
            fzb_result_destroy(out[j]);
            out[j] = nullptr;
        };
        if (rc < 0)
            for (uint32_t j = 0; j < count; j++) drop(j);
        if (rc > 0)
            for (uint32_t id : ids) drop(id);
        return rc < 0 ? rc : FZB_OK;
    }

    // What a pass over the patterns ids[] ends with: the per-pattern results of split_batch or its n raw records
    // reduced where they are, and its stats in the sum.  Every way a pass can still overflow (+1) lies before this
    // point (for the chunked passes: behind the last chunk), so a pass that is redone pattern by pattern has
    // contributed nothing.
    int finish_pass(const std::vector<RawRec> &raw, uint32_t n, const std::vector<uint32_t> &ids, fzb_stats pass,
                    int raw_order, bool unconsolidated) {
        if (!best) return split_batch(raw, ids, pass, raw_order, unconsolidated, out, &sum);
        if (n) {
            std::vector<uint32_t> ordinals(ids.size());
            for (size_t j = 0; j < ids.size(); j++) ordinals[j] = best->ordinal[ids[j]];
            // (a pageable source: the copy has left the vector when it returns)
            CK(cudaMemcpyAsync(h->bestb->d_ids.get(), ordinals.data(), ordinals.size() * sizeof(uint32_t),
                               cudaMemcpyHostToDevice, h->stream));
            TRY(best_accumulate(h, *best, n, h->bestb->d_ids.get(), 0));
            pass.n_launches++;
        }
        for (uint32_t id : ids) done[id] = 1;
        add_stats(&sum, pass);
        return FZB_OK;
    }

    // The patterns no pass settled, each searched on its own by its plan's route (which honours a record set by
    // itself); then the call's stats in *total.  Under the reduction sink the search returns the raw stream only, which
    // is reduced while still in h->d_out and dropped, so that nothing reads it back.
    int finish(fzb_stats *total) {
        const uint32_t f = (flags & ~FZB_F_PER_RECORD) | (best ? FZB_F_NO_FINAL : 0u);
        for (uint32_t i = 0; i < count; i++) {
            if (settled(i)) continue;
            fzb_result *res = nullptr;
            auto planned = [&](Plan &pl) { pl = plans[i]; return FZB_OK; };
            TRY(settle(run_search(h, patterns + offsets[i], f, &res, planned), {}));
            if (!best) {
                add_stats(&sum, res->stats);
                out[i] = res;
                continue;
            }
            // (destroying the result unlinks it from the handle: nothing fetches the records it leaves in h->d_out)
            const int rc = best_accumulate(h, *best, res->raw_n, nullptr, best->ordinal[i]);
            if (res->raw_n) res->stats.n_launches++;
            add_stats(&sum, res->stats);
            fzb_result_destroy(res);
            TRY(rc);
        }
        sum.route = 7;  // batch
        if (total) *total = sum;
        return FZB_OK;
    }
};

// The attempt loop of a batch pass.  `enqueue()` puts the kernels of one attempt on h->stream (behind h->ev[0]) and
// returns FZB_OK, an error, or +1 when a device structure of the pass overflowed.  Returns the same, +1 also when a
// kernel raised CNT_OVERFLOW or the pass emitted more than kMaxRawRecs records; an attempt whose raw records did not
// fit the output buffer is redone with a larger one.  On FZB_OK `raw` holds the records (under the reduction sink they
// stay in h->d_out and `raw` stays empty), `cnts` the counters, and `pass` the time and the bytes scanned.
template <class F>
static int run_batch_pass(const BatchCall &c, F enqueue, std::vector<RawRec> &raw, uint32_t cnts[CNT_COUNT],
                          fzb_stats &pass) {
    fzb_haystack *h = c.h;
    detach_pending(h);  // the kernels are about to overwrite the output buffer an earlier result may still point at
    for (int attempt = 0; attempt < 8; attempt++) {
        h->counters_clean = false;  // (a batch pass leaves its counters behind)
        CK(cudaMemsetAsync(h->d_counters.get(), 0, CNT_COUNT * sizeof(uint32_t), h->stream));
        CK(cudaEventRecord(h->ev[0], h->stream));
        int rc = enqueue();
        if (rc) return rc;
        CK(cudaEventRecord(h->ev[2], h->stream));
        rc = read_counters(h, cnts);
        if (rc) return rc;
        if (cnts[CNT_OVERFLOW]) return 1;
        const uint32_t n = cnts[CNT_OUT];
        // more records than one search may return, over all the patterns of the pass: they go one by one, where
        // each pattern only has to stay within the limit on its own
        if (n > kMaxRawRecs) return 1;
        if (n > h->d_out.size()) {
            TRY(ensure_out_cap(h, n));
            continue;
        }
        if (!c.best) raw.resize(n);  // (the reduction sink reduces the records where they are: finish_pass)
        if (!raw.empty()) {
            CK(cudaMemcpyAsync(raw.data(), h->d_out.get(), (size_t)n * sizeof(RawRec), cudaMemcpyDeviceToHost, h->stream));
            CK(cudaStreamSynchronize(h->stream));
        }
        float ms = 0.f;
        cudaEventElapsedTime(&ms, h->ev[0], h->ev[2]);
        pass.gpu_ms = ms;
        pass.bytes_scanned = h->buf_len;
        return FZB_OK;
    }
    return fail(FZB_E_CUDA, "output buffer kept overflowing");
}

// The scan times, list lengths and chunks of one attempt of a chunked pass (run_chunks).
struct ChunkSums {
    float scan_ms = 0.f;
    uint64_t listed = 0;  // (over all chunks: more than 2^32 on a large haystack)
    uint32_t chunks = 0;
};

// One attempt of a chunked pass (LP, 2-bit) over the own range in chunks of `chunk` positions: per chunk the counters
// cnts[list] (the scan's list) and the one after it cleared, `scan(lo, hi)` between h->ev[1] and h->ev[2], `verify()`,
// and the counters read back into cnts.  Returns FZB_OK, an error, or +1 at the first chunk whose kernels raised
// CNT_OVERFLOW or the counter `full` (a list too small for the chunk).
template <class S, class V>
static int run_chunks(fzb_haystack *h, uint64_t chunk, int list, int full, uint32_t cnts[CNT_COUNT], ChunkSums &s,
                      S scan, V verify) {
    s = ChunkSums{};
    for (uint64_t lo = h->own_lo; lo < h->own_hi; lo += chunk) {
        CK(cudaMemsetAsync(h->d_counters.get() + list, 0, 2 * sizeof(uint32_t), h->stream));
        CK(cudaEventRecord(h->ev[1], h->stream));
        scan(lo, std::min<uint64_t>(h->own_hi, lo + chunk));
        CK(cudaEventRecord(h->ev[2], h->stream));
        TRY(verify());
        CK(cudaGetLastError());
        s.chunks++;
        TRY(read_counters(h, cnts));
        float ms = 0.f;
        cudaEventElapsedTime(&ms, h->ev[1], h->ev[2]);
        s.scan_ms += ms;
        s.listed += cnts[list];
        if (cnts[CNT_OVERFLOW] || cnts[full]) return 1;
    }
    return FZB_OK;
}

// The slot of pattern `id` in a pass, with its plan's limit; the pass sets its L and n_ngrams.
static void fill_pat(BatchPat &bp, const BatchCall &c, uint32_t id) {
    memset(&bp, 0, sizeof bp);
    memcpy(bp.P, c.patterns + c.offsets[id], c.len(id));
    bp.m = (int)c.len(id);
    bp.k = (int)c.plans[id].k;
}

// Builds the posting table of a pass -- open addressing on the key (key * kGramMul), each slot the key and its first
// posting | count << 24, a key with more than 255 postings spilling into further slots -- lets `mark(key)` set the
// key's bits in `bits`, and uploads bits, table, postings, pinfo and the patterns.
template <class F>
static int upload_pass_tables(fzb_haystack *h, const std::unordered_map<uint32_t, std::vector<uint32_t>> &grams,
                              const std::vector<uint32_t> &bits, const std::vector<uint32_t> &pinfo,
                              const std::vector<BatchPat> &pats, F mark) {
    std::vector<uint32_t> postings;
    std::vector<uint2> gtab(kGtabSlots, make_uint2(0, 0));
    for (auto &g : grams) {
        const uint32_t w = g.first;
        mark(w);
        for (size_t first = 0; first < g.second.size(); first += 255) {
            const uint32_t c = (uint32_t)std::min<size_t>(255, g.second.size() - first);
            uint32_t slot = (w * kGramMul) & (kGtabSlots - 1);
            while (gtab[slot].y != 0u) slot = (slot + 1) & (kGtabSlots - 1);
            gtab[slot] = make_uint2(w, (uint32_t)postings.size() | (c << 24));
            postings.insert(postings.end(), g.second.begin() + first, g.second.begin() + first + c);
        }
    }
    TRY(ensure_batch_buffers(h));  // (makes the handle's device current)
    BatchBufs &b = *h->batch;
    CK(cudaMemcpyAsync(b.d_mbits.get(), bits.data(), bits.size() * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(b.d_gtab.get(), gtab.data(), gtab.size() * sizeof(uint2), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(b.d_postings.get(), postings.data(), postings.size() * 4, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(b.d_pinfo.get(), pinfo.data(), pinfo.size() * 4, cudaMemcpyHostToDevice, h->stream));
    // (pageable sources: each copy has left its host vector when it returns)
    CK(cudaMemcpyAsync(b.d_bpats.get(), pats.data(), pats.size() * sizeof(BatchPat), cudaMemcpyHostToDevice, h->stream));
    return FZB_OK;
}

// The handle's geometry and the uploaded tables as the pass kernels see them.
static MultiParams pass_params(const fzb_haystack *h) {
    MultiParams mp{};
    mp.H = h->d;
    mp.buf_lo = (int64_t)h->buf_lo;
    mp.buf_len = (int64_t)h->buf_len;
    mp.N = (int64_t)h->global_len;
    mp.own_lo = (int64_t)h->own_lo;
    mp.own_hi = (int64_t)h->own_hi;
    mp.bits = h->batch->d_mbits.get();
    mp.gtab = h->batch->d_gtab.get();
    mp.gtab_mask = kGtabSlots - 1;
    mp.postings = h->batch->d_postings.get();
    mp.pinfo = h->batch->d_pinfo.get();
    mp.counters = h->d_counters.get();
    return mp;
}

// Entries of each of a lane's two candidate lists in the verify kernels of a generic pass: a start with more live
// candidates sends the pass's patterns one by one, where the single search grows its lists
constexpr int kGenericBatchCap = 256;

// A generic pass: uploads the per-operation limits of the plans of the patterns ids[] (subs | ins << 8 | dels << 16)
// and sizes the candidate lists of `grid` CTAs of the verify kernel.
static int prepare_generic_pass(const BatchCall &c, const std::vector<uint32_t> &ids, int grid) {
    fzb_haystack *h = c.h;
    TRY(ensure_group(h->gbatch, [](GenericBatchBufs &g) -> int { return g.d_glim.alloc(kMaxBatchPats); }));
    std::vector<uint32_t> lim;
    for (uint32_t id : ids) lim.push_back(c.plans[id].subs | c.plans[id].ins << 8 | c.plans[id].dels << 16);
    CK(cudaMemcpyAsync(h->gbatch->d_glim.get(), lim.data(), lim.size() * 4, cudaMemcpyHostToDevice, h->stream));
    return ensure_scratch(h, (uint64_t)grid * kLpThreads * 2 * kGenericBatchCap);
}

// The hit list of the dense passes (k_filter_mdense, k_filter_mdense2), taken by the handle only together with the
// shared-memory attribute of k_filter_mdense.
static int ensure_mhits(fzb_haystack *h) {
    if (h->d_mhits) return FZB_OK;
    DevBuf<unsigned long long> hits;
    TRY(hits.alloc(1u << 23));
    CK(cudaFuncSetAttribute(k_filter_mdense, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMdenseSmem));
    h->d_mhits = std::move(hits);
    return FZB_OK;
}

// 2-bit keys of a pass over a low-entropy haystack (k_ham_batch_scan<true>, k_filter_mdense2): the four most frequent
// pattern bytes of the pass get codes 0..3, every other byte code 0 (DNA reduced from a wide str arrives as bytes
// 1..4).  two_bit_key enters `post` under the key of the first min(L, 8) symbols at s, under every completion of
// the remaining ones.
static void two_bit_code(const uint8_t *patterns, const uint32_t *offsets, const std::vector<uint32_t> &ids,
                         uint8_t code[256]) {
    uint64_t freq[256] = {0};
    for (uint32_t id : ids)
        for (uint32_t b = offsets[id]; b < offsets[id + 1]; b++) freq[patterns[b]]++;
    int order[256];
    for (int c = 0; c < 256; c++) order[c] = c;
    std::stable_sort(order, order + 256, [&](int a, int b) { return freq[a] > freq[b]; });
    for (int c = 0; c < 256; c++) code[c] = 0;
    for (int r = 0; r < 4; r++) code[order[r]] = (uint8_t)r;
}

static void two_bit_key(std::unordered_map<uint32_t, std::vector<uint32_t>> &keys, const uint8_t code[256],
                        const uint8_t *s, uint32_t L, uint32_t post) {
    const uint32_t n = std::min<uint32_t>(L, kHbKeySyms);
    uint32_t key = 0;
    for (uint32_t q = 0; q < n; q++) key |= (uint32_t)code[s[q]] << (2 * q);
    for (uint32_t x = 0; x < (1u << (2 * (kHbKeySyms - n))); x++) keys[key | (x << (2 * n))].push_back(post);
}

// One pass over the haystack for the patterns ids[0..cnt): settles them in the call's sink.  Returns FZB_OK, an
// error, or +1 if the pass overflowed a device structure (the caller then searches these patterns one by one).
// dense = false: the q-sample scan (k_filter_multi / k_verify_multi) over the 4-grams of the patterns;
// dense = true: the n-gram-prefix scan at every position (k_filter_mdense / k_verify_mhits).
// Generic patterns (the generic n-gram route) take the generic verify kernels (k_verify_multi_generic /
// k_verify_mhits_generic) with their plans' per-operation limits.
static int batch_pass(BatchCall &c, const std::vector<uint32_t> &ids, bool dense) {
    fzb_haystack *h = c.h;
    const uint32_t cnt = (uint32_t)ids.size();
    const bool generic = c.plans[ids[0]].generic();
    std::vector<BatchPat> pats(cnt);
    std::vector<uint32_t> pinfo(cnt);
    std::unordered_map<uint32_t, std::vector<uint32_t>> grams;
    grams.reserve(cnt * 48);
    for (uint32_t i = 0; i < cnt; i++) {
        const uint32_t id = ids[i], m = c.len(id), k = c.plans[id].k;
        BatchPat &bp = pats[i];
        fill_pat(bp, c, id);
        bp.L = (int)c.plans[id].L();
        bp.n_ngrams = (int)m / bp.L;
        // The k of pinfo only sets the anchors k_filter_multi marks around a word hit, [g-o-k, g-o+k+m-L].  A generic
        // pattern needs 2k there: its verification runs the NFA from every start of the window [p0-k, p0+m+k) of an
        // n-gram hit, whose end is also the NFA's end of input, so a match that aligns the word with offset o can
        // start anywhere in [g-o-ins, g-o+dels] and its hit p0 anywhere in [g-o-k-dels, g-o+k+dels] (ins + dels <= k).
        const uint32_t mark_k = generic ? 2 * k : k;  // (n-gram route, m <= 64: k <= 20)
        pinfo[i] = m | (mark_k << 8) | ((uint32_t)bp.L << 16);
        if (dense) {  // key: the first 3 bytes of n-gram j; posting: pattern << 8 | j
            for (int j = 0; j < bp.n_ngrams; j++) {
                uint32_t w = 0;
                memcpy(&w, bp.P + j * bp.L, 3);
                grams[w].push_back((i << 8) | (uint32_t)j);
            }
        } else {
            for (uint32_t o = 0; o + 4 <= m; o++) {
                uint32_t w;
                memcpy(&w, bp.P + o, 4);
                grams[w].push_back((i << 8) | o);
            }
        }
    }
    std::vector<uint32_t> bits(kMultiTblWords + (dense ? 0 : kMulti2Words), 0);
    int rc = upload_pass_tables(h, grams, bits, pinfo, pats, [&](uint32_t w) {
        const uint32_t hb = (w * kHashMul) >> (32 - kMultiTblBits);
        bits[hb >> 5] |= 1u << (hb & 31u);
        if (!dense) {
            const uint32_t h2 = multi_hash2(w);
            bits[kMultiTblWords + (h2 >> 5)] |= 1u << (h2 & 31u);
        }
    });
    if (rc) return rc;
    if (dense) TRY(ensure_mhits(h));
    const int ggrid = h->sm_count * 4;  // generic verify kernels: as many lanes (and candidate lists) as run_lp's
    if (generic) TRY(prepare_generic_pass(c, ids, ggrid));
    BatchBufs &b = *h->batch;
    MultiParams mp = pass_params(h);
    mp.bits2 = dense ? nullptr : b.d_mbits.get() + kMultiTblWords;
    mp.set = b.d_mset.get();
    mp.set_mask = (uint32_t)b.d_mset.size() - 1;
    mp.work = b.d_mwork.get();
    mp.work_cap = c.tiny ? std::min<uint32_t>(b.d_mwork.size(), kTinyBatchCap) : (uint32_t)b.d_mwork.size();
    const uint32_t hits_cap = c.tiny ? std::min<uint32_t>(h->d_mhits.size(), kTinyBatchCap) : (uint32_t)h->d_mhits.size();
    const int64_t nvec = (int64_t)(round_up(h->buf_len, 16) / 16);
    const int64_t ntiles = (nvec + kMultiTileVecs - 1) / kMultiTileVecs;
    std::vector<RawRec> raw;
    uint32_t cnts[CNT_COUNT];
    fzb_stats pass{};
    const RecSet rs = rec_set(h);  // (the filters only look at content: only the verify kernels take it)
    rc = run_batch_pass(c, [&]() -> int {
        MdenseParams dp{mp, b.d_bpats.get(), h->d_mhits.get(), hits_cap};
        if (ntiles > 0) {
            const int grid = (int)std::min<int64_t>(ntiles, h->sm_count);
            if (dense)
                k_filter_mdense<<<grid, kMultiThreads, kMdenseSmem, h->stream>>>(dp, nvec, ntiles);
            else
                k_filter_multi<<<grid, kMultiThreads, kMultiSmem, h->stream>>>(mp, nvec, ntiles);
        }
        CK(cudaEventRecord(h->ev[1], h->stream));
        with_recs(h, [&](auto rec) {
            constexpr bool R = decltype(rec)::value;
            if (generic && dense)
                k_verify_mhits_generic<R><<<ggrid, kLpThreads, 0, h->stream>>>(
                    dp, h->gbatch->d_glim.get(), h->d_scratch.get(), kGenericBatchCap, h->d_out.get(), h->d_out.size(),
                    h->d_counters.get(), rs);
            else if (generic)
                k_verify_multi_generic<R><<<ggrid, kLpThreads, 0, h->stream>>>(
                    mp, b.d_bpats.get(), h->gbatch->d_glim.get(), h->d_scratch.get(), kGenericBatchCap, h->d_out.get(),
                    h->d_out.size(), h->d_counters.get(), rs);
            else if (dense)
                k_verify_mhits<R><<<h->sm_count * 8, kMhThreads, 0, h->stream>>>(dp, h->d_out.get(), h->d_out.size(),
                                                                                    h->d_counters.get(), rs);
            else
                k_verify_multi<R><<<h->sm_count * 8, kVmThreads, 0, h->stream>>>(
                    mp, b.d_bpats.get(), h->d_out.get(), h->d_out.size(), h->d_counters.get(), rs);
        });
        CK(cudaGetLastError());
        return FZB_OK;
    }, raw, cnts, pass);
    if (rc > 0 && !dense) {  // work list / set too small for this batch: clean up, let the caller go one by one
        CK(cudaMemsetAsync(b.d_mset.get(), 0, b.d_mset.size() * sizeof(unsigned long long), h->stream));
        CK(cudaStreamSynchronize(h->stream));
    }
    if (rc) return rc;
    float filter_ms = 0.f;
    cudaEventElapsedTime(&filter_ms, h->ev[0], h->ev[1]);
    pass.route = generic ? 9 : dense ? 2 : 1;
    pass.filter_ms = filter_ms;
    pass.n_candidates = cnts[CNT_CAND];
    pass.n_launches = 2;
    // (the generic n-gram route's raw order: n-gram, hit index, then the window's matches in canonical order)
    return c.finish_pass(raw, cnts[CNT_OUT], ids, pass, generic ? 2 : 0, false);
}

// One shared scan for up to 64 LP-route patterns (k_lp_scan_multi / k_lp_verify_multi).  Same return convention
// as batch_pass.  Generic patterns (the generic LP route, with their plans' lowered limits): a generic NFA opens a
// candidate at every start (generic_search.py:81), so the scan applies the counting condition only, and
// k_lp_verify_multi_generic verifies.
static int batch_pass_lp(BatchCall &c, const std::vector<uint32_t> &ids) {
    fzb_haystack *h = c.h;
    const uint32_t cnt = (uint32_t)ids.size();
    const bool generic = c.plans[ids[0]].generic();
    std::vector<BatchPat> pats(cnt);
    std::vector<ulonglong2> lut(256, make_ulonglong2(0ull, 0ull));
    std::vector<uint32_t> pm32((size_t)cnt * 256, 0u);
    LpMultiParams lp{};
    int wmax = 0;
    uint32_t kmax = 0;
    for (uint32_t i = 0; i < cnt; i++) {
        const uint32_t id = ids[i], m = c.len(id), k = c.plans[id].k;
        BatchPat &bp = pats[i];
        fill_pat(bp, c, id);  // (L = n_ngrams = 0: no n-grams)
        for (uint32_t j = 0; j < m; j++) {
            lut[bp.P[j]].x |= 1ull << i;
            pm32[(size_t)i * 256 + bp.P[j]] |= 1u << j;
        }
        if (generic)
            for (int c = 0; c < 256; c++) lut[c].y |= 1ull << i;
        else
            for (uint32_t j = 0; j <= std::min(k, m - 1); j++) lut[bp.P[j]].y |= 1ull << i;
        const uint32_t bias = 32 - (m - k);  // need = m - k in [1, 31]
        for (int b = 0; b < 6; b++)
            if ((bias >> b) & 1u) lp.bias[b] |= 1ull << i;
        wmax = std::max(wmax, (int)(m + k));
        kmax = std::max(kmax, k);
    }
    TRY(ensure_batch_buffers(h));  // (makes the handle's device current)
    TRY(ensure_group(h->lpb, [&](LpBatchBufs &l) -> int {
        TRY(l.d_lmlut.alloc(256, 256 * sizeof(ulonglong2) + 64 * 256 * sizeof(uint32_t)));  // vectors + match masks
        const uint64_t list_cap = std::min<uint64_t>(1u << 26, std::max<uint64_t>(1u << 22, h->owned_buf.size() / 16));
        TRY(l.d_lmlist.alloc(list_cap));
        TRY(l.d_lmkept.alloc(list_cap));
        TRY(l.d_lmhist.alloc(256));
        CK(cudaFuncSetAttribute(k_lp_scan_multi, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kLmSmem));
        return FZB_OK;
    }));
    LpBatchBufs &lb = *h->lpb;
    CK(cudaMemcpyAsync(lb.d_lmlut.get(), lut.data(), 256 * sizeof(ulonglong2), cudaMemcpyHostToDevice, h->stream));
    uint32_t *d_pm32 = reinterpret_cast<uint32_t *>(lb.d_lmlut.get() + 256);
    CK(cudaMemcpyAsync(d_pm32, pm32.data(), pm32.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(h->batch->d_bpats.get(), pats.data(), pats.size() * sizeof(BatchPat), cudaMemcpyHostToDevice, h->stream));
    lp.H = h->d;
    lp.buf_lo = (int64_t)h->buf_lo;
    lp.buf_len = (int64_t)h->buf_len;
    lp.N = (int64_t)h->global_len;
    lp.lut = lb.d_lmlut.get();
    lp.wmax = wmax;
    lp.pats = h->batch->d_bpats.get();
    lp.pm32 = d_pm32;
    lp.list = lb.d_lmlist.get();
    lp.list_cap = c.tiny ? std::min<uint32_t>(lb.d_lmlist.size(), kTinyLpListCap) : (uint32_t)lb.d_lmlist.size();
    lp.counters = h->d_counters.get();
    int per_sm = 2;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_lp_scan_multi, kLmThreads, kLmSmem));
    per_sm = std::max(per_sm, 1);
    const int vgrid = h->sm_count * 4, sim_cap = 256;
    if (generic)
        TRY(prepare_generic_pass(c, ids, vgrid));
    else
        TRY(ensure_scratch(h, (uint64_t)vgrid * kLpThreads * 2 * sim_cap));
    const uint64_t chunk = c.tiny ? kTinyLpChunk : 256ull << 20;  // starts per scan: bounds the survivor list
    std::vector<RawRec> raw;
    uint32_t cnts[CNT_COUNT];
    fzb_stats pass{};
    const RecSet rs = rec_set(h);  // (verify kernels only)
    ChunkSums cs;
    int rc = run_batch_pass(c, [&]() -> int {
        // CNT_LMWORK: the scan's list overflowed
        return run_chunks(h, chunk, CNT_LMLIST, CNT_LMWORK, cnts, cs, [&](uint64_t lo, uint64_t hi) {
            lp.own_lo = (int64_t)lo;
            lp.own_hi = (int64_t)hi;
            k_lp_scan_multi<<<h->sm_count * per_sm, kLmThreads, kLmSmem, h->stream>>>(lp);
        }, [&]() -> int {
            CK(cudaMemsetAsync(h->d_counters.get() + CNT_LMNEXT, 0, sizeof(uint32_t), h->stream));  // verify work counter
            // exact per-pattern windows, then a counting sort by pattern: the scan's list becomes the sorted output
            CK(cudaMemsetAsync(lb.d_lmhist.get(), 0, 256 * sizeof(uint32_t), h->stream));
            k_lm_refine<<<h->sm_count * 8, kLmSortThreads, 0, h->stream>>>(lp, lb.d_lmkept.get(), lb.d_lmhist.get());
            k_lm_scatter<<<h->sm_count * 8, kLmSortThreads, 0, h->stream>>>(lb.d_lmkept.get(), lb.d_lmhist.get(),
                                                                              lb.d_lmhist.get() + 128, lb.d_lmlist.get());
            with_recs(h, [&](auto rec) {
                constexpr bool R = decltype(rec)::value;
                if (generic)
                    k_lp_verify_multi_generic<R><<<vgrid, kLpThreads, 0, h->stream>>>(
                        lp, h->gbatch->d_glim.get(), lb.d_lmlist.get(), lb.d_lmhist.get(), h->d_scratch.get(),
                        kGenericBatchCap, h->d_out.get(), h->d_out.size(), h->d_counters.get(), rs);
                else if (kmax <= 4)
                    k_lp_verify_multi<4, R><<<vgrid, kLpThreads, 0, h->stream>>>(
                        lp, lb.d_lmlist.get(), lb.d_lmhist.get(), h->d_scratch.get(), sim_cap, h->d_out.get(),
                        h->d_out.size(), h->d_counters.get(), rs);
                else
                    k_lp_verify_multi<8, R><<<vgrid, kLpThreads, 0, h->stream>>>(
                        lp, lb.d_lmlist.get(), lb.d_lmhist.get(), h->d_scratch.get(), sim_cap, h->d_out.get(),
                        h->d_out.size(), h->d_counters.get(), rs);
            });
            return FZB_OK;
        });
    }, raw, cnts, pass);
    if (rc) return rc;
    pass.route = generic ? 10 : 3;
    pass.filter_ms = cs.scan_ms;
    pass.n_candidates = cs.listed;
    pass.n_launches = 4 * cs.chunks;
    return c.finish_pass(raw, cnts[CNT_OUT], ids, pass, 1, false);
}

// Admission of n-gram-route Levenshtein patterns to the 2-bit pass (k_filter_mdense2 / k_verify_mhits) on
// low-entropy haystacks: a pattern rides when its work in the pass costs less than its own search.  Per haystack
// position it walks n_ngrams * max(c, 1/4)^min(L, 8) postings and verifies n_ngrams * c^L exact n-gram hits
// (c: collision probability); its own search costs a fixed part, a read of the haystack and a verification per hit.
// Measured on an H100 80GB HBM3 (700 W power limit) with tools/probe_dna_lev_batch.py (DESIGN.md section 5.12):
// - in a pass of 1 024 patterns over 4 GiB of DNA: 0.53 ns of scan per posting walked (almost every posting is an
//   exact hit there, so this includes the byte comparison and the append) and 0.31 ns per hit beyond the scans
//   (verification and the host turnaround between chunks);
// - alone: 1.98 ms + 0.29 ns per hit on 4 GiB (least squares over the 1 024 searches) and 0.196 ms per search on
//   1.5e8 bytes of reads with few hits, i.e. 0.13 ms + 4.3e-4 ns per position.
// So on 4 GiB a pattern with n-grams of 5 symbols costs more in the pass than alone (measured: 52 such patterns
// added 773 ms to the pass against 296 ms searched alone), one with n-grams of 6 symbols less (93 ms against 136 ms).
constexpr double kDnaLevPostNs = 0.53;
constexpr double kDnaLevHitNs = 0.31;
constexpr double kDnaLevAloneMs = 0.13;
constexpr double kDnaLevAloneReadNs = 4.3e-4;
constexpr double kDnaLevAloneHitNs = 0.29;
// Not a cost bound: a pass closes at 4 expected hits per position, so that even a chunk of one 64 KiB tile expects at
// most 2.6e5 hits, far inside the hit list.
constexpr double kDnaLevPassHits = 4.0;
constexpr uint32_t kDnaLevMinL = 5;    // n-grams of at least 5 symbols: at most 64 completions of a key

static uint32_t dna_lev_postings(const Plan &p) {
    return (p.m / p.L()) << (2 * (kHbKeySyms - std::min<uint32_t>(p.L(), kHbKeySyms)));
}

// expected hits per position of pattern `p`; `rides` whether it costs less in a pass over `positions` than alone
static double dna_lev_hits(const fzb_haystack *h, const Plan &p, double positions, bool *rides) {
    const uint32_t L = p.L(), n = p.m / L;
    const double c = h->coll_prob;
    const double post = n * std::pow(std::max(c, 0.25), (double)std::min<uint32_t>(L, kHbKeySyms));
    const double hits = n * std::pow(c, (double)L);
    const double pass_ns = positions * (kDnaLevPostNs * post + kDnaLevHitNs * hits);
    const double alone_ns = kDnaLevAloneMs * 1e6 + positions * (kDnaLevAloneReadNs + kDnaLevAloneHitNs * hits);
    *rides = pass_ns < alone_ns;
    return hits;
}

// One 2-bit n-gram pass (k_filter_mdense2 / k_verify_mhits) for the Levenshtein patterns ids[]; same return convention
// as batch_pass.  The own range is scanned and verified in chunks whose expected hits (hits_per_pos per position)
// fill at most half the hit list; an overflowing chunk sends the pass's patterns one by one.  tiny
// (FZB_F_TINY_LIST): kTinyBatchCap hits and chunks of kTinyLpChunk positions.
static int batch_pass_dna(BatchCall &c, const std::vector<uint32_t> &ids, double hits_per_pos) {
    fzb_haystack *h = c.h;
    const uint32_t cnt = (uint32_t)ids.size();
    std::vector<BatchPat> pats(cnt);
    std::vector<uint32_t> pinfo(cnt);
    Mdense2Params p{};
    two_bit_code(c.patterns, c.offsets, ids, p.code);
    std::unordered_map<uint32_t, std::vector<uint32_t>> keys;  // key -> postings pattern << 8 | n-gram
    keys.reserve(cnt * 64);
    for (uint32_t i = 0; i < cnt; i++) {
        const uint32_t id = ids[i], m = c.len(id), k = c.plans[id].k;
        BatchPat &bp = pats[i];
        fill_pat(bp, c, id);
        bp.L = (int)c.plans[id].L();
        bp.n_ngrams = (int)m / bp.L;
        pinfo[i] = m | (k << 8) | ((uint32_t)bp.L << 16);
        for (int j = 0; j < bp.n_ngrams; j++) two_bit_key(keys, p.code, bp.P + j * bp.L, bp.L, (i << 8) | (uint32_t)j);
    }
    std::vector<uint32_t> bits(kHbKeyWords, 0);
    int rc = upload_pass_tables(h, keys, bits, pinfo, pats, [&](uint32_t w) { bits[w >> 5] |= 1u << (w & 31u); });
    if (rc) return rc;
    TRY(ensure_mhits(h));
    const uint32_t hits_cap = c.tiny ? std::min<uint32_t>(h->d_mhits.size(), kTinyBatchCap) : (uint32_t)h->d_mhits.size();
    p.dp = MdenseParams{pass_params(h), h->batch->d_bpats.get(), h->d_mhits.get(), hits_cap};
    const uint64_t tile = (uint64_t)kMultiTileVecs * 16;
    const uint64_t chunk = c.tiny ? kTinyLpChunk
                                  : std::max(tile, (uint64_t)(hits_cap / 2 / std::max(hits_per_pos, 1e-9)) / tile * tile);
    const int64_t nvec = (int64_t)(round_up(h->buf_len, 16) / 16);
    std::vector<RawRec> raw;
    uint32_t cnts[CNT_COUNT];
    fzb_stats pass{};
    const RecSet rs = rec_set(h);  // (verify kernel only)
    ChunkSums cs;
    rc = run_batch_pass(c, [&]() -> int {
        // CNT_OVERFLOW: the chunk's hits did not fit the list
        return run_chunks(h, chunk, CNT_MHITS, CNT_OVERFLOW, cnts, cs, [&](uint64_t lo, uint64_t hi) {
            p.scan_lo = (int64_t)lo;
            p.scan_hi = (int64_t)hi;
            const int64_t v0 = (p.scan_lo - (int64_t)h->buf_lo) / 16;
            const int64_t v1 = (p.scan_hi - (int64_t)h->buf_lo + 15) / 16;
            const int64_t ntiles = (v1 - v0 + kMultiTileVecs - 1) / kMultiTileVecs;
            p.dp.mp.counters = h->d_counters.get();
            k_filter_mdense2<<<(int)std::min<int64_t>(ntiles, h->sm_count), kMultiThreads, kMdense2Smem, h->stream>>>(
                p, nvec, v0, ntiles);
        }, [&]() -> int {
            with_recs(h, [&](auto rec) {
                constexpr bool R = decltype(rec)::value;
                k_verify_mhits<R><<<h->sm_count * 8, kMhThreads, 0, h->stream>>>(p.dp, h->d_out.get(), h->d_out.size(),
                                                                                    h->d_counters.get(), rs);
            });
            return FZB_OK;
        });
    }, raw, cnts, pass);
    if (rc) return rc;
    pass.route = 2;
    pass.filter_ms = cs.scan_ms;
    pass.n_candidates = cs.listed;
    pass.n_launches = 2 * cs.chunks;
    return c.finish_pass(raw, cnts[CNT_OUT], ids, pass, 0, false);
}

// The q-sample passes over the patterns `admit(i)` takes, in order, each as many as a pass's pattern slots and gram
// table hold.  A pass of one pattern is not worth it.
template <class F>
static int qsample_passes(BatchCall &c, F admit) {
    std::vector<uint32_t> shared;
    for (uint32_t i = 0; i < c.count; i++)
        if (admit(i)) shared.push_back(i);
    size_t done = 0;
    while (done < shared.size()) {
        std::vector<uint32_t> ids;
        uint64_t ngr = 0;
        while (done < shared.size() && ids.size() < kMaxBatchPats) {
            const uint32_t m = c.len(shared[done]);
            if (ngr + (m - 3) > kMaxBatchGrams) break;
            ngr += m - 3;
            ids.push_back(shared[done++]);
        }
        if (ids.size() < 2) break;
        TRY(c.settle(batch_pass(c, ids, false), ids));
    }
    return FZB_OK;
}

// The n-gram-prefix pass over the unsettled n-gram-route patterns `admit(i)` takes (the class's window-slot rule
// among its conditions), in order, while the expected prefix hits per haystack position stay within 0.02 and the
// prefix table has room.
template <class F>
static int dense_pass(BatchCall &c, F admit) {
    std::vector<uint32_t> ids;
    if (c.share && sample_collision_prob(c.h) == FZB_OK) {
        double expect = 0.0;
        uint32_t grams = 0;
        const double c3 = c.h->coll_prob * c.h->coll_prob * c.h->coll_prob;
        for (uint32_t i = 0; i < c.count && ids.size() < kMaxBatchPats; i++) {
            if (c.settled(i) || !admit(i)) continue;
            const uint32_t n = c.len(i) / c.plans[i].L();  // n-grams
            if (expect + n * c3 > 0.02) continue;  // (low-entropy text: prefixes hit everywhere -> one by one)
            if (grams + n > kMaxBatchGrams) continue;  // prefix table capacity
            expect += n * c3;
            grams += n;
            ids.push_back(i);
        }
    }
    return ids.size() >= 2 ? c.settle(batch_pass(c, ids, true), ids) : FZB_OK;
}

// A candidate of a pass bounded by an expected cost and by postings (greedy_passes).
struct PassItem {
    uint32_t i;
    double cost;
    uint32_t postings;
};

// The items in order, each joining the open pass unless that would cross kMaxBatchPats patterns, `max_cost` or
// kMaxBatchGrams postings (so at most that many distinct keys), which first closes the pass: `run(ids, cost)` runs a
// closed pass of at least two patterns (a pass of one is not worth it).
template <class F>
static int greedy_passes(const std::vector<PassItem> &items, double max_cost, F run) {
    std::vector<uint32_t> ids;
    double cost = 0.0;
    uint64_t npost = 0;
    auto close = [&]() -> int {
        const int rc = ids.size() >= 2 ? run(ids, cost) : FZB_OK;
        ids.clear();
        cost = 0.0;
        npost = 0;
        return rc;
    };
    for (const PassItem &it : items) {
        if (ids.size() == kMaxBatchPats || cost + it.cost > max_cost || npost + it.postings > kMaxBatchGrams)
            TRY(close());
        ids.push_back(it.i);
        cost += it.cost;
        npost += it.postings;
    }
    return close();
}

static int levenshtein_batch(BatchCall &c, fzb_stats *total) {
    fzb_haystack *h = c.h;
    // n-gram-route patterns with k > 0 (the k = 0 route is the exact search's) short enough for the passes' pattern
    // slots; among them those whose single search takes the sampled filter, and those whose hit windows fit a slot of
    // k_verify_mhits (the dense and the 2-bit passes)
    auto ngrams = [&](const Plan &p) { return p.route == Route::LevNgrams && p.k > 0 && p.m <= (uint32_t)kBatchMaxM; };
    auto mhits = [&](const Plan &p) {
        return ngrams(p) && p.m - p.L() <= 32 && p.m + 2 * p.k + 12 <= (uint32_t)kMhSlotBytes;
    };
    // the patterns the shared scan can take: the q-sample lemma holds and their 4-grams are selective on this haystack
    TRY(qsample_passes(c, [&](uint32_t i) { return c.share && ngrams(c.plans[i]) && sampled_filter(h, c.plans[i], 0); }));
    // the n-gram-route patterns the lemma does not cover share a scan of their own (n-gram prefixes at every position)
    TRY(dense_pass(c, [&](uint32_t i) { return mhits(c.plans[i]); }));
    // LP-route patterns share scans of 64 patterns each (bit-sliced window counters)
    std::vector<uint32_t> lp_ids;
    for (uint32_t i = 0; c.share && i < c.count; i++) {
        const Plan &p = c.plans[i];
        if (c.settled(i) || p.route != Route::LevLp || p.k >= p.m) continue;
        if (p.m > 31 || p.k > 8 || p.m + p.k > 31) continue;  // automaton masks / 6-bit window counters
        lp_ids.push_back(i);
    }
    for (size_t first = 0; first + 2 <= lp_ids.size(); first += 64) {
        std::vector<uint32_t> ids(lp_ids.begin() + first, lp_ids.begin() + std::min(lp_ids.size(), first + 64));
        if (ids.size() < 2) break;
        TRY(c.settle(batch_pass_lp(c, ids), ids));
    }
    // on low-entropy haystacks (at the 0.15 boundary of k_filter_dense2) the n-gram-route patterns left over that cost
    // less in a pass than alone share 2-bit n-gram scans (k_filter_mdense2), in passes bounded by hits and capacity
    if (c.share && h->coll_prob >= 0.15) {
        const double positions = (double)(h->own_hi - h->own_lo);
        std::vector<PassItem> items;
        for (uint32_t i = 0; i < c.count; i++) {
            const Plan &p = c.plans[i];
            if (c.settled(i) || !mhits(p) || p.L() < kDnaLevMinL) continue;
            if (sampled_filter(h, p, 0)) continue;  // (a q-sample pass that overflowed)
            bool rides = false;
            const double phits = dna_lev_hits(h, p, positions, &rides);
            if (!rides || phits > kDnaLevPassHits) continue;
            items.push_back({i, phits, dna_lev_postings(p)});
        }
        TRY(greedy_passes(items, kDnaLevPassHits, [&](const std::vector<uint32_t> &ids, double hits) {
            return c.settle(batch_pass_dna(c, ids, hits), ids);
        }));
    }
    return c.finish(total);
}

extern "C" int fzb_search_levenshtein_batch(fzb_haystack *h, const uint8_t *patterns, const uint32_t *offsets,
                                            const uint32_t *max_l_dist, uint32_t count, uint32_t flags,
                                            fzb_result **out, fzb_stats *total) {
    HandleLock handle_lock(h);
    if (!h || !out || (count && (!patterns || !offsets || !max_l_dist))) return fail(FZB_E_INVALID, "NULL argument");
    BatchCall c(h, patterns, offsets, count, flags, out, nullptr);
    TRY(c.begin([&](uint32_t i, const uint8_t *p, uint32_t m, Plan &pl) {
        return plan_levenshtein(h, p, m, max_l_dist[i], flags, pl);
    }));
    return levenshtein_batch(c, total);
}

extern "C" int fzb_search_exact(fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t flags,
                                fzb_result **out) {
    return run_search(h, pattern, flags, out, [&](Plan &pl) { return plan_exact(h, pattern, m, flags, pl); });
}

// Points a handle at a view of its buffer for its own lifetime; keeps the handle's geometry and restores all of it
// (global_len and coll_prob included) on every exit.
struct BufferView {
    fzb_haystack *const h;
    uint8_t *const d;
    const uint64_t buf_len, buf_lo, own_lo, own_hi, padded_len, global_len;
    const double coll_prob;
    explicit BufferView(fzb_haystack *hs)
        : h(hs), d(hs->d), buf_len(hs->buf_len), buf_lo(hs->buf_lo), own_lo(hs->own_lo), own_hi(hs->own_hi),
          padded_len(hs->padded_len), global_len(hs->global_len), coll_prob(hs->coll_prob) {}
    ~BufferView() {
        h->d = d;
        h->buf_len = buf_len;
        h->buf_lo = buf_lo;
        h->own_lo = own_lo;
        h->own_hi = own_hi;
        h->padded_len = padded_len;
        h->global_len = global_len;
        h->coll_prob = coll_prob;
    }
    BufferView(const BufferView &) = delete;
    BufferView &operator=(const BufferView &) = delete;
    // the bytes [vlo, vhi) of the sequence (vlo 128-byte aligned relative to the buffer start), owning [lo, hi)
    void set(uint64_t vlo, uint64_t vhi, uint64_t lo, uint64_t hi) {
        h->d = d + (vlo - buf_lo);
        h->buf_lo = vlo;
        h->buf_len = vhi - vlo;
        h->padded_len = round_up(h->buf_len, 128) + 128;
        h->own_lo = lo;
        h->own_hi = hi;
    }
};

// search_exact(subsequence, sequence, start_index, end_index) (search_exact.py:22-56): the occurrences lying wholly
// inside [start, end).  The window is a VIEW of the resident buffer treated like a shard of a sequence that ends
// at `end` (anchors owned from `start`, occurrences clipped at the view's global end), so the bytes outside the
// window are not scanned.
extern "C" int fzb_search_exact_window(fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint64_t start,
                                       uint64_t end, uint32_t flags, fzb_result **out) {
    HandleLock handle_lock(h);
    if (!h || !out) return fail(FZB_E_INVALID, "NULL argument");
    *out = nullptr;
    TRY(refuse_records(h, "the windowed exact search"));
    if (flags & FZB_F_GLOBAL) return fail(FZB_E_INVALID, "windowed exact search is per handle");
    if (!is_whole_sequence(h)) return fail(FZB_E_INVALID, "windowed exact search needs a whole (unsharded) sequence");
    // clamp (search_exact.py:29-30): start into [0, n], end into [start, n]
    start = std::min<uint64_t>(start, h->global_len);
    end = std::max<uint64_t>(start, std::min<uint64_t>(end, h->global_len));
    if (end - start < m) {  // no room for an occurrence (also: the empty window): nothing to launch
        Plan pl;
        int rc0 = plan_exact(h, pattern, m, flags, pl);
        if (rc0) return rc0;
        fzb_result *res;
        rc0 = make_result(out, &res);
        if (rc0) return rc0;
        res->unconsolidated = true;
        res->have_fin = true;
        *out = res;
        return FZB_OK;
    }
    // the view starts a halo before the window (the shard geometry check of the search wants one on both sides;
    // the right one ends at the view's global end), on a 128-byte boundary of the buffer
    const uint64_t halo = round_up((uint64_t)m, 128) + 128;
    BufferView view(h);
    view.set((start > halo ? start - halo : 0) / 128 * 128, end, start, end);
    h->global_len = end;
    h->coll_prob = -1.0;  // (the byte statistics of the window)
    const int rc = fzb_search_exact(h, pattern, m, flags, out);
    if (rc == FZB_OK && *out) (*out)->fetch_raw();  // the records leave the view's buffers before the geometry changes back
    return rc;
}

// TMA descriptors of the buffer viewed as rows of 128 bytes (k_hamming_count): box 256 rows / 8 rows,
// SWIZZLE_128B, out-of-bounds rows (the halo before row 0, the tail) read as zeros.
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int make_row_maps(fzb_haystack *h, CUtensorMap *map256, CUtensorMap *map8) {
    // resolved once per process; a function-local static's initialisation is thread-safe (handles of different
    // threads get here concurrently)
    static const EncodeTiledFn encode = []() -> EncodeTiledFn {
        void *fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess) return nullptr;
        return (fn && q == cudaDriverEntryPointSuccess) ? (EncodeTiledFn)fn : nullptr;
    }();
    if (!encode) {
        cudaGetLastError();
        return fail(FZB_E_CUDA, "cuTensorMapEncodeTiled not available");
    }
    const cuuint64_t rows = h->padded_len / kHcRowBytes;  // whole rows inside the allocation
    const cuuint64_t dims[2] = {(cuuint64_t)kHcRowBytes, rows};
    const cuuint64_t strides[1] = {(cuuint64_t)kHcRowBytes};
    const cuuint32_t estr[2] = {1, 1};
    for (int which = 0; which < 2; which++) {
        const cuuint32_t box[2] = {(cuuint32_t)kHcRowBytes, which == 0 ? 256u : (cuuint32_t)kHcHaloRows};
        CUresult r = encode(which == 0 ? map256 : map8, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, h->d, dims, strides, box,
                            estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                            CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) return fail(FZB_E_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    }
    return FZB_OK;
}

static int search_hamming(fzb_haystack *h, const uint8_t *pattern, const Plan &pl, uint32_t flags, fzb_result *res) {
    const uint32_t m = pl.m;
    int rc;
    ScanParams p;
    fill_params(h, pattern, m, p);
    p.k = (int)pl.k;
    if (flags & FZB_F_TINY_LIST) p.glist_cap = std::min(h->glist_cap, 8u);  // (testing) reach the bitmap-mode retry
    const RecSet rs = rec_set(h);
    CK(cudaSetDevice(h->device));
    res->stats.route = 4;
    res->stats.bytes_scanned = h->buf_len;
    // counting q-sample filter needs W = floor((m-3)/4) >= k+1 aligned words and 4-bit fields (k <= 7)
    const bool counting = !(flags & FZB_F_FORCE_DENSE) && (int)m >= 4 * p.k + 7 && p.k <= 7 && h->buf_len > 0;
    HamCountParams hp{};
    CUtensorMap map256, map8;
    int slices = 0;  // of the counters (ham_recur.h)
    if (counting) {
        hp.Wc = std::min<int>((int)(m - 3) / 4, 8);
        // fewer instructions per word: two slices (counting to 4) where the threshold allows, else three
        slices = hp.Wc - p.k <= 4 ? 2 : 3;
        hp.bias = (1 << slices) - (hp.Wc - p.k);
        hp.nrows = (int64_t)(round_up(h->buf_len, kHcRowBytes) / kHcRowBytes);
        rc = make_row_maps(h, &map256, &map8);
        if (rc) return rc;
        CK(cudaFuncSetAttribute(k_hamming_count<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHcSmem));
        CK(cudaFuncSetAttribute(k_hamming_count<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHcSmem));
    }
    bool bitmap_mode = false;
    PostPlan plan{2, (flags & FZB_F_GLOBAL) != 0};  // FINAL == RAW in (start, end, dist) order, ordered by k_post
    auto enqueue = [&]() -> int {
        if (counting) {
            const int64_t ntiles = (hp.nrows + kHcThreads - 1) / kHcThreads;
            const int grid = (int)std::min<int64_t>(ntiles, (int64_t)h->sm_count * 2);
            if (slices == 2)
                k_hamming_count<2><<<grid, kHcThreads, kHcSmem, h->stream>>>(p, hp, map256, map8);
            else
                k_hamming_count<3><<<grid, kHcThreads, kHcSmem, h->stream>>>(p, hp, map256, map8);
            CK(cudaEventRecord(h->ev[1], h->stream));
            h->ev1_recorded = true;
            // one verify launch: the granule work list -- or, after it overflowed, the whole bitmap
            with_recs(h, [&](auto rec) {
                constexpr bool R = decltype(rec)::value;
                k_verify_ham<R><<<h->sm_count * 4, kVerifyThreads, 0, h->stream>>>(
                    p, h->d_bitmap.size(), h->d_glist.get(), p.glist_cap, bitmap_mode ? 1 : 0, h->d_out.get(),
                    h->d_out.size(), h->d_counters.get(), rs);
            });
            res->stats.n_launches += 1;
        } else {
            with_recs(h, [&](auto rec) {
                constexpr bool R = decltype(rec)::value;
                k_hamming_scan<R><<<h->sm_count * 8, kHamThreads, 0, h->stream>>>(p, h->d_out.get(), h->d_out.size(),
                                                                                  h->d_counters.get(), rs);
            });
        }
        res->stats.n_launches++;
        return FZB_OK;
    };
    for (;;) {
        rc = run_emitting(h, res, enqueue, plan);
        if (rc) return rc;
        if (!counting || bitmap_mode || h->h_counters[CNT_GRAN] <= p.glist_cap) break;
        // the work list overflowed (see search_lev_ngrams)
        bitmap_mode = true;
        plan.global = false;
        p.glist_cap = 0;
        res->discard_attempt();
    }
    res->raw_order = 1;
    return FZB_OK;
}

extern "C" int fzb_search_hamming(fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t k,
                                  uint32_t flags, fzb_result **out) {
    return run_search(h, pattern, flags, out, [&](Plan &pl) { return plan_hamming(h, pattern, m, k, flags, pl); });
}

// ------------------------------------------------------------------------------------------------
// Substitutions-only batches: one scan for many patterns (ham_batch_kernels.cuh)
// ------------------------------------------------------------------------------------------------
// Bounds on the postings walked per haystack position (expected piece hits, from the sampled byte statistics).
// Measured on an H100 80GB HBM3 (400 W power limit), 4 GiB of DNA, 1 024 patterns (tools/probe_ham_batch.py): three
// passes walked 2.21e9 postings in 85 ms of scan, 0.039 ns per posting, against 1.6 ms for one scan of the haystack.
// A pattern whose postings cost more than one scan (0.01 per position on 4 GiB) is searched on its own; a pass is
// closed at 0.25 per position (at most 0.25 x 4.29e9 x 0.039 ns = 42 ms of verification behind one 1.6 ms read of
// 4 GiB; the three measured passes averaged 28 ms).
constexpr double kHamBatchPatExpect = 0.01;
constexpr double kHamBatchExpect = 0.25;

// Key width of pattern `p` in a pass, in symbols: 2-bit keys are always 8 symbols wide (a piece of 5..7 symbols
// is entered under every completion); text keys are the first min(L, 4) bytes of a piece, one width per pass.  0 when
// no pass can take the pattern: too long for the pass's pattern slots, every start matches, or a piece too short for
// a selective key.
static uint32_t ham_batch_key(const Plan &p, bool two_bit) {
    if (p.m > (uint32_t)kBatchMaxM || p.k >= p.m) return 0;
    const uint32_t L = p.L();
    if (two_bit) return L >= 5 ? (uint32_t)kHbKeySyms : 0;
    return L >= 3 ? std::min<uint32_t>(L, 4) : 0;
}

// Postings of pattern `p` in a pass: one per piece, or per completion of a 2-bit key shorter than 8 symbols.
static uint32_t ham_batch_postings(const Plan &p, bool two_bit) {
    const uint32_t L = p.L();
    return (p.k + 1) * (two_bit && L < (uint32_t)kHbKeySyms ? 1u << (2 * (kHbKeySyms - L)) : 1u);
}

// Expected postings per haystack position of pattern `p` in a pass with keys of `key` symbols.
static double ham_batch_cost(const fzb_haystack *h, const Plan &p, uint32_t key, bool two_bit) {
    const uint32_t L = p.L();
    const double c = two_bit ? std::max(h->coll_prob, 0.25) : h->coll_prob;  // (2-bit keys see at most 4 codes)
    return (p.k + 1) * std::pow(c, (double)std::min(L, key));
}

// One k_ham_batch_scan pass for the patterns ids[]; same return convention as batch_pass.  two_bit: the 2-bit keys of
// low-entropy haystacks, else text keys of key_bytes (4 or 3) bytes.
static int batch_pass_ham(BatchCall &c, const std::vector<uint32_t> &ids, bool two_bit, uint32_t key_bytes) {
    fzb_haystack *h = c.h;
    const uint32_t cnt = (uint32_t)ids.size();
    std::vector<BatchPat> pats(cnt);
    std::vector<uint32_t> pinfo(cnt);
    HamBatchParams hp{};
    hp.key_mask = key_bytes == 4 ? 0xFFFFFFFFu : 0x00FFFFFFu;
    if (two_bit) two_bit_code(c.patterns, c.offsets, ids, hp.code);
    std::unordered_map<uint32_t, std::vector<uint32_t>> keys;  // key -> postings pattern << 8 | piece
    keys.reserve(cnt * 8);
    for (uint32_t i = 0; i < cnt; i++) {
        const uint32_t id = ids[i], m = c.len(id), k = c.plans[id].k, L = c.plans[id].L();
        BatchPat &bp = pats[i];
        fill_pat(bp, c, id);
        bp.L = (int)L;
        bp.n_ngrams = (int)k + 1;
        pinfo[i] = m | (k << 8) | (L << 16);
        for (uint32_t j = 0; j <= k; j++) {
            const uint8_t *s = bp.P + j * L;
            if (two_bit) {
                two_bit_key(keys, hp.code, s, L, (i << 8) | j);
            } else {
                uint32_t w;
                memcpy(&w, s, 4);  // (P is zero-padded to kBatchMaxM bytes)
                keys[w & hp.key_mask].push_back((i << 8) | j);
            }
        }
    }
    std::vector<uint32_t> bits(two_bit ? kHbKeyWords : kMultiTblWords + kMulti2Words, 0);
    int rc = upload_pass_tables(h, keys, bits, pinfo, pats, [&](uint32_t w) {
        const uint32_t b = two_bit ? w : (w * kHashMul) >> (32 - kMultiTblBits);
        bits[b >> 5] |= 1u << (b & 31u);
        if (!two_bit) {
            const uint32_t h2 = multi_hash2(w);
            bits[kMultiTblWords + (h2 >> 5)] |= 1u << (h2 & 31u);
        }
    });
    if (rc) return rc;
    hp.mp = pass_params(h);
    hp.mp.bits2 = two_bit ? nullptr : h->batch->d_mbits.get() + kMultiTblWords;
    hp.pats = h->batch->d_bpats.get();
    const size_t smem = two_bit ? kHbSmem2 : kMultiSmem;
    const RecSet rs = rec_set(h);  // (the key and table tests only look at content: only the verification takes it)
    const void *fn = nullptr;
    with_recs(h, [&](auto rec) {
        constexpr bool R = decltype(rec)::value;
        fn = two_bit ? (const void *)k_ham_batch_scan<true, R> : (const void *)k_ham_batch_scan<false, R>;
    });
    CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 1;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kMultiThreads, smem));
    per_sm = std::max(per_sm, 1);
    const int64_t nvec = (int64_t)(round_up(h->buf_len, 16) / 16);
    const int64_t ntiles = (nvec + kMultiTileVecs - 1) / kMultiTileVecs;
    std::vector<RawRec> raw;
    uint32_t cnts[CNT_COUNT];
    fzb_stats pass{};
    rc = run_batch_pass(c, [&]() -> int {
        hp.out = h->d_out.get();  // (the output buffer may have grown since the last attempt)
        hp.cap = h->d_out.size();
        if (ntiles > 0) {
            const int grid = (int)std::min<int64_t>(ntiles, (int64_t)h->sm_count * per_sm);
            with_recs(h, [&](auto rec) {
                constexpr bool R = decltype(rec)::value;
                if (two_bit)
                    k_ham_batch_scan<true, R><<<grid, kMultiThreads, smem, h->stream>>>(hp, nvec, ntiles, rs);
                else
                    k_ham_batch_scan<false, R><<<grid, kMultiThreads, smem, h->stream>>>(hp, nvec, ntiles, rs);
            });
        }
        CK(cudaGetLastError());
        return FZB_OK;
    }, raw, cnts, pass);
    if (rc) return rc;
    if (c.tiny && cnts[CNT_OUT] > kTinyBatchCap) return 1;  // FZB_F_TINY_LIST: the pass's record list holds kTinyBatchCap
    pass.route = 8;
    pass.filter_ms = pass.gpu_ms;
    pass.n_candidates = cnts[CNT_CAND];
    pass.n_launches = 1;
    return c.finish_pass(raw, cnts[CNT_OUT], ids, pass, 1, true);
}

static int hamming_batch(BatchCall &c, fzb_stats *total) {
    fzb_haystack *h = c.h;
    if (c.share && c.count >= 2 && sample_collision_prob(h) == FZB_OK) {
        const bool two_bit = h->coll_prob >= 0.15;  // the boundary of k_filter_dense2
        // one group of passes per key width: 8 symbols (2-bit); 4 bytes, then 3 bytes (text)
        for (uint32_t key = two_bit ? (uint32_t)kHbKeySyms : 4u; key >= (two_bit ? (uint32_t)kHbKeySyms : 3u); key--) {
            std::vector<PassItem> items;
            for (uint32_t i = 0; i < c.count; i++) {
                const Plan &p = c.plans[i];
                if (ham_batch_key(p, two_bit) != key) continue;
                const double cost = ham_batch_cost(h, p, key, two_bit);
                if (cost > kHamBatchPatExpect) continue;
                items.push_back({i, cost, ham_batch_postings(p, two_bit)});
            }
            TRY(greedy_passes(items, kHamBatchExpect, [&](const std::vector<uint32_t> &ids, double) {
                return c.settle(batch_pass_ham(c, ids, two_bit, key), ids);
            }));
        }
    }
    return c.finish(total);
}

extern "C" int fzb_search_hamming_batch(fzb_haystack *h, const uint8_t *patterns, const uint32_t *offsets,
                                        const uint32_t *max_subs, uint32_t count, uint32_t flags, fzb_result **out,
                                        fzb_stats *total) {
    HandleLock handle_lock(h);
    if (!h || !out || (count && (!patterns || !offsets || !max_subs))) return fail(FZB_E_INVALID, "NULL argument");
    BatchCall c(h, patterns, offsets, count, flags, out, nullptr);
    TRY(c.begin([&](uint32_t i, const uint8_t *p, uint32_t m, Plan &pl) {
        return plan_hamming(h, p, m, max_subs[i], flags, pl);
    }));
    return hamming_batch(c, total);
}

extern "C" int fzb_search_generic(fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t max_subs,
                                  uint32_t max_ins, uint32_t max_dels, uint32_t max_l, uint32_t flags,
                                  fzb_result **out) {
    return run_search(h, pattern, flags, out, [&](Plan &pl) {
        return plan_generic(h, pattern, m, max_subs, max_ins, max_dels, max_l, flags, pl);
    });
}

static int generic_batch(BatchCall &c, fzb_stats *total) {
    fzb_haystack *h = c.h;
    // the shared scans take patterns of the two generic routes (not the k = 0 route) no longer than a BatchPat holds
    auto shareable = [&](uint32_t i, Route r) {
        return c.share && !c.settled(i) && c.plans[i].route == r && c.len(i) <= (uint32_t)kBatchMaxM;
    };
    // n-gram route, q-sample lemma holds and its 4-grams are selective on this haystack: q-sample passes, bounded as
    // in the Levenshtein batch
    TRY(qsample_passes(c, [&](uint32_t i) { return shareable(i, Route::GenericNgrams) && sampled_filter(h, c.plans[i], 0); }));
    // the other n-gram-route patterns: one n-gram-prefix pass, under the Levenshtein batch's bounds; a hit's window
    // must fit a warp's slot in k_verify_mhits_generic
    TRY(dense_pass(c, [&](uint32_t i) {
        return shareable(i, Route::GenericNgrams) && c.len(i) + 2 * c.plans[i].k + 8 <= (uint32_t)kMhgSlotBytes;
    }));
    // LP route (with the lowered limit): passes of at most 64 patterns (6-bit window counters, 32-bit masks)
    std::vector<uint32_t> lp_ids;
    for (uint32_t i = 0; i < c.count; i++) {
        if (!shareable(i, Route::GenericLp)) continue;
        const uint32_t m = c.len(i), k = c.plans[i].k;
        if (m > 31 || m + k > 31 || k >= m) continue;
        lp_ids.push_back(i);
    }
    // (the passes are balanced, so that none is left with a single pattern: 65 patterns make passes of 33 and 32)
    const size_t nlp = (lp_ids.size() + 63) / 64;
    for (size_t q = 0; q < nlp && lp_ids.size() >= 2; q++) {
        std::vector<uint32_t> ids(lp_ids.begin() + lp_ids.size() * q / nlp, lp_ids.begin() + lp_ids.size() * (q + 1) / nlp);
        TRY(c.settle(batch_pass_lp(c, ids), ids));
    }
    return c.finish(total);
}

extern "C" int fzb_search_generic_batch(fzb_haystack *h, const uint8_t *patterns, const uint32_t *offsets,
                                        const uint32_t *max_subs, const uint32_t *max_ins, const uint32_t *max_dels,
                                        const uint32_t *max_l_dist, uint32_t count, uint32_t flags, fzb_result **out,
                                        fzb_stats *total) {
    HandleLock handle_lock(h);
    if (!h || !out || (count && (!patterns || !offsets || !max_subs || !max_ins || !max_dels || !max_l_dist)))
        return fail(FZB_E_INVALID, "NULL argument");
    BatchCall c(h, patterns, offsets, count, flags, out, nullptr);
    TRY(c.begin([&](uint32_t i, const uint8_t *p, uint32_t m, Plan &pl) {
        return plan_generic(h, p, m, max_subs[i], max_ins[i], max_dels[i], max_l_dist[i], flags, pl);
    }));
    return generic_batch(c, total);
}

static int search_by_class(fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t max_subs, uint32_t max_ins,
                           uint32_t max_dels, uint32_t max_l, uint32_t flags, fzb_result **out) {
    return run_search(h, pattern, flags, out, [&](Plan &pl) {
        return plan_by_class(h, pattern, m, max_subs, max_ins, max_dels, max_l, flags, pl);
    });
}

// ------------------------------------------------------------------------------------------------
// fzb_best_per_record (DESIGN.md section 5.13): every record of a set assigned its best-matching pattern
// ------------------------------------------------------------------------------------------------
extern "C" int fzb_best_per_record(fzb_haystack *h, const uint8_t *patterns, const uint32_t *offsets,
                                   const uint32_t *max_subs, const uint32_t *max_ins, const uint32_t *max_dels,
                                   const uint32_t *max_l_dist, uint32_t count, uint32_t flags, int32_t *pattern,
                                   int64_t *start, int64_t *end, int32_t *dist, int32_t *second_pattern,
                                   int32_t *second_dist, fzb_stats *total) {
    HandleLock handle_lock(h);
    if (!h || !pattern || !start || !end || !dist || !second_pattern || !second_dist ||
        (count && (!patterns || !offsets || !max_subs || !max_ins || !max_dels || !max_l_dist)))
        return fail(FZB_E_INVALID, "NULL argument");
    if (!h->recs) return fail(FZB_E_INVALID, "fzb_best_per_record needs a handle with a record set");
    if (flags & ~FZB_F_TINY_LIST) return fail(FZB_E_UNSUPPORTED, "fzb_best_per_record takes no flag other than FZB_F_TINY_LIST");
    if (count > kBestMaxPatterns)
        return fail(FZB_E_UNSUPPORTED, "more than %u patterns in one fzb_best_per_record call", kBestMaxPatterns);
    if (h->recs->longest > (1ull << 31))
        return fail(FZB_E_UNSUPPORTED, "fzb_best_per_record needs records shorter than 2^31");
    // every pattern planned as its single search would take it (plan_by_class), before any work; then by class, each
    // class a batch of its own over its subset of the patterns and their plans
    struct Subset {
        std::vector<uint8_t> blob;
        std::vector<uint32_t> offsets{0}, ordinal;
        std::vector<Plan> plans;
    } lev, ham, gen;
    for (uint32_t i = 0; i < count; i++) {
        if (offsets[i + 1] < offsets[i]) return fail(FZB_E_INVALID, "offsets must be non-decreasing");
        const uint8_t *p = patterns + offsets[i];
        const uint32_t m = offsets[i + 1] - offsets[i];
        Plan pl;
        TRY(plan_by_class(h, p, m, max_subs[i], max_ins[i], max_dels[i], max_l_dist[i], flags, pl));
        if (pl.route == Route::Exact) pl.route = Route::LevNgrams;  // (the Levenshtein batch's k == 0 route)
        Subset &sub = pl.route == Route::Hamming ? ham : pl.generic() ? gen : lev;
        sub.blob.insert(sub.blob.end(), p, p + m);
        sub.offsets.push_back((uint32_t)sub.blob.size());
        sub.ordinal.push_back(i);
        sub.plans.push_back(pl);
    }
    CK(cudaSetDevice(h->device));
    const uint64_t nrec = h->recs->d_off.size() - 1;
    if (!h->bestb || h->bestb->d_words.size() < 2 * nrec) {  // built whole, beside the one it replaces
        std::unique_ptr<BestBufs> grown;
        TRY(ensure_group(grown, [&](BestBufs &b) -> int {
            TRY(b.d_words.alloc(2 * nrec));
            return b.d_ids.alloc(kMaxBatchPats);
        }));
        h->bestb = std::move(grown);
    }
    BestState state{h->bestb->d_words.get(), h->bestb->d_words.get() + nrec, nullptr};
    fzb_stats sum{};
    k_best_fill<<<(int)std::min<uint64_t>((2 * nrec + kBestThreads - 1) / kBestThreads, (uint64_t)h->sm_count * 8),
                  kBestThreads, 0, h->stream>>>(state.best, 2 * nrec);
    CK(cudaGetLastError());
    sum.n_launches = 1;
    for (Subset *sub : {&lev, &ham, &gen}) {
        const uint32_t n = (uint32_t)sub->ordinal.size();
        if (n == 0) continue;
        state.ordinal = sub->ordinal.data();
        BatchCall c(h, sub->blob.data(), sub->offsets.data(), n, flags, nullptr, &state);
        c.plans = std::move(sub->plans);
        TRY(sub == &lev ? levenshtein_batch(c, nullptr) : sub == &ham ? hamming_batch(c, nullptr) : generic_batch(c, nullptr));
        add_stats(&sum, c.sum);
    }
    // one read-back of 16 bytes per record, whatever the number of matches
    std::vector<uint64_t> words(2 * nrec);
    CK(cudaMemcpyAsync(words.data(), state.best, 2 * nrec * sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    for (uint64_t r = 0; r < nrec; r++) {
        const uint64_t b = words[r];
        const uint32_t second = (uint32_t)words[nrec + r] & kBestPairNone;
        const bool none = b == kBestEmpty;
        const int64_t len = kBestMaxLen - (int64_t)((b >> 31) & 0x1FFu);
        dist[r] = none ? -1 : (int32_t)(b >> 56);
        pattern[r] = none ? -1 : (int32_t)((b >> 40) & 0xFFFFu);
        start[r] = none ? -1 : (int64_t)(b & 0x7FFFFFFFu);
        end[r] = none ? -1 : start[r] + len;
        second_dist[r] = second == kBestPairNone ? -1 : (int32_t)(second >> 16);
        second_pattern[r] = second == kBestPairNone ? -1 : (int32_t)(second & 0xFFFFu);
    }
    sum.route = 7;  // batch
    if (total) *total = sum;
    return FZB_OK;
}

// ------------------------------------------------------------------------------------------------
// The nearest match without a distance limit (nearest_kernels.cuh): fzb_nearest_distance / fzb_nearest_per_record
// (DESIGN.md sections 5.14, 5.16, 5.18) and their batches fzb_nearest_distance_batch / fzb_nearest_best_per_record
// (sections 5.15, 5.16, 5.18)
// ------------------------------------------------------------------------------------------------
constexpr int64_t kNearBatchMinSeg = 1024;  // bytes per warp: the warm-up (at most 128 bytes) stays <= 1/8 of it

// Gives the handle a nearest group of at least `lanes` batch lanes, `words` answer words and `rec_words` record words
// of a long pattern, built whole beside the one it replaces; a grown group keeps every size of the one before.
static int ensure_near_bufs(fzb_haystack *h, uint64_t lanes, uint64_t words, uint64_t rec_words) {
    const NearBufs *g = h->nearb.get();
    lanes = std::max<uint64_t>(lanes, 1);
    words = std::max<uint64_t>(words, 2);
    const uint64_t scan = 1 + 2 * (uint64_t)kNearMaxGrid + rec_words;
    if (g && g->d_lanes.size() >= lanes && g->d_words.size() >= words && g->d_scan.size() >= scan) return FZB_OK;
    std::unique_ptr<NearBufs> grown;
    TRY(ensure_group(grown, [&](NearBufs &b) -> int {
        const uint64_t nl = std::max<uint64_t>(lanes, g ? g->d_lanes.size() : 0);
        TRY(b.d_lanes.alloc(nl));
        TRY(b.d_pats.alloc(nl * kNearBatchMaxM));
        TRY(b.d_words.alloc(std::max<uint64_t>(words, g ? g->d_words.size() : 0)));
        return b.d_scan.alloc(std::max<uint64_t>(scan, g ? g->d_scan.size() : 0));
    }));
    h->nearb = std::move(grown);
    return FZB_OK;
}

// f(std::integral_constant<int, BITS>{}) for a pattern's word width `bits`: 32 or 64, or with WIDE 128, 192 or 256
template <bool WIDE, class F>
static int with_bits(int bits, F f) {
    if (bits == 32) return f(std::integral_constant<int, 32>{});
    if constexpr (WIDE) {
        if (bits == 128) return f(std::integral_constant<int, 128>{});
        if (bits == 192) return f(std::integral_constant<int, 192>{});
        if (bits == 256) return f(std::integral_constant<int, 256>{});
    }
    return f(std::integral_constant<int, 64>{});
}

template <class F>
static int with_bool(bool b, F f) {
    return b ? f(std::true_type{}) : f(std::false_type{});
}

// A nearest kernel of word width `bits` on the handle's stream, its table in dynamic shared memory
template <auto kernel, class P>
static int near_launch(fzb_haystack *h, dim3 grid, int bits, const P &p) {
    CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)near_smem(bits)));
    kernel<<<grid, kNearThreads, near_smem(bits), h->stream>>>(p, rec_set(h));
    CK(cudaGetLastError());
    return FZB_OK;
}

// k_nearest_scan, k_nearest_hamming_scan under substitutions only; per record on a handle with a record set
static int launch_near_scan(fzb_haystack *h, int bits, bool ham, int grid, const NearParams &p) {
    return with_bits<true>(bits, [&](auto b) {
        return with_recs(h, [&](auto r) {
            constexpr int B = decltype(b)::value;
            constexpr bool R = decltype(r)::value;
            return ham ? near_launch<k_nearest_hamming_scan<B, R>>(h, grid, B, p)
                       : near_launch<k_nearest_scan<B, R>>(h, grid, B, p);
        });
    });
}

// k_nearest_batch_scan, k_nearest_hamming_batch_scan under substitutions only; per record on a handle with a record set
static int launch_near_batch_scan(fzb_haystack *h, int bits, bool ham, dim3 grid, const NearBatchParams &p) {
    return with_bits<false>(bits, [&](auto b) {
        return with_recs(h, [&](auto r) {
            constexpr int B = decltype(b)::value;
            constexpr bool R = decltype(r)::value;
            return ham ? near_launch<k_nearest_hamming_batch_scan<B, R>>(h, grid, B, p)
                       : near_launch<k_nearest_batch_scan<B, R>>(h, grid, B, p);
        });
    });
}

// k_nearest_anchored over all records, p.g lanes per record (a batch: one CTA row per group of `rows`)
static int launch_near_anchored(fzb_haystack *h, int bits, bool ham, bool batch, uint32_t rows, const NearAnchParams &p) {
    const uint64_t per = (uint64_t)(kNearThreads / 32) * (32 / p.g);  // records per CTA and round
    const uint64_t gx = std::min<uint64_t>((p.nrec + per - 1) / per,
                                           std::max<uint64_t>(1, (uint64_t)h->sm_count * near_ctas_per_sm(bits) / rows));
    if (gx == 0) return FZB_OK;  // (no records)
    return with_bool(batch, [&](auto t) {
        constexpr bool T = decltype(t)::value;
        return with_bits<!T>(bits, [&](auto b) {
            return with_bool(ham, [&](auto x) {
                constexpr int B = decltype(b)::value;
                return near_launch<k_nearest_anchored<B, decltype(x)::value, T>>(h, dim3((unsigned)gx, rows), B, p);
            });
        });
    });
}

// The grid of the kernels with one thread per record
static int near_rec_grid(const fzb_haystack *h, uint64_t nrec) {
    return (int)std::min<uint64_t>((nrec + 255) / 256, (uint64_t)h->sm_count * 8);
}

// k_nearest_scan's segment (bytes per thread) and grid for the handle's buffer: segments long against the 2m warm-up
// on a long sequence, short enough to fill the SMs on a short one
static int near_geometry(const fzb_haystack *h, int bits, int32_t *seg) {
    *seg = (int32_t)std::min<uint64_t>(kNearMaxSeg, std::max<uint64_t>(kNearMinSeg,
                                       round_up(h->buf_len / ((uint64_t)h->sm_count * 1024) + 1, 16)));
    const uint64_t tile = (uint64_t)kNearThreads * *seg, ntiles = (h->buf_len + tile - 1) / tile;
    return (int)std::min<uint64_t>(ntiles, std::min<uint64_t>((uint64_t)h->sm_count * near_ctas_per_sm(bits), kNearMaxGrid));
}

// Enqueues one pattern's unanchored scan of the whole buffer, under substitutions only if `ham`.  On a handle with a
// record set every record's word (dist << 32 | end) lands in `words`, prefilled here; otherwise the minimum
// (dist << 48 | first_end) in result[0], prefilled by the caller, and the CTAs' (minimum, count) in `partial`, *grid
// of them.
static int near_scan_enqueue(fzb_haystack *h, const uint8_t *pattern, uint32_t m, bool ham, uint64_t *result,
                             uint64_t *partial, uint64_t *words, fzb_stats &st, int *grid) {
    NearParams p{};
    p.H = h->d;
    p.N = (int64_t)h->buf_len;
    p.m = (int)m;
    p.result = result;
    p.partial = partial;
    p.words = words;
    memcpy(p.P, pattern, m);
    const int bits = m <= 32 ? 32 : (int)round_up(m, 64);
    *grid = near_geometry(h, bits, &p.seg);
    if (h->recs) {
        const uint64_t nrec = h->recs->d_off.size() - 1;
        k_nearest_fill<<<near_rec_grid(h, nrec), 256, 0, h->stream>>>(words, nrec, ham ? kBestEmpty : (uint64_t)m << 32);
        CK(cudaGetLastError());
        st.n_launches++;
    }
    if (*grid > 0) {
        TRY(launch_near_scan(h, bits, ham, *grid, p));
        st.n_launches++;
        st.bytes_scanned += h->buf_len;
    }
    return FZB_OK;
}

// Enqueues one pattern's anchored scan of the records, one lane per record: every record's word dist << 32 | pos
// (all ones: no value) is written to `words`, the symbols read are added to the group's step slot.  'end' walks the
// records backwards with the reversed pattern, except under substitutions only, whose window is compared forwards.
static int near_anchored_enqueue(fzb_haystack *h, const uint8_t *pattern, uint32_t m, bool ham, bool end,
                                 uint64_t *words, fzb_stats &st) {
    NearAnchParams p{};
    p.H = h->d;
    p.nrec = h->recs->d_off.size() - 1;
    p.words = words;
    p.steps = h->nearb->steps();
    p.m = (int32_t)m;
    p.g = 1;
    p.end = end;
    for (uint32_t i = 0; i < m; i++) p.P[i] = pattern[end && !ham ? m - 1 - i : i];
    TRY(launch_near_anchored(h, m <= 32 ? 32 : (int)round_up(m, 64), ham, false, 1, p));
    st.n_launches++;
    return FZB_OK;
}

// 'end': the pos of every record word with a value (a record's own word or a best key) turned into the start
static int near_flip(fzb_haystack *h, uint64_t *words, fzb_stats &st) {
    const uint64_t nrec = h->recs->d_off.size() - 1;
    k_nearest_anchored_flip<<<near_rec_grid(h, nrec), 256, 0, h->stream>>>(words, nrec, rec_set(h));
    CK(cudaGetLastError());
    st.n_launches++;
    return FZB_OK;
}

// The frame of every nearest call on the handle's stream: `scan` between events 0 and 1 (filter_ms), `tail` up to
// event 2 (gpu_ms); with `steps` the symbols read, counted from zero in the group's step slot, become bytes_scanned.
// The calls keep to their own buffer group: the counters, the output area and a pending result of the handle are not
// touched.  On FZB_OK the stream has drained and *stats holds `st`.
template <class Scan, class Tail>
static int near_frame(fzb_haystack *h, bool steps, fzb_stats st, fzb_stats *stats, Scan scan, Tail tail) {
    uint64_t *d_steps = h->nearb->steps();
    CK(cudaEventRecord(h->ev[0], h->stream));
    if (steps) CK(cudaMemsetAsync(d_steps, 0, sizeof(uint64_t), h->stream));
    TRY(scan(st));
    CK(cudaEventRecord(h->ev[1], h->stream));
    TRY(tail(st));
    CK(cudaEventRecord(h->ev[2], h->stream));
    if (steps) CK(cudaMemcpyAsync(&st.bytes_scanned, d_steps, sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, h->ev[0], h->ev[2]));
    st.gpu_ms = ms;
    CK(cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]));
    st.filter_ms = ms;
    if (stats) *stats = st;
    return FZB_OK;
}

// One pattern over the whole buffer, per record on a handle with a record set, under substitutions only if `ham`
// (DESIGN.md section 5.16), anchored at `anchor` (section 5.18).  On FZB_OK the group's words hold the answer: the
// whole sequence's dist << 48 | first_end and n_ends, or one word dist << 32 | end per record (all ones: no value).
static int nearest_single(fzb_haystack *h, const uint8_t *pattern, uint32_t m, bool ham, uint32_t anchor,
                          fzb_stats *stats) {
    CK(cudaSetDevice(h->device));
    TRY(ensure_near_bufs(h, 0, h->recs ? h->recs->d_off.size() - 1 : 0, 0));
    uint64_t *words = h->nearb->d_words.get(), *partial = h->nearb->partials();
    const auto none = [](fzb_stats &) { return FZB_OK; };
    fzb_stats st{};
    if (anchor) {
        st.route = 16;
        return near_frame(h, true, st, stats, [&](fzb_stats &s) {
            TRY(near_anchored_enqueue(h, pattern, m, ham, anchor == FZB_F_ANCHOR_END, words, s));
            return anchor == FZB_F_ANCHOR_END ? near_flip(h, words, s) : FZB_OK;
        }, none);
    }
    st.route = ham ? 13 : 11;
    int grid = 0;
    return near_frame(h, false, st, stats, [&](fzb_stats &s) {
        if (!h->recs) {  // the end position 0 (substitutions only: no value), no end counted yet
            k_nearest_fill<<<1, 32, 0, h->stream>>>(words, 1, ham ? kBestEmpty : (uint64_t)m << 48);
            CK(cudaMemsetAsync(words + 1, 0, sizeof(uint64_t), h->stream));
            CK(cudaGetLastError());
            s.n_launches++;
        }
        return near_scan_enqueue(h, pattern, m, ham, words, partial, words, s, &grid);
    }, [&](fzb_stats &s) {
        if (h->recs) return FZB_OK;
        k_nearest_count<<<1, 256, 0, h->stream>>>(words, partial, (uint32_t)grid, ham ? ~0u : m);
        CK(cudaGetLastError());
        s.n_launches++;
        return FZB_OK;
    });
}

// The scans of all `count` patterns over the whole buffer, per record on a handle with a record set, under
// substitutions only if `ham`: the patterns of up to 64 symbols in groups of 32 lanes (k_nearest_batch_scan, one launch
// per word class), longer ones one by one (near_scan_enqueue, folded by k_nearest_fold per record).  `anchor` (record
// sets only): the same groups and folds through k_nearest_anchored (DESIGN.md section 5.18), g lanes per record.  On
// FZB_OK the group's words hold the answer: one word per pattern, or best[records] then top2[records].
static int nearest_batch(fzb_haystack *h, const uint8_t *patterns, const uint32_t *offsets, uint32_t count, bool ham,
                         uint32_t anchor, fzb_stats *stats) {
    const bool end = anchor == FZB_F_ANCHOR_END, rev = end && !ham;  // rev: 'end' walks back with reversed patterns
    auto len = [&](uint32_t i) { return offsets[i + 1] - offsets[i]; };
    // by (class, m): the lanes of a group share the warm-up of its longest pattern
    std::vector<uint32_t> order, longs;
    for (uint32_t i = 0; i < count; i++) (len(i) <= kNearBatchMaxM ? order : longs).push_back(i);
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) {
        return std::make_pair(len(x) > 32, len(x)) < std::make_pair(len(y) > 32, len(y));
    });
    std::vector<uint32_t> lanes;
    std::vector<uint8_t> pats;
    uint32_t groups[2] = {0, 0};
    for (uint32_t i : order) {
        const int cls = len(i) > 32;
        if (cls == 1 && groups[1] == 0) lanes.resize(round_up(lanes.size(), kNearBatchLanes), 0);
        if (lanes.size() % kNearBatchLanes == 0) groups[cls]++;
        lanes.push_back(len(i) | i << 16);
    }
    lanes.resize(round_up(lanes.size(), kNearBatchLanes), 0);
    pats.assign(lanes.size() * kNearBatchMaxM, 0);
    for (size_t l = 0; l < lanes.size(); l++)
        for (uint32_t i = 0, m = lanes[l] & 0xFFFFu; i < m; i++)
            pats[l * kNearBatchMaxM + i] = patterns[offsets[lanes[l] >> 16] + (rev ? m - 1 - i : i)];

    CK(cudaSetDevice(h->device));
    const uint64_t nrec = h->recs ? h->recs->d_off.size() - 1 : 0;
    TRY(ensure_near_bufs(h, lanes.size(), h->recs ? 2 * nrec : count, longs.empty() ? 0 : nrec));
    const NearBufs *g = h->nearb.get();
    uint64_t *best = g->d_words.get(), *top2 = best + nrec;
    fzb_stats st{};
    st.route = anchor ? 16 : ham ? 14 : 12;
    return near_frame(h, anchor != 0, st, stats, [&](fzb_stats &st) {
        if (!lanes.empty()) {
            CK(cudaMemcpyAsync(g->d_lanes.get(), lanes.data(), lanes.size() * sizeof(uint32_t), cudaMemcpyHostToDevice,
                               h->stream));
            CK(cudaMemcpyAsync(g->d_pats.get(), pats.data(), pats.size(), cudaMemcpyHostToDevice, h->stream));
        }
        if (h->recs) {  // the constants of nearest_kernels.cuh: (min m, its ordinal, end 0) and the two smallest
                        // (m_i, i); nothing under substitutions only, where no pattern has a value before its first window
            uint64_t key = kBestEmpty, pair2 = kBestEmpty;
            for (uint32_t i = 0; i < count && !ham; i++) {
                key = std::min<uint64_t>(key, (uint64_t)len(i) << 48 | (uint64_t)i << 32);
                pair2 = best_top2_merge(pair2, len(i) << 16 | i);
            }
            k_nearest_fill<<<near_rec_grid(h, nrec), 256, 0, h->stream>>>(best, nrec, key);
            k_nearest_fill<<<near_rec_grid(h, nrec), 256, 0, h->stream>>>(top2, nrec, pair2);
            st.n_launches += 2;
        } else {  // every pattern's end position 0 (substitutions only: no value)
            std::vector<uint64_t> init(count);
            for (uint32_t i = 0; i < count; i++) init[i] = ham ? kBestEmpty : (uint64_t)len(i) << 48;
            CK(cudaMemcpyAsync(best, init.data(), count * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
            CK(cudaStreamSynchronize(h->stream));  // (`init` is a pageable local)
        }
        CK(cudaGetLastError());
        uint32_t lane0 = 0;
        for (int cls = 0; cls < 2; cls++) {
            if (!groups[cls]) continue;
            const int bits = cls ? 64 : 32;
            const uint32_t *cls_lanes = g->d_lanes.get() + lane0;
            const uint8_t *cls_pats = g->d_pats.get() + (uint64_t)lane0 * kNearBatchMaxM;
            lane0 += groups[cls] * kNearBatchLanes;
            if (anchor) {  // g: the class's pattern count rounded up to a power of two, at most 32
                const uint32_t n_cls = (uint32_t)std::count_if(order.begin(), order.end(),
                                                               [&](uint32_t i) { return (len(i) > 32) == (cls == 1); });
                NearAnchParams p{};
                p.H = h->d;
                p.nrec = nrec;
                p.lanes = cls_lanes;
                p.pats = cls_pats;
                p.best = best;
                p.top2 = top2;
                p.steps = g->steps();
                p.end = end;
                for (p.g = 1; p.g < (int32_t)std::min<uint32_t>(n_cls, kNearBatchLanes); p.g *= 2) {}
                TRY(launch_near_anchored(h, bits, ham, true, groups[cls], p));
                st.n_launches++;
                continue;
            }
            // one wave of CTAs over all groups, one segment per warp: long segments (a small warm-up share) on a long
            // sequence, at least kNearBatchMinSeg on a short one
            uint64_t gx = std::max<uint64_t>(1, (uint64_t)h->sm_count * near_ctas_per_sm(bits) / groups[cls]);
            const uint64_t warps = gx * (kNearThreads / 32);
            NearBatchParams p{};
            p.H = h->d;
            p.N = (int64_t)h->buf_len;
            p.seg = (int64_t)std::max<uint64_t>(kNearBatchMinSeg, round_up((h->buf_len + warps - 1) / warps, 16));
            gx = std::min<uint64_t>(gx, (h->buf_len + (kNearThreads / 32) * p.seg - 1) / ((kNearThreads / 32) * p.seg));
            p.lanes = cls_lanes;
            p.pats = cls_pats;
            p.whole = best;
            p.best = best;
            p.top2 = top2;
            if (gx == 0) continue;  // (an empty buffer)
            TRY(launch_near_batch_scan(h, bits, ham, dim3((unsigned)gx, groups[cls]), p));
            st.n_launches++;
            st.bytes_scanned += h->buf_len;
        }
        for (uint32_t i : longs) {  // 65-255 symbols: the single scan, pattern by pattern, folded per record
            const uint32_t m = len(i);
            int grid = 0;
            if (anchor)
                TRY(near_anchored_enqueue(h, patterns + offsets[i], m, ham, end, g->rec_words(), st));
            else  // (whole sequence: into the pattern's word, prefilled)
                TRY(near_scan_enqueue(h, patterns + offsets[i], m, ham, best + i, g->partials(), g->rec_words(), st, &grid));
            if (h->recs) {
                k_nearest_fold<<<near_rec_grid(h, nrec), 256, 0, h->stream>>>(g->rec_words(), nrec, ham ? m + 1 : m, i,
                                                                             best, top2);
                CK(cudaGetLastError());
                st.n_launches++;
            }
        }
        return end ? near_flip(h, best, st) : FZB_OK;  // (the winners' ends in the mirrored records -> their starts)
    }, [](fzb_stats &) { return FZB_OK; });
}

// The refusals of a nearest call, in the order that decides its code: `what` names the call; it takes
// FZB_F_SUBSTITUTIONS_ONLY and the flags of `anchors`, needs a record set if `per_record` (and refuses one
// otherwise), and a whole (unsharded) sequence outside a world if `whole`.  A batch's `count` patterns are checked
// before the record set; a single search checks its one pattern after this call.
static int check_nearest(const fzb_haystack *h, const char *what, uint32_t flags, uint32_t anchors, bool per_record,
                         bool whole, const uint8_t *patterns = nullptr, const uint32_t *offsets = nullptr,
                         uint32_t count = 0) {
    if (per_record && !h->recs) return fail(FZB_E_INVALID, "%s needs a handle with a record set", what);
    if (flags & ~(FZB_F_SUBSTITUTIONS_ONLY | anchors))
        return fail(FZB_E_UNSUPPORTED, "%s takes no flag other than FZB_F_SUBSTITUTIONS_ONLY%s", what,
                    anchors ? " and one anchor" : "");
    if ((flags & anchors) == (FZB_F_ANCHOR_START | FZB_F_ANCHOR_END))
        return fail(FZB_E_INVALID, "FZB_F_ANCHOR_START and FZB_F_ANCHOR_END exclude each other");
    if (whole && (!is_whole_sequence(h) || h->comm || h->local_world || h->peer))
        return fail(FZB_E_UNSUPPORTED, "%s needs a whole (unsharded) sequence outside a world", what);
    if (count > kBestMaxPatterns) return fail(FZB_E_UNSUPPORTED, "more than %u patterns in one %s call", kBestMaxPatterns, what);
    for (uint32_t i = 0; i < count; i++) {
        if (offsets[i + 1] < offsets[i]) return fail(FZB_E_INVALID, "offsets must be non-decreasing");
        TRY(check_pattern(h, patterns + offsets[i], offsets[i + 1] - offsets[i], 0));
    }
    if (!per_record) return refuse_records(h, what);
    if (h->recs->longest > (1ull << 32)) return fail(FZB_E_UNSUPPORTED, "%s needs records shorter than 2^32", what);
    return FZB_OK;
}

// The first n answer words of the call that just ran
static int near_read(fzb_haystack *h, std::vector<uint64_t> &words, uint64_t n) {
    words.resize(n);
    CK(cudaMemcpyAsync(words.data(), h->nearb->d_words.get(), n * sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return FZB_OK;
}

extern "C" int fzb_nearest_distance(fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t flags,
                                    uint32_t *dist, uint64_t *n_ends, uint64_t *first_end, fzb_stats *stats) {
    HandleLock handle_lock(h);
    if (!h || !dist || !n_ends || !first_end) return fail(FZB_E_INVALID, "NULL argument");
    TRY(check_nearest(h, "fzb_nearest_distance", flags, 0, false, true));
    TRY(check_pattern(h, pattern, m, 0));
    TRY(nearest_single(h, pattern, m, (flags & FZB_F_SUBSTITUTIONS_ONLY) != 0, 0, stats));
    std::vector<uint64_t> out;
    TRY(near_read(h, out, 2));
    const bool none = out[0] == kBestEmpty;  // (substitutions only: the sequence is shorter than the pattern)
    *dist = none ? UINT32_MAX : (uint32_t)(out[0] >> 48);
    *first_end = none ? UINT64_MAX : out[0] & kNearNoEnd;
    *n_ends = out[1];
    return FZB_OK;
}

extern "C" int fzb_nearest_per_record(fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t flags,
                                      int32_t *dist, int64_t *end, fzb_stats *stats) {
    HandleLock handle_lock(h);
    if (!h || !dist || !end) return fail(FZB_E_INVALID, "NULL argument");
    TRY(check_nearest(h, "fzb_nearest_per_record", flags, FZB_F_ANCHOR_START | FZB_F_ANCHOR_END, true, false));
    TRY(check_pattern(h, pattern, m, 0));
    TRY(nearest_single(h, pattern, m, (flags & FZB_F_SUBSTITUTIONS_ONLY) != 0,
                       flags & (FZB_F_ANCHOR_START | FZB_F_ANCHOR_END), stats));
    // one read-back of 8 bytes per record
    const uint64_t nrec = h->recs->d_off.size() - 1;
    std::vector<uint64_t> words;
    TRY(near_read(h, words, nrec));
    for (uint64_t r = 0; r < nrec; r++) {
        const bool none = words[r] == kBestEmpty;  // (substitutions only: a record shorter than the pattern)
        dist[r] = none ? -1 : (int32_t)(words[r] >> 32);
        end[r] = none ? -1 : (int64_t)(words[r] & 0xFFFFFFFFull);
    }
    return FZB_OK;
}

extern "C" int fzb_nearest_distance_batch(fzb_haystack *h, const uint8_t *patterns, const uint32_t *offsets,
                                          uint32_t count, uint32_t flags, uint32_t *dist, uint64_t *first_end,
                                          fzb_stats *stats) {
    HandleLock handle_lock(h);
    if (!h || (count && (!patterns || !offsets || !dist || !first_end))) return fail(FZB_E_INVALID, "NULL argument");
    TRY(check_nearest(h, "fzb_nearest_distance_batch", flags, 0, false, true, patterns, offsets, count));
    if (stats) *stats = fzb_stats{};
    if (count == 0) return FZB_OK;
    TRY(nearest_batch(h, patterns, offsets, count, (flags & FZB_F_SUBSTITUTIONS_ONLY) != 0, 0, stats));
    // one read-back of 8 bytes per pattern
    std::vector<uint64_t> words;
    TRY(near_read(h, words, count));
    for (uint32_t i = 0; i < count; i++) {
        const bool none = words[i] == kBestEmpty;  // (substitutions only: a pattern longer than the sequence)
        dist[i] = none ? UINT32_MAX : (uint32_t)(words[i] >> 48);
        first_end[i] = none ? UINT64_MAX : words[i] & kNearNoEnd;
    }
    return FZB_OK;
}

extern "C" int fzb_nearest_best_per_record(fzb_haystack *h, const uint8_t *patterns, const uint32_t *offsets,
                                           uint32_t count, uint32_t flags, int32_t *pattern, int32_t *dist,
                                           int64_t *end, int32_t *second_pattern, int32_t *second_dist,
                                           fzb_stats *stats) {
    HandleLock handle_lock(h);
    if (!h || !pattern || !dist || !end || !second_pattern || !second_dist || (count && (!patterns || !offsets)))
        return fail(FZB_E_INVALID, "NULL argument");
    TRY(check_nearest(h, "fzb_nearest_best_per_record", flags, FZB_F_ANCHOR_START | FZB_F_ANCHOR_END, true, true,
                      patterns, offsets, count));
    const uint64_t nrec = h->recs->d_off.size() - 1;
    if (stats) *stats = fzb_stats{};
    if (count == 0) {
        for (uint64_t r = 0; r < nrec; r++) {
            pattern[r] = dist[r] = second_pattern[r] = second_dist[r] = -1;
            end[r] = -1;
        }
        return FZB_OK;
    }
    TRY(nearest_batch(h, patterns, offsets, count, (flags & FZB_F_SUBSTITUTIONS_ONLY) != 0,
                      flags & (FZB_F_ANCHOR_START | FZB_F_ANCHOR_END), stats));
    // one read-back of 16 bytes per record
    std::vector<uint64_t> words;
    TRY(near_read(h, words, 2 * nrec));
    for (uint64_t r = 0; r < nrec; r++) {
        const uint64_t b = words[r];
        const uint32_t second = (uint32_t)words[nrec + r] & kBestPairNone;
        const bool none = b == kBestEmpty;  // (substitutions only: no pattern fits in the record)
        dist[r] = none ? -1 : (int32_t)(b >> 48);
        pattern[r] = none ? -1 : (int32_t)((b >> 32) & 0xFFFFu);
        end[r] = none ? -1 : (int64_t)(b & 0xFFFFFFFFull);
        second_dist[r] = second == kBestPairNone ? -1 : (int32_t)(second >> 16);
        second_pattern[r] = second == kBestPairNone ? -1 : (int32_t)(second & 0xFFFFu);
    }
    return FZB_OK;
}

// ------------------------------------------------------------------------------------------------
// fzb_align (DESIGN.md section 5.17): the edit operations of matches, one warp per item
// ------------------------------------------------------------------------------------------------
// The class of a pattern by choose_search_class's rule on normalised limits (as plan_by_class decides it)
static uint8_t align_class(uint32_t max_subs, uint32_t max_ins, uint32_t max_dels, uint32_t max_l) {
    if (max_l == 0) return kAlignExact;
    if (max_ins == 0 && max_dels == 0) return kAlignHamming;
    if (max_l <= std::min(max_subs, std::min(max_ins, max_dels))) return kAlignLevenshtein;
    return kAlignGeneric;
}

// Item i checked and turned into an AlignItem with its clamped bounds; *need = its shared-memory bytes, 0 for an item
// that cannot have an alignment (its outputs stay -1 and it is not launched).
static int prepare_align_item(const fzb_haystack *h, const std::vector<uint64_t> &off, uint64_t i, const uint32_t *offsets,
                              uint32_t count, const uint32_t *max_subs, const uint32_t *max_ins,
                              const uint32_t *max_dels, const uint32_t *max_l_dist, const uint32_t *item_pattern,
                              const int64_t *item_start, const int64_t *item_end, const int32_t *item_dist,
                              const uint64_t *op_offsets, AlignItem &it, uint64_t *need) {
    const unsigned long long ii = i;
    const uint32_t p = item_pattern[i];
    if (p >= count) return fail(FZB_E_INVALID, "item %llu: unknown pattern index %u", ii, p);
    const int64_t s = item_start[i], e = item_end[i];
    const uint64_t n = h->global_len;
    if (e < 0 || (uint64_t)e > n || s < -1) return fail(FZB_E_INVALID, "item %llu: outside the buffer", ii);
    if (s > e) return fail(FZB_E_INVALID, "item %llu: start > end", ii);
    if (item_dist[i] < 0) return fail(FZB_E_INVALID, "item %llu: negative cost bound", ii);
    int64_t lo = 0;
    if (!off.empty()) {  // the record holding end position e: off[r] <= e <= off[r + 1] - 1
        const uint64_t r = (uint64_t)(std::upper_bound(off.begin(), off.end(), (uint64_t)e) - off.begin()) - 1;
        if (r + 1 >= off.size()) return fail(FZB_E_INVALID, "item %llu: outside the records", ii);
        lo = (int64_t)off[r];
        if (s >= 0 && s < lo) return fail(FZB_E_INVALID, "item %llu: the window crosses a record edge", ii);
    }
    const uint32_t m = offsets[p + 1] - offsets[p];
    const uint8_t cls = align_class(max_subs[p], max_ins[p], max_dels[p], max_l_dist[p]);
    if (s < 0 && (cls == kAlignExact || cls == kAlignGeneric))
        return fail(FZB_E_INVALID, "item %llu: a free start needs a Levenshtein or substitutions-only pattern", ii);
    if (s >= 0 && (cls == kAlignExact || cls == kAlignHamming) && (uint64_t)(e - s) != m)
        return fail(FZB_E_INVALID, "item %llu: the window of an exact or substitutions-only pattern must have its length", ii);
    const int64_t d = item_dist[i];
    if (s < 0 && cls == kAlignLevenshtein && d > (int64_t)m)
        return fail(FZB_E_UNSUPPORTED, "item %llu: a free start with a cost bound above the pattern's length", ii);
    const uint64_t w_room = s >= 0 ? (uint64_t)(e - s) : cls == kAlignHamming ? m : (uint64_t)std::min<int64_t>(m + d, e - lo);
    if (op_offsets[i + 1] < op_offsets[i] || op_offsets[i + 1] - op_offsets[i] < m + w_room)
        return fail(FZB_E_INVALID, "item %llu: room for fewer than m + w ops", ii);

    it = AlignItem{};
    it.s = s;
    it.e = e;
    it.lo = lo;
    it.op_off = op_offsets[i];
    it.idx = i;
    it.pat_off = offsets[p];
    it.m = (uint16_t)m;
    it.cls = cls;
    *need = 0;
    const int64_t L = max_l_dist[p];
    if (cls == kAlignExact || cls == kAlignHamming) {
        it.d = (int32_t)std::min<int64_t>(std::min<int64_t>(d, m), cls == kAlignExact ? 0 : std::min<int64_t>(max_subs[p], L));
        *need = 1;
        return FZB_OK;
    }
    // no alignment costs more than max(m, w): a larger bound of an anchored item is lowered to it
    int64_t de = std::min(d, L);
    if (s >= 0) de = std::min<int64_t>(de, std::max<int64_t>(m, e - s));
    if (s < 0 && de < d) return FZB_OK;  // (a free start at d > max_l_dist: no alignment within the limits)
    if (de >= kAlignInf) return fail(FZB_E_UNSUPPORTED, "item %llu: a cost bound of %d or more", ii, kAlignInf);
    it.d = (int32_t)de;
    if (cls == kAlignLevenshtein) {
        if (s >= 0) {
            int kmin;
            const int bw = align_lev_band((int)m, std::min<int64_t>(e - s, 2 * (int64_t)kAlignInf), (int)de, &kmin);
            if (bw == 0) return FZB_OK;  // |w - m| > d
            *need = align_vals_bytes(1, bw) + align_table_bytes(1, (int)m, bw);
        } else {
            *need = std::max<uint64_t>(align_vals_bytes(1, 2 * (int)de + 1) + 2 * (2 * de + 1),
                                       align_vals_bytes(1, (int)de + 1) + align_table_bytes(1, (int)m, (int)de + 1));
        }
    } else {
        const int64_t ins = std::min<int64_t>(max_ins[p], de), dels = std::min<int64_t>(max_dels[p], de);
        const int64_t subs = std::min<int64_t>(std::min<int64_t>(max_subs[p], de), m);
        it.subs = (uint16_t)subs;
        it.ins = (uint16_t)std::min<int64_t>(ins, 0xFFFF);
        it.dels = (uint16_t)std::min<int64_t>(dels, 0xFFFF);
        it.lim = (uint16_t)std::min<int64_t>(de, subs + ins + dels);
        *need = align_vals_bytes((int)ins + 1, (int)dels + 1) + align_table_bytes((int)ins + 1, (int)m, (int)dels + 1);
        if (*need > (uint64_t)kAlignSmemMax)
            return fail(FZB_E_UNSUPPORTED,
                        "item %llu: the generic table of %llu bytes exceeds the %d bytes of shared memory of an item",
                        ii, (unsigned long long)*need, kAlignSmemMax);
    }
    if (*need > (uint64_t)kAlignSmemMax)
        return fail(FZB_E_UNSUPPORTED, "item %llu: a band of %llu bytes exceeds the %d bytes of shared memory of an item",
                    ii, (unsigned long long)*need, kAlignSmemMax);
    return FZB_OK;
}

extern "C" int fzb_align(fzb_haystack *h, const uint8_t *patterns, const uint32_t *offsets, uint32_t count,
                         const uint32_t *max_subs, const uint32_t *max_ins, const uint32_t *max_dels,
                         const uint32_t *max_l_dist, const uint32_t *item_pattern, const int64_t *item_start,
                         const int64_t *item_end, const int32_t *item_dist, uint64_t n_items, uint32_t flags,
                         int64_t *start, int32_t *cost, int32_t *n_subs, int32_t *n_ins, int32_t *n_dels,
                         const uint64_t *op_offsets, uint8_t *ops, fzb_stats *stats) {
    HandleLock handle_lock(h);
    if (!h || (count && (!patterns || !offsets || !max_subs || !max_ins || !max_dels || !max_l_dist)) ||
        (n_items && (!item_pattern || !item_start || !item_end || !item_dist || !start || !cost || !n_subs || !n_ins ||
                     !n_dels || !op_offsets || !ops)))
        return fail(FZB_E_INVALID, "NULL argument");
    if (flags) return fail(FZB_E_UNSUPPORTED, "fzb_align takes no flag");
    if (!is_whole_sequence(h) || h->comm || h->local_world || h->peer)
        return fail(FZB_E_UNSUPPORTED, "fzb_align needs a whole (unsharded) sequence outside a world");
    for (uint32_t p = 0; p < count; p++) {
        if (offsets[p + 1] < offsets[p]) return fail(FZB_E_INVALID, "offsets must be non-decreasing");
        TRY(check_pattern(h, patterns + offsets[p], offsets[p + 1] - offsets[p], 0));
    }
    if (stats) *stats = fzb_stats{};
    if (n_items == 0) return FZB_OK;
    CK(cudaSetDevice(h->device));
    std::vector<uint64_t> off;
    if (h->recs) {
        off.resize(h->recs->d_off.size());
        CK(cudaMemcpyAsync(off.data(), h->recs->d_off.get(), off.size() * sizeof(uint64_t), cudaMemcpyDeviceToHost,
                           h->stream));
        CK(cudaStreamSynchronize(h->stream));
    }
    // every item checked before any work; the launched ones ordered by their shared-memory bucket
    std::vector<AlignItem> items;
    std::vector<uint64_t> per_bucket(kAlignBuckets, 0);
    std::vector<uint8_t> bucket(n_items, 0xFF);
    for (uint64_t i = 0; i < n_items; i++) {
        AlignItem it;
        uint64_t need;
        TRY(prepare_align_item(h, off, i, offsets, count, max_subs, max_ins, max_dels, max_l_dist, item_pattern,
                               item_start, item_end, item_dist, op_offsets, it, &need));
        if (!need) continue;
        int b = 0;
        while ((uint64_t)kAlignBucketBytes[b] < need) b++;
        bucket[i] = (uint8_t)b;
        per_bucket[b]++;
    }
    std::vector<uint64_t> first(kAlignBuckets + 1, 0);
    for (int b = 0; b < kAlignBuckets; b++) first[b + 1] = first[b] + per_bucket[b];
    items.resize(first[kAlignBuckets]);
    {
        std::vector<uint64_t> at(first.begin(), first.end() - 1);
        for (uint64_t i = 0; i < n_items; i++) {
            if (bucket[i] == 0xFF) continue;
            uint64_t need;
            TRY(prepare_align_item(h, off, i, offsets, count, max_subs, max_ins, max_dels, max_l_dist, item_pattern,
                                   item_start, item_end, item_dist, op_offsets, items[at[bucket[i]]++], &need));
        }
    }
    const uint64_t n_ops = op_offsets[n_items], n_pat = count ? offsets[count] : 0;
    // the call's own buffers, freed when it returns: the handle's counters, output area and pending result stay as
    // they were
    DevBuf<AlignItem> d_items;
    DevBuf<uint8_t> d_pats, d_ops;
    DevBuf<int64_t> d_start;
    DevBuf<int32_t> d_ints;
    TRY(d_items.alloc(std::max<uint64_t>(items.size(), 1)));
    TRY(d_pats.alloc(std::max<uint64_t>(n_pat, 1)));
    TRY(d_ops.alloc(std::max<uint64_t>(n_ops, 1)));
    TRY(d_start.alloc(n_items));
    TRY(d_ints.alloc(4 * n_items));
    AlignOut out{d_start.get(), d_ints.get(), d_ints.get() + n_items, d_ints.get() + 2 * n_items,
                 d_ints.get() + 3 * n_items, d_ops.get()};
    fzb_stats st{};
    st.route = 15;
    st.n_candidates = items.size();
    CK(cudaEventRecord(h->ev[0], h->stream));
    CK(cudaMemsetAsync(d_start.get(), 0xFF, n_items * sizeof(int64_t), h->stream));  // -1 everywhere
    CK(cudaMemsetAsync(d_ints.get(), 0xFF, 4 * n_items * sizeof(int32_t), h->stream));
    if (!items.empty())
        CK(cudaMemcpyAsync(d_items.get(), items.data(), items.size() * sizeof(AlignItem), cudaMemcpyHostToDevice,
                           h->stream));
    if (n_pat) CK(cudaMemcpyAsync(d_pats.get(), patterns, n_pat, cudaMemcpyHostToDevice, h->stream));
    CK(cudaFuncSetAttribute(k_align, cudaFuncAttributeMaxDynamicSharedMemorySize, kAlignSmemMax));
    for (int b = 0; b < kAlignBuckets; b++) {
        const uint64_t nb = first[b + 1] - first[b];
        if (!nb) continue;
        const int per_sm = std::max(1, std::min(32, (int)(200 * 1024 / kAlignBucketBytes[b])));
        const int grid = (int)std::min<uint64_t>(nb, (uint64_t)h->sm_count * per_sm);
        k_align<<<grid, 32, kAlignBucketBytes[b], h->stream>>>(h->d, d_pats.get(), d_items.get() + first[b], nb, out);
        CK(cudaGetLastError());
        st.n_launches++;
    }
    CK(cudaEventRecord(h->ev[1], h->stream));
    CK(cudaMemcpyAsync(start, d_start.get(), n_items * sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream));
    int32_t *cols[4] = {cost, n_subs, n_ins, n_dels};
    for (int c = 0; c < 4; c++)
        CK(cudaMemcpyAsync(cols[c], d_ints.get() + c * n_items, n_items * sizeof(int32_t), cudaMemcpyDeviceToHost,
                           h->stream));
    if (n_ops) CK(cudaMemcpyAsync(ops, d_ops.get(), n_ops, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, h->ev[0], h->ev[1]));
    st.gpu_ms = st.filter_ms = ms;
    if (stats) *stats = st;
    return FZB_OK;
}

// One cached workspace per device for the one-shot call: the analogue of the reference's reusable
// chunk buffer (__init__.py:141-145) -- a call then costs one H2D copy plus the kernels instead of
// a 4 GiB cudaMalloc/cudaFree pair and a dozen small allocations.
static std::mutex g_ws_mutex;
static fzb_haystack *g_ws[64];

extern "C" void fzb_release_workspace(void) {
    std::lock_guard<std::mutex> lock(g_ws_mutex);
    for (auto &h : g_ws) {
        if (h) fzb_haystack_destroy(h);
        h = nullptr;
    }
}

extern "C" int fzb_find_near_matches(const uint8_t *pattern, uint32_t m, const uint8_t *haystack, uint64_t n,
                                     uint32_t max_subs, uint32_t max_ins, uint32_t max_dels, uint32_t max_l,
                                     int device, fzb_result **out) {
    if (!out) return fail(FZB_E_INVALID, "out is NULL");
    *out = nullptr;
    if (device < 0 || device >= 64 || device >= fzb_device_count())
        return fail(FZB_E_CUDA, "CUDA device %d not available (%d devices)", device, fzb_device_count());
    std::lock_guard<std::mutex> lock(g_ws_mutex);
    fzb_haystack *&h = g_ws[device];
    if (!h || round_up(n, 128) + 128 > h->owned_buf.size()) {
        if (h) fzb_haystack_destroy(h);
        h = nullptr;
        const uint64_t cap = std::max<uint64_t>(n + n / 8, 1u << 20);  // head-room: repeated calls with growing inputs
        int rc = fzb_haystack_alloc(cap, 0, cap, 0, cap, device, &h, nullptr);
        if (rc) return rc;
    }
    int rc = fzb_haystack_upload(h, haystack, n);
    if (rc) return rc;
    return search_by_class(h, pattern, m, max_subs, max_ins, max_dels, max_l, 0, out);
}

// ------------------------------------------------------------------------------------------------
// has_near_match: "is there any match?" with early termination.  The reference's has_near_match_* helpers
// (substitutions_only.py:18-34,139-145,218-233; generic_search.py:240-253; _substitutions_only.c:4-17) stop at the
// first hit of a left-to-right scan.  A GPU scans everywhere at once, so the stop is made coarse instead: the
// sequence is searched in chunks of geometrically growing size (64 MiB, 256 MiB, 1 GiB, the rest), each chunk a
// VIEW of the resident buffer searched exactly like a shard (own range = the chunk, halo from its neighbours,
// window clipping at the global ends only -- so the union of the chunks' raw streams is the whole raw stream);
// the call returns after the first chunk that yields a raw match.  A match near the start costs ~0.1 ms
// whatever the length of the sequence; no match at all costs the full scan plus three chunk turn-arounds.
// ------------------------------------------------------------------------------------------------
extern "C" int fzb_has_near_match(fzb_haystack *h, const uint8_t *pattern, uint32_t m, uint32_t max_subs,
                                  uint32_t max_ins, uint32_t max_dels, uint32_t max_l, int *found) {
    HandleLock handle_lock(h);
    if (!h || !found) return fail(FZB_E_INVALID, "NULL argument");
    *found = 0;
    TRY(refuse_records(h, "has_near_match"));
    int rc = check_pattern(h, pattern, m, 0);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    if (h->buf_len) sample_collision_prob(h);  // byte statistics of the WHOLE buffer (the views reuse them)
    BufferView whole(h);  // (its fields: the geometry of the whole buffer)
    const uint64_t halo = round_up((uint64_t)m + std::min<uint64_t>(max_l, m), 128) + 128;
    uint64_t chunk = 64ull << 20, lo = whole.own_lo;
    if (const char *e = getenv("FZB_HAS_CHUNK_BYTES"))  // testing: chunk seams on small sequences
        chunk = std::max<uint64_t>(128, round_up(strtoull(e, nullptr, 10), 128));
    do {  // (at least one pass: an empty sequence still has its k >= m matches)
        uint64_t hi = std::min(whole.own_hi, round_up(lo + chunk, 128));
        if (whole.own_hi - hi < chunk / 4) hi = whole.own_hi;  // no tiny last chunk
        // the chunk plus its halo, 128-byte aligned relative to the buffer start
        const uint64_t want_lo = lo > whole.buf_lo + halo ? lo - halo : whole.buf_lo;
        whole.set(whole.buf_lo + (want_lo - whole.buf_lo) / 128 * 128, std::min(whole.buf_lo + whole.buf_len, hi + halo),
                  lo, hi);
        fzb_result *res = nullptr;
        rc = search_by_class(h, pattern, m, max_subs, max_ins, max_dels, max_l, FZB_F_NO_FINAL, &res);  // raw stream only
        if (rc == FZB_OK && fzb_result_count(res, FZB_RAW) > 0) *found = 1;
        if (res) fzb_result_destroy(res);
        lo = hi;
        chunk *= 4;
    } while (rc == FZB_OK && !*found && lo < whole.own_hi);
    return rc;
}

extern "C" int fzb_debug_counters(const fzb_haystack *h, uint32_t out[32]) {
    if (!h || !out) return fail(FZB_E_INVALID, "NULL argument");
    memset(out, 0, 32 * sizeof(uint32_t));
    memcpy(out, h->h_counters.get(), CNT_COUNT * sizeof(uint32_t));
    if (h->peer) memcpy(out + 16, h->peer->h_ghdr.get(), 16 * sizeof(uint32_t));
    return FZB_OK;
}

// ------------------------------------------------------------------------------------------------
// test hook: the expansion routines of the verify kernels on caller-supplied (sub, seq, budget) cases
// ------------------------------------------------------------------------------------------------
extern "C" int fzb_debug_expand(const uint8_t *subs, const uint32_t *sub_off, const uint8_t *seqs,
                                const uint32_t *seq_off, const int32_t *max_l, const int32_t *variant, uint32_t count,
                                int device, int32_t *out) {
    if (count && (!subs || !sub_off || !seqs || !seq_off || !max_l || !variant || !out))
        return fail(FZB_E_INVALID, "NULL argument");
    if (device < 0 || device >= fzb_device_count()) return fail(FZB_E_CUDA, "CUDA device %d not available", device);
    if (count == 0) return FZB_OK;
    for (uint32_t i = 0; i < count; i++) {
        if (sub_off[i + 1] < sub_off[i] || seq_off[i + 1] < seq_off[i]) return fail(FZB_E_INVALID, "bad offsets");
        if (sub_off[i + 1] - sub_off[i] >= (uint32_t)kDbgMax || seq_off[i + 1] - seq_off[i] >= 2u * kDbgMax)
            return fail(FZB_E_UNSUPPORTED, "case %u too long for the debug entry", i);
        if (variant[i] < 0 || variant[i] > 2 || max_l[i] < 0) return fail(FZB_E_INVALID, "bad variant / budget");
    }
    CK(cudaSetDevice(device));
    const size_t nsub = std::max<size_t>(sub_off[count], 1), nseq = std::max<size_t>(seq_off[count], 1);
    DevBuf<uint8_t> d_subs, d_seqs;
    DevBuf<uint32_t> d_so, d_qo;
    DevBuf<int32_t> d_k, d_v, d_out;
    TRY(d_subs.alloc(nsub));
    TRY(d_seqs.alloc(nseq));
    TRY(d_so.alloc(count + 1));
    TRY(d_qo.alloc(count + 1));
    TRY(d_k.alloc(count));
    TRY(d_v.alloc(count));
    TRY(d_out.alloc((uint64_t)count * 8));
    CK(cudaMemcpy(d_subs.get(), subs, sub_off[count], cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_seqs.get(), seqs, seq_off[count], cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_so.get(), sub_off, (count + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_qo.get(), seq_off, (count + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_k.get(), max_l, count * sizeof(int32_t), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_v.get(), variant, count * sizeof(int32_t), cudaMemcpyHostToDevice));
    k_debug_expand<<<count, 32>>>(d_subs.get(), d_so.get(), d_seqs.get(), d_qo.get(), d_k.get(), d_v.get(), d_out.get());
    CK(cudaGetLastError());
    CK(cudaMemcpy(out, d_out.get(), (size_t)count * 8 * sizeof(int32_t), cudaMemcpyDeviceToHost));
    return FZB_OK;
}

// ------------------------------------------------------------------------------------------------
// results
// ------------------------------------------------------------------------------------------------
extern "C" uint64_t fzb_result_count(const fzb_result *r, int which) {
    if (!r) return 0;
    if (which != FZB_RAW && r->has_global) return r->gcount;
    if (which == FZB_RAW) return r->raw_n;
    return r->fin.size();
}

extern "C" int fzb_result_copy(const fzb_result *r, int which, int64_t *start, int64_t *end, int32_t *dist,
                               int32_t *anchor_ngram, int64_t *anchor_idx) {
    if (!r) return fail(FZB_E_INVALID, "result is NULL");
    if (which == FZB_RAW) const_cast<fzb_result *>(r)->order_raw();
    if (which != FZB_RAW && r->has_global) const_cast<fzb_result *>(r)->fetch_raw();  // global rows are fetched lazily
    const std::vector<RawRec> &v = (which != FZB_RAW && r->has_global) ? r->gfin : (which == FZB_RAW ? r->raw : r->fin);
    const bool anchors = (which == FZB_RAW) && (r->stats.route <= 2);
    for (size_t i = 0; i < v.size(); i++) {
        if (start) start[i] = v[i].start;
        if (end) end[i] = v[i].end;
        if (dist) dist[i] = v[i].dist;
        if (anchor_ngram) anchor_ngram[i] = anchors ? v[i].ngram : -1;
        if (anchor_idx) anchor_idx[i] = anchors ? v[i].idx : -1;
    }
    return FZB_OK;
}

extern "C" int fzb_result_stats(const fzb_result *r, fzb_stats *out) {
    if (!r || !out) return fail(FZB_E_INVALID, "NULL argument");
    *out = r->stats;
    return FZB_OK;
}

extern "C" void fzb_result_destroy(fzb_result *r) {
    if (!r) return;
    {
        std::lock_guard<std::mutex> lock(g_pending_mutex);
        if (r->owner) {
            r->owner->pending = nullptr;
            r->owner = nullptr;
        }
    }
    delete r;
}
