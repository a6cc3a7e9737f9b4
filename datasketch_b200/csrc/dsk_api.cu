// dsk_api.cu -- the C-ABI (include/dsk.h): argument validation, permutation analysis,
// kernel selection, and the pipelined host-buffer entry point.
#include <atomic>
#include <mutex>
#include <new>
#include <string.h>
#include <vector>

#include "dsk_common.cuh"
#include "shingle_kernels.cuh"   // the shingle kernels are compiled here, beside their entry points

namespace dsk {

// ---- error plumbing -----------------------------------------------------------------
static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int cuda_fail(cudaError_t e, const char *what) {
    set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
    if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver) return DSK_ERR_NO_DEVICE;
    if (e == cudaErrorMemoryAllocation) return DSK_ERR_NOMEM;
    return DSK_ERR_CUDA;
}

// ---- per-device info cache ---------------------------------------------------------------
struct DevInfo {
    bool known = false;
    int sm_count = 0, cc_major = 0, cc_minor = 0;
    size_t total_mem = 0;
};
static DevInfo g_dev[64];
static std::mutex g_dev_mu;

static int get_dev(int device, DevInfo **out) {
    if (device < 0 || device >= 64) {
        set_error("device index %d out of range", device);
        return DSK_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(g_dev_mu);
    DevInfo &d = g_dev[device];
    if (!d.known) {
        int n = 0;
        DSK_CUDA(cudaGetDeviceCount(&n));
        if (device >= n) {
            set_error("CUDA device %d not present (%d devices); this engine has no CPU fallback", device, n);
            return DSK_ERR_NO_DEVICE;
        }
        cudaDeviceProp p;
        DSK_CUDA(cudaGetDeviceProperties(&p, device));
        d.sm_count = p.multiProcessorCount;
        d.cc_major = p.major;
        d.cc_minor = p.minor;
        d.total_mem = p.totalGlobalMem;
        d.known = true;
    }
    *out = &d;
    return DSK_OK;
}

// ---- permutation analysis -------------------------------------------------------------------
// inverse of an odd 64-bit integer modulo 2^64 (Newton iteration doubles the valid bits)
static uint64_t inv_odd_u64(uint64_t a) {
    uint64_t x = a;  // correct to 3 bits
    for (int i = 0; i < 6; ++i) x *= 2 - a * x;
    return x;
}

// Is there a token value h in [0, 2^32) with ((a*h + b) mod 2^64) in the set where
// `% (2^61-1)` takes its conditional subtract, i.e. (x & p) + (x >> 61) >= p ?
// That set has 36 elements: top3 = j in 0..7 and low61 in [p - j, 2^61 - 1].
static bool perm_unsafe_u32(uint64_t a, uint64_t b) {
    const uint64_t p = (1ull << 61) - 1;
    for (uint64_t j = 0; j < 8; ++j) {
        for (uint64_t lo = p - j; lo <= p; ++lo) {
            const uint64_t x = (j << 61) | lo;
            const uint64_t target = x - b;  // a*h == target (mod 2^64)
            if (a == 0) {
                if (target == 0) return true;
                continue;
            }
            const int e = __builtin_ctzll(a);
            if (e > 0 && (target & ((1ull << e) - 1)) != 0) continue;
            const int nb = 64 - e;  // h is determined modulo 2^nb
            if (nb < 32) return true;  // some representative is always < 2^32
            uint64_t h0 = (target >> e) * inv_odd_u64(a >> e);
            if (nb < 64) h0 &= (1ull << nb) - 1;
            if (h0 < (1ull << 32)) return true;
        }
    }
    return false;
}

}  // namespace dsk

using namespace dsk;

struct dsk_perm {
    int device = 0;
    int num_perm = 0;
    int kpad = 0;
    int n_unsafe = 0;
    uint32_t *d_tab = nullptr;  // a_lo | a_hi | b_lo | b_hi | b_lo + 7 | b_lo + 8, each kpad entries
    unsigned *d_counters = nullptr;  // kCounterSets x kCounterStride work counters (one set per in-flight launch)
    // A launch leases one counter set; the event recorded behind the launch makes the NEXT user of that set wait
    // (stream-ordered, on the device) until the kernel that still reads it has finished -- 64+ launches of one handle
    // outstanding on different streams would otherwise share counters and skip documents.
    mutable std::mutex mu;
    mutable unsigned next_set = 0;
    mutable cudaEvent_t ev[64] = {};
    mutable bool ev_live[64] = {};
    std::vector<uint64_t> a, b;
};
static constexpr int kCounterSets = 64, kCounterStride = 64;

// lease a counter set for one launch on stream s: holds the handle's mutex from acquire to release so that the
// wait -> launch -> record sequence of concurrent host threads cannot interleave
struct CounterLease {
    const dsk_perm *p;
    int set;
    cudaStream_t s;
    unsigned *ptr;
    CounterLease(const dsk_perm *perm, cudaStream_t stream) : p(perm), s(stream) {
        p->mu.lock();
        set = (int)(p->next_set++ % kCounterSets);
        if (p->ev_live[set]) cudaStreamWaitEvent(s, p->ev[set], 0);
        ptr = p->d_counters + (size_t)set * kCounterStride;
    }
    ~CounterLease() {
        if (!p->ev[set]) {
            if (cudaEventCreateWithFlags(&p->ev[set], cudaEventDisableTiming) != cudaSuccess) p->ev[set] = nullptr;
        }
        p->ev_live[set] = p->ev[set] && cudaEventRecord(p->ev[set], s) == cudaSuccess;
        p->mu.unlock();
    }
};

// Entry points that take a handle launch on the HANDLE's device: the caller's current device is switched for the call and
// restored (SURVEY.md 8b: one process may drive several devices).
struct DevGuard {
    int prev = 0;
    bool switched = false;
    explicit DevGuard(int device) {
        if (cudaGetDevice(&prev) == cudaSuccess && prev != device) switched = cudaSetDevice(device) == cudaSuccess;
    }
    ~DevGuard() { if (switched) cudaSetDevice(prev); }
};

struct dsk_wmh {
    int device = 0, ss = 0, ss_pad = 0, dim = 0;
    float *d_par = nullptr;  // rs_t | lncs_t | betas_t, each [dim][ss_pad]
};

struct dsk_lsh {
    int device = 0;
    LshDev dev{};
    int sw = 1;                    // words per sample: 1 (MinHash), 2 (weighted: (k, t) packed, dev.k / dev.r count words)
    int64_t n_docs = 0;
    uint32_t *removed = nullptr;   // removal bitmap, (cap_docs + 31) / 32 words: allocated by the first dsk_lsh_remove
    bool has_removals = false;     // a dsk_lsh_remove since the last compaction: the walks run their removal-aware kernels
    const uint32_t *walk_bitmap() const { return has_removals ? removed : nullptr; }
    uint64_t changes = 0;          // bumped by every call that changes the index (insert, removal, compaction)
    mutable struct {               // the last dsk_lsh_unique_count, which dsk_lsh_unique_commit must follow
        bool armed;
        const uint32_t *sig;
        const void *ws;
        int64_t n;
        int min_count;
        uint64_t changes;
    } unique{};
};

struct dsk_lsh_ensemble {
    int device = 0;
    EnsembleDev dev{};    // device buffers allocated by dsk_lsh_ensemble_index
    int64_t n_sets = 0;   // 0 until the index is built
};

extern "C" {

int dsk_version(void) { return DSK_VERSION; }

const char *dsk_last_error(void) { return g_err; }

int dsk_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

int dsk_device_info(int device, int *sm_count, int *cc_major, int *cc_minor, size_t *total_mem) {
    DevInfo *d;
    int rc = get_dev(device, &d);
    if (rc) return rc;
    if (sm_count) *sm_count = d->sm_count;
    if (cc_major) *cc_major = d->cc_major;
    if (cc_minor) *cc_minor = d->cc_minor;
    if (total_mem) *total_mem = d->total_mem;
    return DSK_OK;
}

int dsk_perm_create(const uint64_t *h_a, const uint64_t *h_b, int num_perm, int device, dsk_perm **out) {
    if (!h_a || !h_b || !out || num_perm <= 0 || num_perm > 256 * kCounterStride) {
        set_error("dsk_perm_create: bad arguments (num_perm=%d; supported range 1..%d)", num_perm, 256 * kCounterStride);
        return DSK_ERR_INVALID;
    }
    DevInfo *d;
    int rc = get_dev(device, &d);
    if (rc) return rc;
    // arch-specific sm_90a code loads on compute capability 9.0 only
    if (d->cc_major != 9 || d->cc_minor != 0) {
        set_error("device %d is sm_%d%d; this library ships sm_90a code only", device, d->cc_major, d->cc_minor);
        return DSK_ERR_NO_DEVICE;
    }
    dsk_perm *p = new (std::nothrow) dsk_perm();
    if (!p) return DSK_ERR_NOMEM;
    p->device = device;
    p->num_perm = num_perm;
    p->kpad = (num_perm + 255) / 256 * 256;
    p->a.assign(h_a, h_a + num_perm);
    p->b.assign(h_b, h_b + num_perm);
    std::vector<uint32_t> tab((size_t)6 * p->kpad, 0u);
    for (int i = 0; i < num_perm; ++i) {
        tab[i] = (uint32_t)h_a[i];
        tab[p->kpad + i] = (uint32_t)(h_a[i] >> 32);
        tab[2 * p->kpad + i] = (uint32_t)h_b[i];
        tab[3 * p->kpad + i] = (uint32_t)(h_b[i] >> 32);
        if (perm_unsafe_u32(h_a[i], h_b[i])) p->n_unsafe++;
    }
    // Padding slots (a lane's permutations beyond num_perm; their results are never stored) repeat real
    // permutations.  Zeros would make every token of a document tie in such a slot, and a tie sends the whole
    // warp through the two-phase kernel's exact slow path for every document (measured: num_perm=192 ran 5x slower).
    for (int i = num_perm; i < p->kpad; ++i) {
        const int src = i % num_perm;
        for (int q = 0; q < 4; ++q) tab[(size_t)q * p->kpad + i] = tab[(size_t)q * p->kpad + src];
    }
    for (int i = 0; i < p->kpad; ++i) {
        tab[(size_t)4 * p->kpad + i] = tab[(size_t)2 * p->kpad + i] + 7u;
        tab[(size_t)5 * p->kpad + i] = tab[(size_t)2 * p->kpad + i] + 8u;
    }
    int prev = 0;
    cudaGetDevice(&prev);
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaMalloc(&p->d_tab, tab.size() * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMalloc(&p->d_counters, sizeof(unsigned) * kCounterSets * kCounterStride);
    if (e == cudaSuccess) e = cudaMemcpy(p->d_tab, tab.data(), tab.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        if (p->d_tab) cudaFree(p->d_tab);
        if (p->d_counters) cudaFree(p->d_counters);
        delete p;
        return cuda_fail(e, "dsk_perm_create upload");
    }
    *out = p;
    return DSK_OK;
}

int dsk_perm_analyze(const uint64_t *h_a, const uint64_t *h_b, int num_perm, uint8_t *out_unsafe) {
    int n = 0;
    for (int i = 0; i < num_perm; ++i) {
        const bool u = perm_unsafe_u32(h_a[i], h_b[i]);
        if (out_unsafe) out_unsafe[i] = u ? 1 : 0;
        n += u;
    }
    return n;
}

int dsk_perm_info(const dsk_perm *p, int *num_perm, int *n_unsafe, int *device) {
    if (!p) {
        set_error("dsk_perm_info: null handle");
        return DSK_ERR_INVALID;
    }
    if (num_perm) *num_perm = p->num_perm;
    if (n_unsafe) *n_unsafe = p->n_unsafe;
    if (device) *device = p->device;
    return DSK_OK;
}

void dsk_perm_destroy(dsk_perm *p) {
    if (!p) return;
    if (p->d_tab) {
        int prev = 0;
        cudaGetDevice(&prev);
        cudaSetDevice(p->device);
        cudaFree(p->d_tab);
        if (p->d_counters) cudaFree(p->d_counters);
        for (int i = 0; i < kCounterSets; ++i)
            if (p->ev[i]) cudaEventDestroy(p->ev[i]);
        cudaSetDevice(prev);
    }
    delete p;
}

static int pick_mode(const dsk_perm *perm, int token_is_u64, int flags, int *mode) {
    // The two-phase kernel has a variant for every input (BulkParams::gen): the default one needs 32-bit tokens and
    // permutations that cannot reach the conditional subtract of `% (2^61-1)`; the general ones take the subtract in their
    // exact stage (window 8 instead of 7).  DIRECT evaluates r = lo32(x) + top3(x) everywhere and keeps that requirement.
    const bool fast_ok = !token_is_u64 && perm->n_unsafe == 0;
    switch (flags) {
        case DSK_KERNEL_AUTO:
        case DSK_KERNEL_TWO_PHASE: *mode = MODE_TWO_PHASE; return DSK_OK;
        case DSK_KERNEL_DIRECT:
            if (!fast_ok) {
                set_error("DSK_KERNEL_DIRECT is not exact here (token_is_u64=%d, unsafe permutations=%d); use DSK_KERNEL_AUTO / TWO_PHASE / EXACT",
                          token_is_u64, perm->n_unsafe);
                return DSK_ERR_INVALID;
            }
            *mode = MODE_DIRECT;
            return DSK_OK;
        case DSK_KERNEL_EXACT: *mode = MODE_EXACT; return DSK_OK;
        default: set_error("unknown kernel flag %d", flags); return DSK_ERR_INVALID;
    }
}

size_t dsk_minhash_bulk_workspace_size(int64_t n_docs, int64_t n_tokens) {
    (void)n_docs;
    return n_tokens < 0 ? 0 : minhash_sig_workspace_bytes(n_tokens);
}

int dsk_minhash_bulk(const dsk_perm *perm, const void *d_tokens, int token_is_u64, const int64_t *d_offsets,
                     int64_t n_docs, int64_t n_tokens, const void *d_init, int64_t init_stride, int init_is_u64,
                     void *d_out, int out_is_u64, int flags, void *stream) {
    return dsk_minhash_bulk_ws(perm, d_tokens, token_is_u64, d_offsets, n_docs, n_tokens, d_init, init_stride, init_is_u64,
                               d_out, out_is_u64, flags, nullptr, 0, stream);
}

int dsk_minhash_bulk_ws(const dsk_perm *perm, const void *d_tokens, int token_is_u64, const int64_t *d_offsets,
                        int64_t n_docs, int64_t n_tokens, const void *d_init, int64_t init_stride, int init_is_u64,
                        void *d_out, int out_is_u64, int flags, void *d_workspace, size_t workspace_bytes, void *stream) {
    if (!perm || !d_offsets || !d_out || n_docs < 0 || n_tokens < 0 || (n_tokens > 0 && !d_tokens)) {
        set_error("dsk_minhash_bulk: bad arguments");
        return DSK_ERR_INVALID;
    }
    if (d_workspace && (((uintptr_t)d_workspace & 15) != 0 || workspace_bytes < minhash_sig_workspace_bytes(n_tokens))) {
        set_error("dsk_minhash_bulk_ws: workspace must be 16-byte aligned and hold dsk_minhash_bulk_workspace_size() = %zu bytes",
                  minhash_sig_workspace_bytes(n_tokens));
        return DSK_ERR_INVALID;
    }
    if (n_docs == 0) return DSK_OK;
    if (((uintptr_t)d_tokens & 15) != 0) {
        set_error("dsk_minhash_bulk: d_tokens must be 16-byte aligned");
        return DSK_ERR_ALIGN;
    }
    if (((uintptr_t)d_out & 15) != 0 || ((uintptr_t)d_offsets & 7) != 0) {
        set_error("dsk_minhash_bulk: d_out must be 16-byte aligned and d_offsets 8-byte aligned");
        return DSK_ERR_ALIGN;
    }
    int mode;
    int rc = pick_mode(perm, token_is_u64, flags, &mode);
    if (rc) return rc;
    DevInfo *dev;
    rc = get_dev(perm->device, &dev);
    if (rc) return rc;
    BulkParams prm{};
    prm.tokens = d_tokens;
    prm.offsets = d_offsets;
    prm.n_docs = n_docs;
    prm.n_tokens = n_tokens;
    prm.a_lo = perm->d_tab;
    prm.a_hi = perm->d_tab + perm->kpad;
    prm.b_lo = perm->d_tab + 2 * perm->kpad;
    prm.b_hi = perm->d_tab + 3 * perm->kpad;
    prm.b_lo7 = perm->d_tab + 4 * perm->kpad;
    prm.b_lo8 = perm->d_tab + 5 * perm->kpad;
    prm.gen = token_is_u64 ? 2 : (perm->n_unsafe ? 1 : 0);
    prm.k = perm->num_perm;
    prm.init = d_init;
    prm.init_stride = init_stride;
    prm.init_is_u64 = init_is_u64;
    prm.out = d_out;
    prm.out_is_u64 = out_is_u64;
    prm.docs_per_unit = 0;
    prm.n_peers = 0;
    prm.peer_row_offset = 0;
    if (d_workspace && minhash_sig_workspace_bytes(n_tokens) > 0) {   // long documents are cut into pieces on the device
        prm.long_doc_tokens = kLongDocTokensApi;
        prm.piece_shift = kPieceShiftApi;
        prm.piece_hdr = static_cast<unsigned *>(d_workspace);
        prm.pieces = reinterpret_cast<PieceDesc *>(static_cast<char *>(d_workspace) + kPieceHdrBytes);
    }
    DevGuard guard(perm->device);
    CounterLease lease(perm, (cudaStream_t)stream);
    prm.work_counter = lease.ptr;
    DSK_CUDA(launch_minhash_bulk(prm, mode, token_is_u64, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_minhash_bulk_gather(const dsk_perm *perm, const void *d_tokens, int token_is_u64, const int64_t *d_offsets,
                            int64_t n_docs, int64_t n_tokens, void *const *h_peer_out, int n_peers,
                            int64_t row_offset, int out_is_u64, int flags, void *stream) {
    if (!perm || !d_offsets || !h_peer_out || n_peers < 1 || n_peers > 8 || n_docs < 0 || n_tokens < 0 ||
        row_offset < 0 || (n_tokens > 0 && !d_tokens)) {
        set_error("dsk_minhash_bulk_gather: bad arguments (1 <= n_peers <= 8)");
        return DSK_ERR_INVALID;
    }
    if (n_docs == 0) return DSK_OK;
    if (((uintptr_t)d_tokens & 15) != 0) {
        set_error("dsk_minhash_bulk_gather: d_tokens must be 16-byte aligned");
        return DSK_ERR_ALIGN;
    }
    int mode;
    int rc = pick_mode(perm, token_is_u64, flags, &mode);
    if (rc) return rc;
    DevInfo *dev;
    rc = get_dev(perm->device, &dev);
    if (rc) return rc;
    BulkParams prm{};
    prm.tokens = d_tokens;
    prm.offsets = d_offsets;
    prm.n_docs = n_docs;
    prm.n_tokens = n_tokens;
    prm.a_lo = perm->d_tab;
    prm.a_hi = perm->d_tab + perm->kpad;
    prm.b_lo = perm->d_tab + 2 * perm->kpad;
    prm.b_hi = perm->d_tab + 3 * perm->kpad;
    prm.b_lo7 = perm->d_tab + 4 * perm->kpad;
    prm.b_lo8 = perm->d_tab + 5 * perm->kpad;
    prm.gen = token_is_u64 ? 2 : (perm->n_unsafe ? 1 : 0);
    prm.k = perm->num_perm;
    prm.init = nullptr;
    prm.init_stride = 0;
    prm.init_is_u64 = 0;
    prm.out = nullptr;
    prm.out_is_u64 = out_is_u64;
    prm.docs_per_unit = 0;
    prm.n_peers = n_peers;
    prm.peer_row_offset = row_offset;
    for (int i = 0; i < 8; ++i) prm.peer_out[i] = i < n_peers ? h_peer_out[i] : nullptr;
    for (int i = 0; i < n_peers; ++i)
        if (!h_peer_out[i] || ((uintptr_t)h_peer_out[i] & 15) != 0) {
            set_error("dsk_minhash_bulk_gather: peer pointer %d is null or not 16-byte aligned", i);
            return DSK_ERR_ALIGN;
        }
    DevGuard guard(perm->device);
    CounterLease lease(perm, (cudaStream_t)stream);
    prm.work_counter = lease.ptr;
    DSK_CUDA(launch_minhash_bulk(prm, mode, token_is_u64, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_sig_merge_min(const uint32_t *d_x, const uint32_t *d_y, int64_t n_elems, uint32_t *d_out, void *stream) {
    if (n_elems < 0 || (n_elems > 0 && (!d_x || !d_y || !d_out))) {
        set_error("dsk_sig_merge_min: bad arguments");
        return DSK_ERR_INVALID;
    }
    int device = 0;
    DSK_CUDA(cudaGetDevice(&device));
    DevInfo *dev;
    int rc = get_dev(device, &dev);
    if (rc) return rc;
    DSK_CUDA(launch_sig_merge_min(d_x, d_y, n_elems, d_out, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

static int current_dev(DevInfo **dev) {
    int device = 0;
    DSK_CUDA(cudaGetDevice(&device));
    return get_dev(device, dev);
}

int dsk_lean_pack(const void *d_sig, int sig_is_u64, int64_t n, int num_perm, int64_t seed, int big_endian,
                  uint8_t *d_rec, void *stream) {
    if (n < 0 || num_perm <= 0 || (n > 0 && (!d_sig || !d_rec))) {
        set_error("dsk_lean_pack: bad arguments");
        return DSK_ERR_INVALID;
    }
    if (((uintptr_t)d_rec & 3) != 0 || ((uintptr_t)d_sig & 3) != 0) {
        set_error("dsk_lean_pack: buffers must be 4-byte aligned");
        return DSK_ERR_ALIGN;
    }
    DevInfo *dev;
    int rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_lean_pack(d_sig, sig_is_u64, n, num_perm, seed, big_endian, d_rec, dev->sm_count,
                              (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lean_unpack(const uint8_t *d_rec, int64_t n, int num_perm, int64_t seed, int big_endian, void *d_sig,
                    int sig_is_u64, int *d_status, void *stream) {
    if (n < 0 || num_perm <= 0 || !d_status || (n > 0 && (!d_sig || !d_rec))) {
        set_error("dsk_lean_unpack: bad arguments");
        return DSK_ERR_INVALID;
    }
    if (((uintptr_t)d_rec & 3) != 0 || ((uintptr_t)d_sig & 3) != 0) {
        set_error("dsk_lean_unpack: buffers must be 4-byte aligned");
        return DSK_ERR_ALIGN;
    }
    DevInfo *dev;
    int rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_lean_unpack(d_rec, n, num_perm, seed, big_endian, d_sig, sig_is_u64, d_status, dev->sm_count,
                                (cudaStream_t)stream));
    return DSK_OK;
}

static int check_bands(const char *who, int64_t n, int num_perm, int b, int r) {
    if (n < 0 || num_perm <= 0 || b <= 0 || r <= 0 || (int64_t)b * r > num_perm) {
        set_error("%s: need n >= 0, b, r > 0 and b*r <= num_perm (got b=%d r=%d num_perm=%d)", who, b, r, num_perm);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

int dsk_band_keys(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint8_t *d_keys, void *stream) {
    int rc = check_bands("dsk_band_keys", n, num_perm, b, r);
    if (rc) return rc;
    if (n > 0 && (!d_sig || !d_keys)) {
        set_error("dsk_band_keys: null buffer");
        return DSK_ERR_INVALID;
    }
    if (((uintptr_t)d_keys & 7) != 0) {
        set_error("dsk_band_keys: d_keys must be 8-byte aligned");
        return DSK_ERR_ALIGN;
    }
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_band_keys_be(d_sig, n, num_perm, b, r, d_keys, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_band_fingerprints(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint64_t *d_fp, void *stream) {
    int rc = check_bands("dsk_band_fingerprints", n, num_perm, b, r);
    if (rc) return rc;
    if (n > 0 && (!d_sig || !d_fp)) {
        set_error("dsk_band_fingerprints: null buffer");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_band_fingerprints(d_sig, n, num_perm, b, r, d_fp, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_band_sums(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint64_t *d_keys, void *stream) {
    int rc = check_bands("dsk_band_sums", n, num_perm, b, r);
    if (rc) return rc;
    if (n > 0 && (!d_sig || !d_keys)) {
        set_error("dsk_band_sums: null buffer");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_band_sums(d_sig, n, num_perm, b, r, d_keys, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

static int check_bloom(const char *who, const void *d_bits, uint64_t words_per_table, uint64_t n_bits, int n_hashes) {
    if (!d_bits || n_bits == 0 || n_hashes <= 0 || n_hashes > 64 || words_per_table * 32 < n_bits ||
        ((uintptr_t)d_bits & 3) != 0) {
        set_error("%s: need a 4-byte aligned bit array, 0 < n_hashes <= 64 and words_per_table * 32 >= n_bits > 0", who);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

int dsk_bloom_insert(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint32_t *d_bits,
                     uint64_t words_per_table, uint64_t n_bits, int n_hashes, void *stream) {
    int rc = check_bands("dsk_bloom_insert", n, num_perm, b, r);
    if (rc) return rc;
    rc = check_bloom("dsk_bloom_insert", d_bits, words_per_table, n_bits, n_hashes);
    if (rc) return rc;
    if (n > 0 && !d_sig) {
        set_error("dsk_bloom_insert: null signature matrix");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_bloom_insert(d_sig, n, num_perm, b, r, d_bits, words_per_table, n_bits, n_hashes, dev->sm_count,
                                 (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_bloom_query(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, const uint32_t *d_bits,
                    uint64_t words_per_table, uint64_t n_bits, int n_hashes, uint8_t *d_hit, void *stream) {
    int rc = check_bands("dsk_bloom_query", n, num_perm, b, r);
    if (rc) return rc;
    rc = check_bloom("dsk_bloom_query", d_bits, words_per_table, n_bits, n_hashes);
    if (rc) return rc;
    if (n > 0 && (!d_sig || !d_hit)) {
        set_error("dsk_bloom_query: null buffer");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_bloom_query(d_sig, n, num_perm, b, r, d_bits, words_per_table, n_bits, n_hashes, d_hit, dev->sm_count,
                                (cudaStream_t)stream));
    return DSK_OK;
}

// the n * b * n_hashes probe entries of a batch are numbered in int32: at most kBloomUniqueMaxEntries (checked without
// overflow: b and n_hashes are positive ints, so b * n_hashes fits int64)
static bool bloom_unique_fits(int64_t n, int b, int n_hashes) {
    return n <= kBloomUniqueMaxEntries / ((int64_t)b * n_hashes);
}

size_t dsk_bloom_unique_workspace_size(int64_t n, int num_perm, int b, int r, int n_hashes) {
    if (n <= 0 || num_perm <= 0 || b <= 0 || r <= 0 || (int64_t)b * r > num_perm || n_hashes <= 0 || n_hashes > 64 ||
        !bloom_unique_fits(n, b, n_hashes))
        return 0;
    return bloom_unique_workspace_bytes(n, b, n_hashes);
}

int dsk_bloom_unique(const uint32_t *d_sig, int64_t n, int num_perm, int b, int r, uint32_t *d_bits, uint64_t words_per_table,
                     uint64_t n_bits, int n_hashes, void *d_ws, size_t ws_bytes, uint8_t *d_keep, void *stream) {
    const char *who = "dsk_bloom_unique";
    int rc = check_bands(who, n, num_perm, b, r);
    if (rc) return rc;
    rc = check_bloom(who, d_bits, words_per_table, n_bits, n_hashes);
    if (rc) return rc;
    if (n_bits > (UINT64_MAX - 1) / (uint64_t)b) {   // the batch table's key band * n_bits + pos must not reach the empty key
        set_error("%s: b * n_bits must be below 2^64 (got b=%d n_bits=%llu)", who, b, (unsigned long long)n_bits);
        return DSK_ERR_INVALID;
    }
    if (n == 0) return DSK_OK;
    if (!d_sig || !d_ws || !d_keep) {
        set_error("%s: null buffer", who);
        return DSK_ERR_INVALID;
    }
    if (((uintptr_t)d_sig & 3) != 0 || ((uintptr_t)d_ws & 15) != 0) {
        set_error("%s: d_sig must be 4-byte and d_ws 16-byte aligned", who);
        return DSK_ERR_ALIGN;
    }
    if (!bloom_unique_fits(n, b, n_hashes)) {
        set_error("%s: n * b * n_hashes must be at most 2^30 (got n=%lld b=%d n_hashes=%d); split the batch", who,
                  (long long)n, b, n_hashes);
        return DSK_ERR_INVALID;
    }
    const size_t need = bloom_unique_workspace_bytes(n, b, n_hashes);
    if (ws_bytes < need) {
        set_error("%s: the workspace must hold dsk_bloom_unique_workspace_size() = %zu bytes (got %zu)", who, need, ws_bytes);
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(bloom_unique(d_sig, n, num_perm, b, r, d_bits, words_per_table, n_bits, n_hashes, d_ws, d_keep, dev->sm_count,
                          (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_wmh_create(const float *h_rs, const float *h_ln_cs, const float *h_betas, int sample_size, int dim, int device,
                   dsk_wmh **out) {
    if (!h_rs || !h_ln_cs || !h_betas || !out || sample_size <= 0 || dim <= 0) {
        set_error("dsk_wmh_create: bad arguments");
        return DSK_ERR_INVALID;
    }
    DevInfo *d;
    int rc = get_dev(device, &d);
    if (rc) return rc;
    dsk_wmh *g = new (std::nothrow) dsk_wmh();
    if (!g) return DSK_ERR_NOMEM;
    g->device = device; g->ss = sample_size; g->dim = dim; g->ss_pad = (sample_size + 31) / 32 * 32;
    const size_t plane = (size_t)dim * g->ss_pad, src_elems = (size_t)sample_size * dim;
    int prev = 0;
    cudaGetDevice(&prev);
    float *tmp = nullptr;
    cudaError_t e = cudaSetDevice(device);
    if (e == cudaSuccess) e = cudaMalloc(&g->d_par, 3 * plane * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&tmp, src_elems * sizeof(float));
    const float *srcs[3] = {h_rs, h_ln_cs, h_betas};
    for (int i = 0; i < 3 && e == cudaSuccess; ++i) {
        e = cudaMemcpy(tmp, srcs[i], src_elems * sizeof(float), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = launch_wmh_transpose(tmp, sample_size, dim, g->ss_pad, g->d_par + i * plane, 0);
        if (e == cudaSuccess) e = cudaStreamSynchronize(0);
    }
    if (tmp) cudaFree(tmp);
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        if (g->d_par) cudaFree(g->d_par);
        delete g;
        return cuda_fail(e, "dsk_wmh_create");
    }
    *out = g;
    return DSK_OK;
}

void dsk_wmh_destroy(dsk_wmh *g) {
    if (!g) return;
    if (g->d_par) {
        int prev = 0;
        cudaGetDevice(&prev);
        cudaSetDevice(g->device);
        cudaFree(g->d_par);
        cudaSetDevice(prev);
    }
    delete g;
}

int dsk_wmh_minhash(const dsk_wmh *g, const float *d_v, int64_t n, int64_t *d_out, int32_t *d_status, int flags,
                    void *stream) {
    if (!g || n < 0 || (flags & ~(DSK_WMH_MINHASH_MANY | DSK_WMH_INPUT_LOG)) != 0 || (n > 0 && (!d_v || !d_out || !d_status))) {
        set_error("dsk_wmh_minhash: bad arguments");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = get_dev(g->device, &dev);
    if (rc) return rc;
    const size_t plane = (size_t)g->dim * g->ss_pad;
    DevGuard guard(g->device);
    DSK_CUDA(launch_wmh(g->d_par, g->d_par + plane, g->d_par + 2 * plane, g->ss, g->ss_pad, g->dim, d_v, n, d_out,
                        d_status, (flags & DSK_WMH_MINHASH_MANY) != 0, (flags & DSK_WMH_INPUT_LOG) != 0, dev->sm_count,
                        (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_wmh_minhash_csr(const dsk_wmh *g, const int64_t *d_indptr, const int32_t *d_indices, const float *d_vals, int64_t n,
                        int64_t *d_out, int32_t *d_status, int flags, void *stream) {
    if (!g || n < 0 || (flags & ~(DSK_WMH_MINHASH_MANY | DSK_WMH_INPUT_LOG)) != 0 ||
        (n > 0 && (!d_indptr || !d_indices || !d_vals || !d_out || !d_status))) {
        set_error("dsk_wmh_minhash_csr: bad arguments");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = get_dev(g->device, &dev);
    if (rc) return rc;
    const size_t plane = (size_t)g->dim * g->ss_pad;
    DevGuard guard(g->device);
    DSK_CUDA(launch_wmh_csr(g->d_par, g->d_par + plane, g->d_par + 2 * plane, g->ss, g->ss_pad, g->dim, d_indptr, d_indices,
                            d_vals, n, d_out, d_status, (flags & DSK_WMH_MINHASH_MANY) != 0,
                            (flags & DSK_WMH_INPUT_LOG) != 0, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

// num_perm samples of sw words each; b and r count samples
static int lsh_create(const char *who, int num_perm, int sw, int b, int r, int64_t capacity_docs, int device, dsk_lsh **out) {
    int rc = check_bands(who, capacity_docs, num_perm, b, r);
    if (rc) return rc;
    if (!out || capacity_docs <= 0 || capacity_docs >= (1ll << 31)) {
        set_error("%s: capacity_docs must be in [1, 2^31)", who);
        return DSK_ERR_INVALID;
    }
    if (num_perm > INT32_MAX / sw) {
        set_error("%s: num_perm must be at most %d (got %d)", who, INT32_MAX / sw, num_perm);
        return DSK_ERR_INVALID;
    }
    DevInfo *d;
    rc = get_dev(device, &d);
    if (rc) return rc;
    dsk_lsh *ix = new (std::nothrow) dsk_lsh();
    if (!ix) return DSK_ERR_NOMEM;
    ix->device = device;
    ix->sw = sw;
    num_perm *= sw;
    r *= sw;
    LshDev &v = ix->dev;
    v.k = num_perm; v.b = b; v.r = r; v.cap_docs = capacity_docs;
    v.cap_slots = 1024;
    while (v.cap_slots < 2 * capacity_docs) v.cap_slots <<= 1;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaError_t e = cudaSetDevice(device);
    const size_t slots = (size_t)b * v.cap_slots;
    if (e == cudaSuccess) e = cudaMalloc(&v.sig, (size_t)capacity_docs * num_perm * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMalloc(&v.slots, slots * 2 * sizeof(uint64_t));
    if (e == cudaSuccess) e = cudaMalloc(&v.next, (size_t)b * capacity_docs * sizeof(int32_t));
    if (e == cudaSuccess) e = cudaMemset(v.slots, 0xFF, slots * 2 * sizeof(uint64_t));   // empty key, head = -1
    cudaSetDevice(prev);
    if (e != cudaSuccess) {
        int rc2 = cuda_fail(e, who);
        dsk_lsh_destroy(ix);
        return rc2;
    }
    *out = ix;
    return DSK_OK;
}

int dsk_lsh_create(int num_perm, int b, int r, int64_t capacity_docs, int device, dsk_lsh **out) {
    return lsh_create("dsk_lsh_create", num_perm, 1, b, r, capacity_docs, device, out);
}

int dsk_lsh_create_weighted(int sample_size, int b, int r, int64_t capacity_docs, int device, dsk_lsh **out) {
    return lsh_create("dsk_lsh_create_weighted", sample_size, 2, b, r, capacity_docs, device, out);
}

void dsk_lsh_destroy(dsk_lsh *ix) {
    if (!ix) return;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(ix->device);
    if (ix->dev.sig) cudaFree(ix->dev.sig);
    if (ix->dev.slots) cudaFree(ix->dev.slots);
    if (ix->dev.next) cudaFree(ix->dev.next);
    if (ix->removed) cudaFree(ix->removed);
    cudaSetDevice(prev);
    delete ix;
}

int dsk_lsh_size(const dsk_lsh *ix, int64_t *n_docs, int64_t *capacity_docs) {
    if (!ix) {
        set_error("dsk_lsh_size: null handle");
        return DSK_ERR_INVALID;
    }
    if (n_docs) *n_docs = ix->n_docs;
    if (capacity_docs) *capacity_docs = ix->dev.cap_docs;
    return DSK_OK;
}

int dsk_lsh_insert(dsk_lsh *ix, const uint32_t *d_sig, int64_t n, void *stream) {
    if (!ix || n < 0 || (n > 0 && !d_sig)) {
        set_error("dsk_lsh_insert: bad arguments");
        return DSK_ERR_INVALID;
    }
    if (ix->n_docs + n > ix->dev.cap_docs) {
        set_error("dsk_lsh_insert: capacity exceeded (%lld + %lld > %lld)", (long long)ix->n_docs, (long long)n,
                  (long long)ix->dev.cap_docs);
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(launch_lsh_insert(ix->dev, d_sig, ix->n_docs, n, dev->sm_count, (cudaStream_t)stream));
    ix->n_docs += n;
    ++ix->changes;
    return DSK_OK;
}

int dsk_lsh_insert_tokens(dsk_lsh *ix, const dsk_perm *perm, const void *d_tokens, int token_is_u64,
                          const int64_t *d_offsets, int64_t n_docs, int64_t n_tokens, void *stream) {
    if (!ix || !perm || !d_offsets || n_docs < 0 || n_tokens < 0 || (n_tokens > 0 && !d_tokens)) {
        set_error("dsk_lsh_insert_tokens: bad arguments");
        return DSK_ERR_INVALID;
    }
    if (ix->sw != 1) {
        set_error("dsk_lsh_insert_tokens: the index holds weighted MinHash rows; tokens give MinHash rows");
        return DSK_ERR_INVALID;
    }
    if (perm->num_perm != ix->dev.k || perm->device != ix->device) {
        set_error("dsk_lsh_insert_tokens: the permutation handle has num_perm=%d on device %d, the index num_perm=%d on device %d",
                  perm->num_perm, perm->device, ix->dev.k, ix->device);
        return DSK_ERR_INVALID;
    }
    if (ix->n_docs + n_docs > ix->dev.cap_docs) {
        set_error("dsk_lsh_insert_tokens: capacity exceeded (%lld + %lld > %lld)", (long long)ix->n_docs, (long long)n_docs,
                  (long long)ix->dev.cap_docs);
        return DSK_ERR_INVALID;
    }
    if (n_docs == 0) return DSK_OK;
    if (((uintptr_t)d_tokens & 15) != 0 || ((uintptr_t)d_offsets & 7) != 0) {
        set_error("dsk_lsh_insert_tokens: d_tokens must be 16-byte aligned and d_offsets 8-byte aligned");
        return DSK_ERR_ALIGN;
    }
    DevInfo *dev;
    int rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    uint32_t *rows = ix->dev.sig + ix->n_docs * ix->dev.k;   // the new documents' rows in the index's own storage
    BulkParams prm{};
    prm.tokens = d_tokens;
    prm.offsets = d_offsets;
    prm.n_docs = n_docs;
    prm.n_tokens = n_tokens;
    prm.a_lo = perm->d_tab;
    prm.a_hi = perm->d_tab + perm->kpad;
    prm.b_lo = perm->d_tab + 2 * perm->kpad;
    prm.b_hi = perm->d_tab + 3 * perm->kpad;
    prm.b_lo7 = perm->d_tab + 4 * perm->kpad;
    prm.b_lo8 = perm->d_tab + 5 * perm->kpad;
    prm.gen = token_is_u64 ? 2 : (perm->n_unsafe ? 1 : 0);
    prm.k = perm->num_perm;
    prm.out = rows;
    prm.out_is_u64 = 0;
    const bool fused = prm.gen == 0 && prm.k <= 256 && (((uintptr_t)rows & 15) == 0);
    DevGuard guard(ix->device);
    {
        CounterLease lease(perm, (cudaStream_t)stream);
        prm.work_counter = lease.ptr;
        if (fused) {
            prm.lsh_slots = ix->dev.slots;
            prm.lsh_next = ix->dev.next;
            prm.lsh_cap_slots = ix->dev.cap_slots;
            prm.lsh_doc0 = ix->n_docs;
            prm.lsh_b = ix->dev.b;
            prm.lsh_r = ix->dev.r;
        }
        DSK_CUDA(launch_minhash_bulk(prm, MODE_TWO_PHASE, token_is_u64, dev->sm_count, (cudaStream_t)stream));
    }
    if (!fused)   // rows are in place already: the insert kernel's copy of them is a self-copy
        DSK_CUDA(launch_lsh_insert(ix->dev, rows, ix->n_docs, n_docs, dev->sm_count, (cudaStream_t)stream));
    ix->n_docs += n_docs;
    ++ix->changes;
    return DSK_OK;
}

int dsk_lsh_query_count(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int64_t *d_counts, void *stream) {
    if (!ix || nq < 0 || (nq > 0 && (!d_qsig || !d_counts))) {
        set_error("dsk_lsh_query_count: bad arguments");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(launch_lsh_query(ix->dev, d_qsig, nq, ix->n_docs, d_counts, nullptr, nullptr, 0, ix->walk_bitmap(), dev->sm_count,
                              (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lsh_query_fill(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, const int64_t *d_ptr, int32_t *d_idx,
                       void *stream) {
    if (!ix || nq < 0 || (nq > 0 && (!d_qsig || !d_ptr))) {
        set_error("dsk_lsh_query_fill: bad arguments");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(launch_lsh_query(ix->dev, d_qsig, nq, ix->n_docs, nullptr, d_ptr, d_idx, 1, ix->walk_bitmap(), dev->sm_count,
                              (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_exclusive_scan(const int64_t *d_in, int64_t n, int64_t *d_out, int64_t *d_scratch, void *stream) {
    if (n < 0 || !d_out || (n > 0 && (!d_in || !d_scratch))) {
        set_error("dsk_exclusive_scan: bad arguments");
        return DSK_ERR_INVALID;
    }
    DSK_CUDA(launch_exclusive_scan(d_in, n, d_out, d_scratch, (cudaStream_t)stream));
    return DSK_OK;
}

static int check_self_join(const char *who, const dsk_lsh *ix, int min_count) {
    if (!ix) {
        set_error("%s: null handle", who);
        return DSK_ERR_INVALID;
    }
    const int samples = ix->dev.k / ix->sw;   // eq counts samples
    if (min_count < 0 || min_count > samples) {
        set_error("%s: min_count must be in [0, %s=%d] (got %d)", who, ix->sw == 1 ? "num_perm" : "sample_size", samples,
                  min_count);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

int dsk_lsh_pairs_count(const dsk_lsh *ix, int min_count, int64_t *d_counts, void *stream) {
    int rc = check_self_join("dsk_lsh_pairs_count", ix, min_count);
    if (rc) return rc;
    if (ix->n_docs > 0 && !d_counts) {
        set_error("dsk_lsh_pairs_count: null buffer");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(launch_lsh_pairs(ix->dev, ix->sw, ix->n_docs, min_count, d_counts, nullptr, nullptr, nullptr, ix->walk_bitmap(), dev->sm_count,
                              (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lsh_pairs_fill(const dsk_lsh *ix, int min_count, const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq,
                       void *stream) {
    int rc = check_self_join("dsk_lsh_pairs_fill", ix, min_count);
    if (rc) return rc;
    if (ix->n_docs > 0 && (!d_ptr || !d_idx || !d_eq)) {
        set_error("dsk_lsh_pairs_fill: null buffer");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(launch_lsh_pairs(ix->dev, ix->sw, ix->n_docs, min_count, nullptr, d_ptr, d_idx, d_eq, ix->walk_bitmap(), dev->sm_count,
                              (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lsh_clusters(const dsk_lsh *ix, int min_count, int32_t *d_labels, void *stream) {
    int rc = check_self_join("dsk_lsh_clusters", ix, min_count);
    if (rc) return rc;
    if (ix->n_docs > 0 && !d_labels) {
        set_error("dsk_lsh_clusters: null buffer");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(launch_lsh_clusters(ix->dev, ix->sw, ix->n_docs, min_count, d_labels, ix->walk_bitmap(), dev->sm_count,
                                 (cudaStream_t)stream));
    return DSK_OK;
}

// handle, min_count in [0, num_perm], nq >= 0 and, when nq > 0, the query matrix and every output buffer
static int check_query_pairs(const char *who, const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count,
                             bool bufs) {
    int rc = check_self_join(who, ix, min_count);
    if (rc) return rc;
    if (nq < 0) {
        set_error("%s: nq must be >= 0 (got %lld)", who, (long long)nq);
        return DSK_ERR_INVALID;
    }
    if (nq > 0 && (!d_qsig || !bufs)) {
        set_error("%s: null buffer", who);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

static int run_query_pairs(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count, int64_t *d_counts,
                           const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq, void *stream) {
    if (nq == 0) return DSK_OK;
    DevInfo *dev;
    int rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(launch_lsh_query_pairs(ix->dev, ix->sw, d_qsig, nq, ix->n_docs, min_count, d_counts, d_ptr, d_idx, d_eq,
                                    ix->walk_bitmap(), dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lsh_query_jaccard_count(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count, int64_t *d_counts,
                                void *stream) {
    int rc = check_query_pairs("dsk_lsh_query_jaccard_count", ix, d_qsig, nq, min_count, d_counts != nullptr);
    if (rc) return rc;
    return run_query_pairs(ix, d_qsig, nq, min_count, d_counts, nullptr, nullptr, nullptr, stream);
}

int dsk_lsh_query_jaccard_fill(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count, const int64_t *d_ptr,
                               int32_t *d_idx, int32_t *d_eq, void *stream) {
    int rc = check_query_pairs("dsk_lsh_query_jaccard_fill", ix, d_qsig, nq, min_count, d_ptr && d_idx && d_eq);
    if (rc) return rc;
    return run_query_pairs(ix, d_qsig, nq, min_count, nullptr, d_ptr, d_idx, d_eq, stream);
}

int dsk_lsh_query_best(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count, int32_t *d_idx, int32_t *d_eq,
                       void *stream) {
    int rc = check_query_pairs("dsk_lsh_query_best", ix, d_qsig, nq, min_count, d_idx && d_eq);
    if (rc) return rc;
    return run_query_pairs(ix, d_qsig, nq, min_count, nullptr, nullptr, d_idx, d_eq, stream);
}

static int check_topk(const char *who, int k) {
    if (k < 1 || k > 32) {
        set_error("%s: k must be in [1, 32] (got %d)", who, k);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

// the first k kept candidates of nq query rows (qsig), or of every document's own row (qsig == nullptr, nq = n_docs)
static int run_topk(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count, int k, int32_t *d_idx,
                    int32_t *d_eq, void *stream) {
    if (nq == 0) return DSK_OK;
    DevInfo *dev;
    int rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(launch_lsh_topk(ix->dev, ix->sw, d_qsig, nq, ix->n_docs, min_count, k, d_idx, d_eq, ix->walk_bitmap(),
                             dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lsh_query_topk(const dsk_lsh *ix, const uint32_t *d_qsig, int64_t nq, int min_count, int k, int32_t *d_idx,
                       int32_t *d_eq, void *stream) {
    int rc = check_query_pairs("dsk_lsh_query_topk", ix, d_qsig, nq, min_count, d_idx && d_eq);
    if (!rc) rc = check_topk("dsk_lsh_query_topk", k);
    if (rc) return rc;
    return run_topk(ix, d_qsig, nq, min_count, k, d_idx, d_eq, stream);
}

int dsk_lsh_neighbors(const dsk_lsh *ix, int min_count, int k, int32_t *d_idx, int32_t *d_eq, void *stream) {
    int rc = check_self_join("dsk_lsh_neighbors", ix, min_count);
    if (!rc) rc = check_topk("dsk_lsh_neighbors", k);
    if (rc) return rc;
    if (ix->n_docs > 0 && (!d_idx || !d_eq)) {
        set_error("dsk_lsh_neighbors: null buffer");
        return DSK_ERR_INVALID;
    }
    return run_topk(ix, nullptr, ix->n_docs, min_count, k, d_idx, d_eq, stream);
}

static int check_ids(const char *who, const dsk_lsh *ix, const void *d_docs, int64_t n, const void *d_out) {
    if (!ix) {
        set_error("%s: null handle", who);
        return DSK_ERR_INVALID;
    }
    if (n < 0) {
        set_error("%s: n must be >= 0 (got %lld)", who, (long long)n);
        return DSK_ERR_INVALID;
    }
    if (n > 0 && (!d_docs || !d_out)) {
        set_error("%s: null buffer", who);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

int dsk_lsh_remove(dsk_lsh *ix, const int32_t *d_docs, int64_t n, int64_t *d_status, void *stream) {
    int rc = check_ids("dsk_lsh_remove", ix, d_docs, n, d_status);
    if (rc || n == 0) return rc;
    DevInfo *dev;
    rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    const size_t words = (size_t)(ix->dev.cap_docs + 31) / 32;
    if (!ix->removed) {   // an index that never removes anything keeps the memory dsk_lsh_create gave it
        uint32_t *bits = nullptr;
        DSK_CUDA(cudaMalloc(&bits, words * sizeof(uint32_t)));
        const cudaError_t e = cudaMemsetAsync(bits, 0, words * sizeof(uint32_t), (cudaStream_t)stream);
        if (e != cudaSuccess) {
            cudaFree(bits);
            return cuda_fail(e, "dsk_lsh_remove bitmap");
        }
        ix->removed = bits;
    }
    ix->has_removals = true;
    ++ix->changes;
    DSK_CUDA(launch_lsh_remove(ix->removed, d_docs, n, ix->n_docs, d_status, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lsh_alive(const dsk_lsh *ix, const int32_t *d_docs, int64_t n, uint8_t *d_out, void *stream) {
    int rc = check_ids("dsk_lsh_alive", ix, d_docs, n, d_out);
    if (rc || n == 0) return rc;
    DevInfo *dev;
    rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(launch_lsh_alive(ix->walk_bitmap(), d_docs, n, ix->n_docs, d_out, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

size_t dsk_lsh_compact_workspace_size(const dsk_lsh *ix) {
    return ix ? lsh_compact_workspace_bytes(ix->n_docs, ix->dev.k) : 0;
}

int dsk_lsh_compact(dsk_lsh *ix, int32_t *d_remap, void *d_ws, size_t ws_bytes, void *stream) {
    if (!ix) {
        set_error("dsk_lsh_compact: null handle");
        return DSK_ERR_INVALID;
    }
    const int64_t n = ix->n_docs;
    const size_t need = lsh_compact_workspace_bytes(n, ix->dev.k);
    if (n > 0 && (!d_remap || !d_ws)) {
        set_error("dsk_lsh_compact: null buffer");
        return DSK_ERR_INVALID;
    }
    if (n > 0 && (((uintptr_t)d_ws & 15) != 0 || ws_bytes < need)) {
        set_error("dsk_lsh_compact: the workspace must be 16-byte aligned and hold dsk_lsh_compact_workspace_size() = %zu bytes (got %zu)",
                  need, ws_bytes);
        return DSK_ERR_INVALID;
    }
    if (n == 0) {
        ix->has_removals = false;
        return DSK_OK;
    }
    DevInfo *dev;
    int rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    const cudaStream_t s = (cudaStream_t)stream;
    if (!ix->has_removals) {   // nothing removed: the identity remap, no synchronisation, no rebuild
        DSK_CUDA(launch_lsh_identity(d_remap, n, dev->sm_count, s));
        return DSK_OK;
    }
    int64_t m = n;
    DSK_CUDA(lsh_compact(ix->dev, ix->removed, n, d_remap, d_ws, &m, dev->sm_count, s));
    DSK_CUDA(cudaMemsetAsync(ix->removed, 0, (size_t)(n + 31) / 32 * sizeof(uint32_t), s));
    ix->has_removals = false;
    ix->n_docs = m;
    ++ix->changes;
    return DSK_OK;
}

// ---- insert_unique: count (batch table, stage A, earlier partners) -> dsk_exclusive_scan -> commit ----------------------
size_t dsk_lsh_unique_workspace_size(const dsk_lsh *ix, int64_t n) {
    return ix && n > 0 ? lsh_unique_workspace_bytes(ix->dev, n) : 0;
}

// handle, n >= 0, min_count in [0, num_perm], and for n > 0 the rows, a 16-byte aligned workspace of the size
// dsk_lsh_unique_workspace_size gives and every buffer (bufs)
static int check_unique(const char *who, const dsk_lsh *ix, const uint32_t *d_sig, int64_t n, int min_count, const void *d_ws,
                        size_t ws_bytes, bool bufs) {
    int rc = check_self_join(who, ix, min_count);
    if (rc) return rc;
    if (n < 0) {
        set_error("%s: n must be >= 0 (got %lld)", who, (long long)n);
        return DSK_ERR_INVALID;
    }
    if (n == 0) return DSK_OK;
    if (!d_sig || !d_ws || !bufs) {
        set_error("%s: null buffer", who);
        return DSK_ERR_INVALID;
    }
    const size_t need = lsh_unique_workspace_bytes(ix->dev, n);
    if (((uintptr_t)d_ws & 15) != 0 || ws_bytes < need) {
        set_error("%s: the workspace must be 16-byte aligned and hold dsk_lsh_unique_workspace_size() = %zu bytes (got %zu)",
                  who, need, ws_bytes);
        return DSK_ERR_INVALID;
    }
    if (ix->sw == 2 && ((uintptr_t)d_sig & 7) != 0) {   // the batch walk reads a sample of these rows with one 8-byte load
        set_error("%s: d_sig must be 8-byte aligned for a weighted index", who);
        return DSK_ERR_ALIGN;
    }
    return DSK_OK;
}

int dsk_lsh_unique_count(const dsk_lsh *ix, const uint32_t *d_sig, int64_t n, int min_count, void *d_ws, size_t ws_bytes,
                         int64_t *d_counts, void *stream) {
    int rc = check_unique("dsk_lsh_unique_count", ix, d_sig, n, min_count, d_ws, ws_bytes, d_counts != nullptr);
    if (rc) return rc;
    ix->unique.armed = false;
    if (n == 0) return DSK_OK;
    DevInfo *dev;
    rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    DSK_CUDA(lsh_unique_count(ix->dev, ix->sw, ix->n_docs, d_sig, n, min_count, d_ws, d_counts, ix->walk_bitmap(), dev->sm_count,
                              (cudaStream_t)stream));
    ix->unique = {true, d_sig, d_ws, n, min_count, ix->changes};
    return DSK_OK;
}

int dsk_lsh_unique_commit(dsk_lsh *ix, const uint32_t *d_sig, int64_t n, int min_count, void *d_ws, size_t ws_bytes,
                          const int64_t *d_ptr, int32_t *d_pidx, int32_t *d_peq, uint8_t *d_kept, int32_t *d_match,
                          int32_t *d_eq, int64_t *h_inserted, void *stream) {
    int rc = check_unique("dsk_lsh_unique_commit", ix, d_sig, n, min_count, d_ws, ws_bytes,
                          d_ptr && d_pidx && d_peq && d_kept && d_match && d_eq && h_inserted);
    if (rc) return rc;
    if (n == 0) {
        if (h_inserted) *h_inserted = 0;
        return DSK_OK;
    }
    const auto &u = ix->unique;
    if (!u.armed || u.sig != d_sig || u.ws != d_ws || u.n != n || u.min_count != min_count || u.changes != ix->changes) {
        set_error("dsk_lsh_unique_commit: must follow dsk_lsh_unique_count of the same d_sig, n, min_count and d_ws, with no "
                  "change of the index in between");
        return DSK_ERR_INVALID;
    }
    ix->unique.armed = false;
    DevInfo *dev;
    rc = get_dev(ix->device, &dev);
    if (rc) return rc;
    DevGuard guard(ix->device);
    const cudaStream_t s = (cudaStream_t)stream;
    int64_t m = 0;
    DSK_CUDA(lsh_unique_resolve(ix->dev, ix->sw, ix->n_docs, d_sig, n, min_count, d_ws, d_ptr, d_pidx, d_peq, d_kept, d_match, d_eq,
                                &m, dev->sm_count, s));
    *h_inserted = 0;
    if (ix->n_docs + m > ix->dev.cap_docs) {
        set_error("dsk_lsh_unique_commit: capacity exceeded (%lld + %lld kept > %lld); the index is unchanged",
                  (long long)ix->n_docs, (long long)m, (long long)ix->dev.cap_docs);
        return DSK_ERR_INVALID;
    }
    DSK_CUDA(lsh_unique_insert(ix->dev, ix->n_docs, d_sig, n, m, d_ws, dev->sm_count, s));
    ix->n_docs += m;
    ++ix->changes;
    *h_inserted = m;
    return DSK_OK;
}

// ---- MinHashLSHEnsemble ------------------------------------------------------------------------------------------------
static int64_t ensemble_cap_slots(int64_t n) {
    int64_t c = 2;
    while (c < 2 * n) c <<= 1;
    return c;
}

static void ensemble_free(dsk_lsh_ensemble *e);

size_t dsk_lsh_ensemble_index_bytes(const dsk_lsh_ensemble *e, int64_t n_sets) {
    if (!e || n_sets <= 0) return 0;
    const EnsembleDev &en = e->dev;
    size_t bytes = (size_t)n_sets * en.tab[0].k * 4 + (size_t)n_sets * 4 + (size_t)(en.num_part + 1) * 8;
    for (int t = 0; t < en.n_tabs; ++t)
        bytes += (size_t)en.tab[t].b * ((size_t)ensemble_cap_slots(n_sets) * 16 + (size_t)n_sets * 4);
    return bytes;
}

int dsk_lsh_ensemble_create(int num_perm, int num_part, const int32_t *h_b, const int32_t *h_r, int n_params, int device,
                            dsk_lsh_ensemble **out) {
    if (!out || !h_b || !h_r || num_perm < 2 || num_part < 1 || n_params < 1 || n_params > kEnsembleMaxParams) {
        set_error("dsk_lsh_ensemble_create: need num_perm >= 2, num_part >= 1, 1 <= n_params <= %d and the (b, r) table",
                  kEnsembleMaxParams);
        return DSK_ERR_INVALID;
    }
    for (int i = 0; i < n_params; ++i) {
        if (h_b[i] < 1 || h_r[i] < 1 || (int64_t)h_b[i] * h_r[i] > num_perm) {
            set_error("dsk_lsh_ensemble_create: row %d of the (b, r) table needs b, r >= 1 and b*r <= num_perm (got b=%d r=%d "
                      "num_perm=%d)", i, h_b[i], h_r[i], num_perm);
            return DSK_ERR_INVALID;
        }
    }
    DevInfo *d;
    int rc = get_dev(device, &d);
    if (rc) return rc;
    dsk_lsh_ensemble *e = new (std::nothrow) dsk_lsh_ensemble();
    if (!e) return DSK_ERR_NOMEM;
    e->device = device;
    EnsembleDev &en = e->dev;
    en.num_part = num_part;
    en.n_params = n_params;
    for (int i = 0; i < n_params; ++i) {   // one table set per distinct r, in order of first appearance
        int t = 0;
        while (t < en.n_tabs && en.tab[t].r != h_r[i]) ++t;
        if (t == en.n_tabs) {
            LshDev &v = en.tab[en.n_tabs++];
            v.k = num_perm;
            v.r = h_r[i];
            v.b = num_perm / h_r[i];
        }
        en.pb[i] = h_b[i];
        en.pt[i] = t;
    }
    for (int t = en.n_tabs; t < kEnsembleMaxParams; ++t) en.tab[t].k = num_perm;
    *out = e;
    return DSK_OK;
}

static void ensemble_free(dsk_lsh_ensemble *e) {
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(e->device);
    EnsembleDev &en = e->dev;
    if (en.tab[0].sig) cudaFree(en.tab[0].sig);
    if (en.map) cudaFree(en.map);
    if (en.part_start) cudaFree(en.part_start);
    for (int t = 0; t < en.n_tabs; ++t) {
        if (en.tab[t].slots) cudaFree(en.tab[t].slots);
        if (en.tab[t].next) cudaFree(en.tab[t].next);
        en.tab[t].sig = nullptr;
        en.tab[t].slots = nullptr;
        en.tab[t].next = nullptr;
        en.tab[t].cap_docs = en.tab[t].cap_slots = 0;
    }
    en.map = nullptr;
    en.part_start = nullptr;
    e->n_sets = 0;
    cudaSetDevice(prev);
}

void dsk_lsh_ensemble_destroy(dsk_lsh_ensemble *e) {
    if (!e) return;
    ensemble_free(e);
    delete e;
}

int dsk_lsh_ensemble_size(const dsk_lsh_ensemble *e, int64_t *n_sets) {
    if (!e) {
        set_error("dsk_lsh_ensemble_size: null handle");
        return DSK_ERR_INVALID;
    }
    if (n_sets) *n_sets = e->n_sets;
    return DSK_OK;
}

int dsk_lsh_ensemble_index(dsk_lsh_ensemble *e, const uint32_t *d_sig, int64_t n, const int32_t *d_order,
                           const int64_t *h_part_start, void *stream) {
    if (!e) {
        set_error("dsk_lsh_ensemble_index: null handle");
        return DSK_ERR_INVALID;
    }
    if (e->n_sets > 0) {
        set_error("dsk_lsh_ensemble_index: Cannot call index again on a non-empty index");
        return DSK_ERR_INVALID;
    }
    if (n < 1 || n >= (1ll << 31)) {
        set_error("dsk_lsh_ensemble_index: n must be in [1, 2^31) (got %lld)", (long long)n);
        return DSK_ERR_INVALID;
    }
    if (!d_sig || !d_order || !h_part_start) {
        set_error("dsk_lsh_ensemble_index: null buffer");
        return DSK_ERR_INVALID;
    }
    EnsembleDev &en = e->dev;
    bool ok = h_part_start[0] == 0 && h_part_start[en.num_part] == n;
    for (int p = 0; p < en.num_part && ok; ++p) ok = h_part_start[p] <= h_part_start[p + 1];
    if (!ok) {
        set_error("dsk_lsh_ensemble_index: h_part_start must rise from 0 to n over num_part + 1 = %d entries", en.num_part + 1);
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = get_dev(e->device, &dev);
    if (rc) return rc;
    DevGuard guard(e->device);
    const int k = en.tab[0].k;
    const int64_t cap = ensemble_cap_slots(n);
    uint32_t *sig = nullptr;
    cudaError_t err = cudaMalloc(&sig, (size_t)n * k * 4);
    for (int t = 0; t < en.n_tabs; ++t) {
        en.tab[t].sig = sig;
        en.tab[t].cap_docs = n;
        en.tab[t].cap_slots = cap;
    }
    if (err == cudaSuccess) err = cudaMalloc(&en.map, (size_t)n * 4);
    if (err == cudaSuccess) err = cudaMalloc(&en.part_start, (size_t)(en.num_part + 1) * 8);
    for (int t = 0; t < en.n_tabs && err == cudaSuccess; ++t) {
        err = cudaMalloc(&en.tab[t].slots, (size_t)en.tab[t].b * cap * 16);
        if (err == cudaSuccess) err = cudaMalloc(&en.tab[t].next, (size_t)en.tab[t].b * n * 4);
    }
    if (err == cudaSuccess)
        err = cudaMemcpy(en.part_start, h_part_start, (size_t)(en.num_part + 1) * 8, cudaMemcpyHostToDevice);
    if (err == cudaSuccess) err = ensemble_index(en, d_sig, d_order, n, dev->sm_count, (cudaStream_t)stream);
    if (err != cudaSuccess) {   // nothing is kept: the handle is empty again and can index
        cudaGetLastError();
        const size_t need = dsk_lsh_ensemble_index_bytes(e, n);
        int rc2 = cuda_fail(err, "dsk_lsh_ensemble_index");
        if (err == cudaErrorMemoryAllocation)
            set_error("dsk_lsh_ensemble_index: cannot allocate the %zu bytes of device memory an index of %lld sets needs",
                      need, (long long)n);
        ensemble_free(e);
        return rc2;
    }
    e->n_sets = n;
    return DSK_OK;
}

// handle, nq >= 0 and, when nq > 0, the query matrix, the selection table and every output buffer
static int check_ensemble_query(const char *who, const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq,
                                const int32_t *d_sel, bool bufs) {
    if (!e) {
        set_error("%s: null handle", who);
        return DSK_ERR_INVALID;
    }
    if (nq < 0 || nq > INT64_MAX / e->dev.num_part) {
        set_error("%s: nq must be >= 0 (got %lld)", who, (long long)nq);
        return DSK_ERR_INVALID;
    }
    if (nq > 0 && (!d_qsig || !d_sel || !bufs)) {
        set_error("%s: null buffer", who);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

int dsk_lsh_ensemble_query_count(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq, const int32_t *d_sel,
                                 int64_t *d_counts, void *stream) {
    int rc = check_ensemble_query("dsk_lsh_ensemble_query_count", e, d_qsig, nq, d_sel, d_counts != nullptr);
    if (rc || nq == 0) return rc;
    DevGuard guard(e->device);
    if (e->n_sets == 0) {   // nothing indexed: no partition has an upper bound, no query has a candidate
        DSK_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)nq * e->dev.num_part * 8, (cudaStream_t)stream));
        return DSK_OK;
    }
    DevInfo *dev;
    rc = get_dev(e->device, &dev);
    if (rc) return rc;
    DSK_CUDA(ensemble_query(e->dev, d_qsig, nq, d_sel, d_counts, nullptr, nullptr, nullptr, dev->sm_count,
                            (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lsh_ensemble_query_fill(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq, const int32_t *d_sel,
                                const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq, void *stream) {
    int rc = check_ensemble_query("dsk_lsh_ensemble_query_fill", e, d_qsig, nq, d_sel, d_ptr && d_idx);
    if (rc || nq == 0 || e->n_sets == 0) return rc;
    DevInfo *dev;
    rc = get_dev(e->device, &dev);
    if (rc) return rc;
    DevGuard guard(e->device);
    DSK_CUDA(ensemble_query(e->dev, d_qsig, nq, d_sel, nullptr, d_ptr, d_idx, d_eq, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

// check_ensemble_query, plus min_containment in [0, 1] (NaN fails both comparisons)
static int check_ensemble_containment(const char *who, const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq,
                                      const int32_t *d_sel, bool bufs, double min_containment) {
    int rc = check_ensemble_query(who, e, d_qsig, nq, d_sel, bufs);
    if (rc) return rc;
    if (!(min_containment >= 0.0 && min_containment <= 1.0)) {
        set_error("%s: min_containment must be in [0, 1] (got %g)", who, min_containment);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

// the count and fill of the query and self-join flavours; qsig == nullptr is the self-join (nq = the number of sets)
static int ensemble_containment_call(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq, const int64_t *d_qsizes,
                                     const int32_t *d_sel, const int64_t *d_set_sizes, double min_containment,
                                     int64_t *d_counts, const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq,
                                     double *d_containment, void *stream) {
    DevGuard guard(e->device);
    if (e->n_sets == 0) {   // nothing indexed: no candidates
        if (d_counts) DSK_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)nq * e->dev.num_part * 8, (cudaStream_t)stream));
        return DSK_OK;
    }
    DevInfo *dev;
    int rc = get_dev(e->device, &dev);
    if (rc) return rc;
    DSK_CUDA(ensemble_containment(e->dev, d_qsig, nq, d_qsizes, d_sel, d_set_sizes, min_containment, d_counts, d_ptr, d_idx,
                                  d_eq, d_containment, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lsh_ensemble_containment_count(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq, const int64_t *d_qsizes,
                                       const int32_t *d_sel, const int64_t *d_set_sizes, double min_containment,
                                       int64_t *d_counts, void *stream) {
    int rc = check_ensemble_containment("dsk_lsh_ensemble_containment_count", e, d_qsig, nq, d_sel,
                                        d_qsizes && d_set_sizes && d_counts, min_containment);
    if (rc || nq == 0) return rc;
    return ensemble_containment_call(e, d_qsig, nq, d_qsizes, d_sel, d_set_sizes, min_containment, d_counts, nullptr, nullptr,
                                     nullptr, nullptr, stream);
}

int dsk_lsh_ensemble_containment_fill(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq, const int64_t *d_qsizes,
                                      const int32_t *d_sel, const int64_t *d_set_sizes, double min_containment,
                                      const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq, double *d_containment,
                                      void *stream) {
    int rc = check_ensemble_containment("dsk_lsh_ensemble_containment_fill", e, d_qsig, nq, d_sel,
                                        d_qsizes && d_set_sizes && d_ptr && d_idx && d_eq && d_containment, min_containment);
    if (rc || nq == 0) return rc;
    return ensemble_containment_call(e, d_qsig, nq, d_qsizes, d_sel, d_set_sizes, min_containment, nullptr, d_ptr, d_idx,
                                     d_eq, d_containment, stream);
}

int dsk_lsh_ensemble_containment_topk(const dsk_lsh_ensemble *e, const uint32_t *d_qsig, int64_t nq, const int64_t *d_qsizes,
                                      const int32_t *d_sel, const int64_t *d_set_sizes, double min_containment, int k,
                                      int32_t *d_idx, int32_t *d_eq, double *d_containment, void *stream) {
    const char *who = "dsk_lsh_ensemble_containment_topk";
    int rc = check_ensemble_containment(who, e, d_qsig, nq, d_sel, d_qsizes && d_set_sizes && d_idx && d_eq && d_containment,
                                        min_containment);
    if (rc) return rc;
    if (k < 1 || k > 32) {
        set_error("%s: k must be in [1, 32] (got %d)", who, k);
        return DSK_ERR_INVALID;
    }
    if (nq == 0) return DSK_OK;
    DevInfo *dev;
    rc = get_dev(e->device, &dev);
    if (rc) return rc;
    DevGuard guard(e->device);
    DSK_CUDA(ensemble_containment_topk(e->dev, d_qsig, nq, d_qsizes, d_sel, d_set_sizes, min_containment, k, d_idx, d_eq,
                                       d_containment, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_lsh_ensemble_self_containment_count(const dsk_lsh_ensemble *e, const int32_t *d_sel, const int64_t *d_set_sizes,
                                            double min_containment, int64_t *d_counts, void *stream) {
    const char *who = "dsk_lsh_ensemble_self_containment_count";
    const int64_t n = e ? e->n_sets : 0;
    int rc = check_ensemble_containment(who, e, nullptr, 0, d_sel, true, min_containment);
    if (rc || n == 0) return rc;
    if (!d_sel || !d_set_sizes || !d_counts) {
        set_error("%s: null buffer", who);
        return DSK_ERR_INVALID;
    }
    return ensemble_containment_call(e, nullptr, n, nullptr, d_sel, d_set_sizes, min_containment, d_counts, nullptr, nullptr,
                                     nullptr, nullptr, stream);
}

int dsk_lsh_ensemble_self_containment_fill(const dsk_lsh_ensemble *e, const int32_t *d_sel, const int64_t *d_set_sizes,
                                           double min_containment, const int64_t *d_ptr, int32_t *d_idx, int32_t *d_eq,
                                           double *d_containment, void *stream) {
    const char *who = "dsk_lsh_ensemble_self_containment_fill";
    const int64_t n = e ? e->n_sets : 0;
    int rc = check_ensemble_containment(who, e, nullptr, 0, d_sel, true, min_containment);
    if (rc || n == 0) return rc;
    if (!d_sel || !d_set_sizes || !d_ptr || !d_idx || !d_eq || !d_containment) {
        set_error("%s: null buffer", who);
        return DSK_ERR_INVALID;
    }
    return ensemble_containment_call(e, nullptr, n, nullptr, d_sel, d_set_sizes, min_containment, nullptr, d_ptr, d_idx, d_eq,
                                     d_containment, stream);
}

// ---- MinHashLSHEnsemble's size partitioner -------------------------------------------------------------------------------
// acc += a * b rounded up to 256 bytes; false if it does not fit in size_t
static bool ws_add(size_t &acc, uint64_t a, uint64_t b) {
    if (a != 0 && b > (SIZE_MAX - 512) / a) return false;
    const size_t part = (size_t)((a * b + 255) / 256 * 256);
    if (acc > SIZE_MAX - part) return false;
    acc += part;
    return true;
}

// workspace layout: sizes, counts [n] int64; the terms rows of the cost launch (large n); for 2 <= num_part < n the triangle
// [n(n+1)/2], the tables [num_part - 1][n] (doubles) and the upper indices [num_part] int64
static size_t partition_ws(int64_t n, int num_part, size_t *off_terms, size_t *off_cost, size_t *off_tab, size_t *off_upper) {
    size_t acc = 0;
    bool ok = ws_add(acc, (uint64_t)n, 16);
    if (off_terms) *off_terms = acc;
    ok = ok && ws_add(acc, (uint64_t)partition_term_rows(n), (uint64_t)n * 8);
    if (num_part >= 2 && num_part < n) {
        if (off_cost) *off_cost = acc;
        ok = ok && (uint64_t)n < (1ull << 32) && ws_add(acc, (uint64_t)n * (uint64_t)(n + 1) / 2, 8);
        if (off_tab) *off_tab = acc;
        ok = ok && ws_add(acc, (uint64_t)(num_part - 1) * 8, (uint64_t)n);
        if (off_upper) *off_upper = acc;
        ok = ok && ws_add(acc, (uint64_t)num_part, 8);
    }
    return ok ? acc : SIZE_MAX;
}

size_t dsk_ensemble_partition_workspace_size(int64_t n_sizes, int num_part) {
    if (n_sizes < 1 || num_part < 1) return 0;
    return partition_ws(n_sizes, num_part, nullptr, nullptr, nullptr, nullptr);
}

int dsk_ensemble_partition(const int64_t *h_sizes, const int64_t *h_counts, int64_t n_sizes, int num_part, void *d_workspace,
                           size_t workspace_bytes, int device, int64_t *h_upper_idx, double *d_cost, void *stream) {
    const char *who = "dsk_ensemble_partition";
    if (n_sizes < 1 || num_part < 1) {
        set_error("%s: need n_sizes >= 1 and num_part >= 1 (got %lld and %d)", who, (long long)n_sizes, num_part);
        return DSK_ERR_INVALID;
    }
    if (!h_sizes || !h_counts || !h_upper_idx) {
        set_error("%s: null buffer", who);
        return DSK_ERR_INVALID;
    }
    const int64_t kMax = (int64_t)1 << 62;
    for (int64_t i = 0; i < n_sizes; ++i) {
        if (h_sizes[i] <= 0 || h_sizes[i] >= kMax || (i > 0 && h_sizes[i] <= h_sizes[i - 1])) {
            set_error("%s: sizes must be strictly ascending, each in [1, 2^62) (sizes[%lld] = %lld)", who, (long long)i,
                      (long long)h_sizes[i]);
            return DSK_ERR_INVALID;
        }
        if (h_counts[i] <= 0 || h_counts[i] >= kMax) {
            set_error("%s: counts must be in [1, 2^62) (counts[%lld] = %lld)", who, (long long)i, (long long)h_counts[i]);
            return DSK_ERR_INVALID;
        }
    }
    const bool trivial = num_part < 2 || num_part >= n_sizes;
    if (trivial) {   // one partition, or one per size: no table (the triangle only if asked for)
        if (num_part < 2) h_upper_idx[0] = n_sizes - 1;
        else for (int64_t i = 0; i < n_sizes; ++i) h_upper_idx[i] = i;
        if (!d_cost) return DSK_OK;
    }
    size_t off_terms = 0, off_cost = 0, off_tab = 0, off_upper = 0;
    const size_t need = partition_ws(n_sizes, num_part, &off_terms, &off_cost, &off_tab, &off_upper);
    if (need == SIZE_MAX) {
        set_error("%s: the workspace for n_sizes = %lld and num_part = %d does not fit in size_t", who, (long long)n_sizes,
                  num_part);
        return DSK_ERR_INVALID;
    }
    if (!d_workspace || workspace_bytes < need || ((uintptr_t)d_workspace & 15u) != 0) {
        set_error("%s: the workspace must be 16-byte aligned and hold %zu bytes (got %zu at %p)", who, need, workspace_bytes,
                  d_workspace);
        return DSK_ERR_INVALID;
    }
    if (d_cost && ((uintptr_t)d_cost & 7u) != 0) {
        set_error("%s: d_cost must be 8-byte aligned", who);
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = get_dev(device, &dev);
    if (rc) return rc;
    DevGuard guard(device);
    const cudaStream_t s = (cudaStream_t)stream;
    unsigned char *ws = static_cast<unsigned char *>(d_workspace);
    int64_t *sizes = reinterpret_cast<int64_t *>(ws), *counts = sizes + n_sizes;
    double *g_terms = partition_term_rows(n_sizes) ? reinterpret_cast<double *>(ws + off_terms) : nullptr;
    double *cost = d_cost ? d_cost : reinterpret_cast<double *>(ws + off_cost);
    double *tab = trivial ? nullptr : reinterpret_cast<double *>(ws + off_tab);
    int64_t *upper = reinterpret_cast<int64_t *>(ws + off_upper);
    DSK_CUDA(cudaMemcpyAsync(sizes, h_sizes, (size_t)n_sizes * 8, cudaMemcpyHostToDevice, s));
    DSK_CUDA(cudaMemcpyAsync(counts, h_counts, (size_t)n_sizes * 8, cudaMemcpyHostToDevice, s));
    DSK_CUDA(ensemble_partition(sizes, counts, n_sizes, num_part, cost, tab, g_terms, upper, dev->sm_count, s));
    if (!trivial) DSK_CUDA(cudaMemcpyAsync(h_upper_idx, upper, (size_t)num_part * 8, cudaMemcpyDeviceToHost, s));
    DSK_CUDA(cudaStreamSynchronize(s));
    return DSK_OK;
}

int dsk_jaccard_pairs(const uint32_t *d_sig, int64_t n_rows, int num_perm, const int64_t *d_i, const int64_t *d_j,
                      int64_t m, int32_t *d_count, void *stream) {
    if (n_rows < 0 || num_perm <= 0 || m < 0 || (m > 0 && (!d_sig || !d_i || !d_j || !d_count))) {
        set_error("dsk_jaccard_pairs: bad arguments");
        return DSK_ERR_INVALID;
    }
    if ((num_perm & 3) == 0 && ((uintptr_t)d_sig & 15) != 0) {
        set_error("dsk_jaccard_pairs: d_sig must be 16-byte aligned");
        return DSK_ERR_ALIGN;
    }
    DevInfo *dev;
    int rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_jaccard_pairs(d_sig, n_rows, num_perm, d_i, d_j, m, d_count, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

size_t dsk_jaccard_topk_workspace_size(int64_t nq, int64_t n, int num_perm) {
    return (nq < 0 || n < 0) ? 0 : jaccard_topk_workspace_bytes(nq, n, num_perm);
}

int dsk_jaccard_topk(const uint32_t *d_q, int64_t nq, const uint32_t *d_db, int64_t n, int num_perm, int topk,
                     int64_t self_base, int32_t *d_cnt, int64_t *d_idx, void *stream) {
    return dsk_jaccard_topk_ws(d_q, nq, d_db, n, num_perm, topk, self_base, d_cnt, d_idx, nullptr, 0, stream);
}

int dsk_jaccard_topk_ws(const uint32_t *d_q, int64_t nq, const uint32_t *d_db, int64_t n, int num_perm, int topk,
                        int64_t self_base, int32_t *d_cnt, int64_t *d_idx, void *d_workspace, size_t workspace_bytes,
                        void *stream) {
    if (nq < 0 || n < 0 || num_perm <= 0 || num_perm > 4096 || topk <= 0 || topk > 32 ||
        (nq > 0 && (!d_q || !d_cnt || !d_idx)) || (n > 0 && !d_db)) {
        set_error("dsk_jaccard_topk: bad arguments (need 0 < topk <= 32, 0 < num_perm <= 4096)");
        return DSK_ERR_INVALID;
    }
    if ((num_perm & 3) == 0 && ((uintptr_t)d_db & 15) != 0) {
        set_error("dsk_jaccard_topk: d_db must be 16-byte aligned");
        return DSK_ERR_ALIGN;
    }
    const size_t need = jaccard_topk_workspace_bytes(nq, n, num_perm);
    if (d_workspace && (((uintptr_t)d_workspace & 15) != 0 || workspace_bytes < need)) {
        set_error("dsk_jaccard_topk_ws: workspace must be 16-byte aligned and hold dsk_jaccard_topk_workspace_size() = %zu bytes", need);
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = current_dev(&dev);
    if (rc) return rc;
    if (d_workspace && need > 0)   // fingerprint prefilter, then exact counts of the surviving pairs
        DSK_CUDA(launch_jaccard_topk_pf(d_q, nq, d_db, n, num_perm, topk, self_base, d_cnt, d_idx, d_workspace, dev->sm_count,
                                        (cudaStream_t)stream));
    else
        DSK_CUDA(launch_jaccard_topk(d_q, nq, d_db, n, num_perm, topk, self_base, d_cnt, d_idx, dev->sm_count,
                                     (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_sha1_tokens(const uint8_t *d_bytes, const int64_t *d_byte_offsets, int64_t n_tokens, void *d_out,
                    int out_is_u64, void *stream) {
    if (n_tokens < 0 || (n_tokens > 0 && (!d_byte_offsets || !d_out))) {
        set_error("dsk_sha1_tokens: bad arguments");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_sha1_tokens(d_bytes, d_byte_offsets, n_tokens, d_out, out_is_u64, dev->sm_count,
                                (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_hash_tokens(const uint8_t *d_bytes, const int64_t *d_byte_offsets, int64_t n_tokens, int kind, uint32_t seed,
                    uint32_t *d_out, void *stream) {
    if (n_tokens < 0 || (kind != DSK_HASH_XXH32 && kind != DSK_HASH_MURMUR3_32) ||
        (n_tokens > 0 && (!d_byte_offsets || !d_out))) {
        set_error("dsk_hash_tokens: bad arguments (kind must be DSK_HASH_XXH32 or DSK_HASH_MURMUR3_32)");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_hash_tokens(d_bytes, d_byte_offsets, n_tokens, kind, seed, d_out, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

size_t dsk_shingle_workspace_size(int64_t n_docs, int64_t n_bytes) {
    return n_docs < 0 || n_bytes < 0 ? 0 : shingle_workspace_bytes(n_docs, n_bytes);
}

static int check_shingle(const char *who, const uint8_t *d_text, const int64_t *d_doc_offsets, int64_t n_docs,
                         int64_t n_bytes, int unit, int n, const void *d_ws, size_t ws_bytes) {
    if (n_docs < 0 || n_bytes < 0 || n < 1 || (unit != DSK_SHINGLE_WORD && unit != DSK_SHINGLE_CHAR) || !d_doc_offsets ||
        (n_bytes > 0 && !d_text)) {
        set_error("%s: bad arguments (n_docs, n_bytes >= 0, n >= 1, unit DSK_SHINGLE_WORD or DSK_SHINGLE_CHAR)", who);
        return DSK_ERR_INVALID;
    }
    const size_t need = shingle_workspace_bytes(n_docs, n_bytes);
    if (!d_ws || ((uintptr_t)d_ws & 15) != 0 || ws_bytes < need) {
        set_error("%s: the workspace must be 16-byte aligned and hold dsk_shingle_workspace_size() = %zu bytes (got %zu)", who,
                  need, ws_bytes);
        return DSK_ERR_INVALID;
    }
    if (((uintptr_t)d_doc_offsets & 7) != 0) {
        set_error("%s: d_doc_offsets must be 8-byte aligned", who);
        return DSK_ERR_ALIGN;
    }
    return DSK_OK;
}

int dsk_shingle_count(const uint8_t *d_text, const int64_t *d_doc_offsets, int64_t n_docs, int64_t n_bytes, int unit, int n,
                      int64_t *d_tok_offsets, int32_t *d_doc_status, void *d_ws, size_t ws_bytes, void *stream) {
    int rc = check_shingle("dsk_shingle_count", d_text, d_doc_offsets, n_docs, n_bytes, unit, n, d_ws, ws_bytes);
    if (rc) return rc;
    if (!d_tok_offsets || !d_doc_status) {
        set_error("dsk_shingle_count: null output");
        return DSK_ERR_INVALID;
    }
    if (((uintptr_t)d_tok_offsets & 7) != 0 || ((uintptr_t)d_doc_status & 3) != 0) {
        set_error("dsk_shingle_count: d_tok_offsets must be 8-byte and d_doc_status 4-byte aligned");
        return DSK_ERR_ALIGN;
    }
    if (n_docs == 0) {   // no document: no byte is read
        DSK_CUDA(cudaMemsetAsync(d_tok_offsets, 0, sizeof(int64_t), (cudaStream_t)stream));
        DSK_CUDA(cudaMemsetAsync(d_doc_status, 0, sizeof(int32_t), (cudaStream_t)stream));
        return DSK_OK;
    }
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(shingle_count(d_text, d_doc_offsets, n_docs, n_bytes, unit == DSK_SHINGLE_WORD, n, d_tok_offsets, d_doc_status,
                           d_ws, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_shingle_hash(const uint8_t *d_text, const int64_t *d_doc_offsets, int64_t n_docs, int64_t n_bytes, int unit, int n,
                     int hash_kind, uint32_t seed, const int64_t *d_tok_offsets, uint32_t *d_tokens, void *d_ws,
                     size_t ws_bytes, void *stream) {
    int rc = check_shingle("dsk_shingle_hash", d_text, d_doc_offsets, n_docs, n_bytes, unit, n, d_ws, ws_bytes);
    if (rc) return rc;
    if (hash_kind != 0 && hash_kind != DSK_HASH_XXH32 && hash_kind != DSK_HASH_MURMUR3_32) {
        set_error("dsk_shingle_hash: hash_kind must be 0 (sha1_hash32), DSK_HASH_XXH32 or DSK_HASH_MURMUR3_32 (got %d)",
                  hash_kind);
        return DSK_ERR_INVALID;
    }
    if (!d_tok_offsets || !d_tokens) {
        set_error("dsk_shingle_hash: null buffer");
        return DSK_ERR_INVALID;
    }
    if (((uintptr_t)d_tok_offsets & 7) != 0 || ((uintptr_t)d_tokens & 3) != 0) {
        set_error("dsk_shingle_hash: d_tok_offsets must be 8-byte and d_tokens 4-byte aligned");
        return DSK_ERR_ALIGN;
    }
    if (n_docs == 0) return DSK_OK;
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(shingle_hash(d_text, d_doc_offsets, n_docs, n_bytes, unit == DSK_SHINGLE_WORD, n, hash_kind, seed, d_tok_offsets,
                          d_tokens, d_ws, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

static int bbit_slot(int b) {
    if (b < 0 || b > 32) return -1;
    if (b == 1) return 1;
    if (b == 2) return 2;
    if (b <= 4) return 4;
    if (b <= 8) return 8;
    if (b <= 16) return 16;
    return 32;
}

int dsk_bbit_pack(const uint32_t *d_sig, int64_t n, int num_perm, int b, uint64_t *d_blocks, void *stream) {
    const int slot = bbit_slot(b);
    if (slot < 0 || n < 0 || num_perm <= 0 || (n > 0 && (!d_sig || !d_blocks))) {
        set_error("dsk_bbit_pack: bad arguments (b must be in [0, 32])");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_bbit_pack(d_sig, n, num_perm, b, slot, d_blocks, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_bbit_unpack(const uint64_t *d_blocks, int64_t n, int num_perm, int b, uint32_t *d_sig, void *stream) {
    const int slot = bbit_slot(b);
    if (slot < 0 || n < 0 || num_perm <= 0 || (n > 0 && (!d_sig || !d_blocks))) {
        set_error("dsk_bbit_unpack: bad arguments (b must be in [0, 32])");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_bbit_unpack(d_blocks, n, num_perm, slot, d_sig, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_forest_query(const uint32_t *d_sig, const int32_t *d_order, int64_t n, int num_perm, int l, int k,
                     const uint32_t *d_qsig, int64_t nq, int topk, int32_t *d_out, void *stream) {
    if (n < 0 || nq < 0 || num_perm <= 0 || l <= 0 || k <= 0 || (int64_t)l * k > num_perm || topk <= 0 || topk > 1024 ||
        (nq > 0 && (!d_qsig || !d_out)) || (n > 0 && (!d_sig || !d_order))) {
        set_error("dsk_forest_query: bad arguments (need l*k <= num_perm, 0 < topk <= 1024)");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    int rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_forest_query(d_sig, d_order, n, num_perm, l, k, d_qsig, nq, topk, d_out, dev->sm_count,
                                 (cudaStream_t)stream));
    return DSK_OK;
}

// The ranked and weighted forest walks.  num_perm, l and k count samples (weighted rows are [n, 2 * num_perm] words).
static int check_forest(const char *who, const uint32_t *d_sig, const int32_t *d_order, int64_t n, int num_perm, int weighted,
                        int l, int k, const uint32_t *d_qsig, int64_t nq) {
    if (n < 0 || nq < 0 || num_perm <= 0 || num_perm > (1 << 29) || l <= 0 || k <= 0 || (int64_t)l * k > num_perm ||
        (weighted != 0 && weighted != 1) || (n > 0 && (!d_sig || !d_order)) || (nq > 0 && !d_qsig)) {
        set_error("%s: bad arguments (need 0 < l*k <= num_perm, weighted 0 or 1, buffers where work exists)", who);
        return DSK_ERR_INVALID;
    }
    if (weighted && ((n > 0 && ((uintptr_t)d_sig & 7) != 0) || (nq > 0 && ((uintptr_t)d_qsig & 7) != 0))) {
        set_error("%s: weighted rows must be 8-byte aligned", who);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

static int check_forest_topk(const char *who, int num_perm, int candidates, int min_count, int topk, int64_t rows,
                             const int32_t *d_idx, const int32_t *d_eq) {
    if (topk < 1 || topk > 32 || candidates < topk || candidates > 1024 || min_count < 0 || min_count > num_perm ||
        (rows > 0 && (!d_idx || !d_eq))) {
        set_error("%s: bad arguments (need 1 <= topk <= 32, topk <= candidates <= 1024, 0 <= min_count <= num_perm, "
                  "output buffers)", who);
        return DSK_ERR_INVALID;
    }
    return DSK_OK;
}

int dsk_forest_query_weighted(const uint32_t *d_sig, const int32_t *d_order, int64_t n, int sample_size, int l, int k,
                              const uint32_t *d_qsig, int64_t nq, int topk, int32_t *d_out, void *stream) {
    int rc = check_forest("dsk_forest_query_weighted", d_sig, d_order, n, sample_size, 1, l, k, d_qsig, nq);
    if (rc) return rc;
    if (topk <= 0 || topk > 1024 || (nq > 0 && !d_out)) {
        set_error("dsk_forest_query_weighted: bad arguments (need 0 < topk <= 1024, an output buffer)");
        return DSK_ERR_INVALID;
    }
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_forest(FOREST_SET, 2, d_sig, d_order, n, 2 * sample_size, l, k, d_qsig, nq, topk, d_out, nullptr, 0, 0,
                           dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_forest_query_topk(const uint32_t *d_sig, const int32_t *d_order, int64_t n, int num_perm, int weighted, int l,
                          int k, const uint32_t *d_qsig, int64_t nq, int candidates, int min_count, int topk,
                          int32_t *d_idx, int32_t *d_eq, void *stream) {
    int rc = check_forest("dsk_forest_query_topk", d_sig, d_order, n, num_perm, weighted, l, k, d_qsig, nq);
    if (!rc) rc = check_forest_topk("dsk_forest_query_topk", num_perm, candidates, min_count, topk, nq, d_idx, d_eq);
    if (rc) return rc;
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_forest(FOREST_QUERY_TOPK, weighted ? 2 : 1, d_sig, d_order, n, weighted ? 2 * num_perm : num_perm, l, k,
                           d_qsig, nq, candidates, d_idx, d_eq, topk, min_count, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

int dsk_forest_neighbors(const uint32_t *d_sig, const int32_t *d_order, int64_t n, int num_perm, int weighted, int l, int k,
                         int candidates, int min_count, int topk, int32_t *d_idx, int32_t *d_eq, void *stream) {
    int rc = check_forest("dsk_forest_neighbors", d_sig, d_order, n, num_perm, weighted, l, k, d_sig, n);
    if (!rc) rc = check_forest_topk("dsk_forest_neighbors", num_perm, candidates, min_count, topk, n, d_idx, d_eq);
    if (rc) return rc;
    DevInfo *dev;
    rc = current_dev(&dev);
    if (rc) return rc;
    DSK_CUDA(launch_forest(FOREST_SELF_TOPK, weighted ? 2 : 1, d_sig, d_order, n, weighted ? 2 * num_perm : num_perm, l, k,
                           nullptr, 0, candidates, d_idx, d_eq, topk, min_count, dev->sm_count, (cudaStream_t)stream));
    return DSK_OK;
}

// ---- host-buffer pipeline --------------------------------------------------------------------
extern "C++" {
namespace {
constexpr int kSlots = 3;
struct HostPipe {
    int device = -1;
    cudaStream_t stream[kSlots] = {};
    void *d_tok[kSlots] = {};
    int64_t *d_off[kSlots] = {};
    void *d_out[kSlots] = {};
    void *d_init[kSlots] = {};
    int64_t *h_off[kSlots] = {};  // pinned staging for rebased offsets
    // long documents are split into pieces: partial signatures + segment pointers
    uint32_t *d_part[kSlots] = {};
    int64_t *d_seg[kSlots] = {};
    int64_t *h_seg[kSlots] = {};
    size_t cap_tok = 0, cap_off_dev = 0, cap_off_host = 0, cap_out = 0, cap_init = 0, cap_part = 0, cap_seg_dev = 0,
           cap_seg_host = 0;   // bytes per slot of each buffer class
};
HostPipe g_pipe[64];
std::mutex g_pipe_mu;

// one buffer class of the pipeline (kSlots buffers of equal capacity); a failed (re)allocation leaves it EMPTY
// (all slots null, capacity 0), so the next call allocates again instead of copying to a null pointer
template <typename T>
int pipe_grow(T *(&slot)[kSlots], size_t &cap, size_t want_bytes, bool pinned) {
    if (want_bytes <= cap) return DSK_OK;
    for (int i = 0; i < kSlots; ++i) {
        if (slot[i]) {
            if (pinned) cudaFreeHost(slot[i]);
            else cudaFree(slot[i]);
        }
        slot[i] = nullptr;
    }
    cap = 0;
    for (int i = 0; i < kSlots; ++i) {
        void *ptr = nullptr;
        const cudaError_t e = pinned ? cudaMallocHost(&ptr, want_bytes + 64) : cudaMalloc(&ptr, want_bytes + 64);
        if (e != cudaSuccess) {
            for (int q = 0; q < i; ++q) {
                if (pinned) cudaFreeHost(slot[q]);
                else cudaFree(slot[q]);
                slot[q] = nullptr;
            }
            return cuda_fail(e, "host pipeline buffer allocation");
        }
        slot[i] = static_cast<T *>(ptr);
    }
    cap = want_bytes;
    return DSK_OK;
}

int pipe_reserve(HostPipe &hp, int device, size_t tok_bytes, size_t docs, size_t out_bytes, size_t init_bytes,
                 size_t part_bytes, size_t seg_docs) {
    if (hp.device < 0) {
        for (int i = 0; i < kSlots; ++i) DSK_CUDA(cudaStreamCreateWithFlags(&hp.stream[i], cudaStreamNonBlocking));
        hp.device = device;
    }
    int rc;
    if ((rc = pipe_grow(hp.d_tok, hp.cap_tok, tok_bytes, false))) return rc;
    const size_t off_bytes = (docs + 1) * sizeof(int64_t);
    if (off_bytes > hp.cap_off_dev && (rc = pipe_grow(hp.d_off, hp.cap_off_dev, off_bytes, false))) return rc;
    if (off_bytes > hp.cap_off_host && (rc = pipe_grow(hp.h_off, hp.cap_off_host, off_bytes, true))) return rc;
    if ((rc = pipe_grow(hp.d_out, hp.cap_out, out_bytes, false))) return rc;
    if (part_bytes && (rc = pipe_grow(hp.d_part, hp.cap_part, part_bytes, false))) return rc;
    if (seg_docs) {
        const size_t seg_bytes = (seg_docs + 1) * sizeof(int64_t);
        if ((rc = pipe_grow(hp.d_seg, hp.cap_seg_dev, seg_bytes, false))) return rc;
        if ((rc = pipe_grow(hp.h_seg, hp.cap_seg_host, seg_bytes, true))) return rc;
    }
    if (init_bytes && (rc = pipe_grow(hp.d_init, hp.cap_init, init_bytes, false))) return rc;
    return DSK_OK;
}

void pipe_release(HostPipe &hp) {
    if (hp.device < 0) return;
    int prev = 0;
    cudaGetDevice(&prev);
    cudaSetDevice(hp.device);
    for (int i = 0; i < kSlots; ++i) {
        if (hp.stream[i]) { cudaStreamSynchronize(hp.stream[i]); cudaStreamDestroy(hp.stream[i]); }
        if (hp.d_tok[i]) cudaFree(hp.d_tok[i]);
        if (hp.d_off[i]) cudaFree(hp.d_off[i]);
        if (hp.d_out[i]) cudaFree(hp.d_out[i]);
        if (hp.d_init[i]) cudaFree(hp.d_init[i]);
        if (hp.d_part[i]) cudaFree(hp.d_part[i]);
        if (hp.d_seg[i]) cudaFree(hp.d_seg[i]);
        if (hp.h_off[i]) cudaFreeHost(hp.h_off[i]);
        if (hp.h_seg[i]) cudaFreeHost(hp.h_seg[i]);
    }
    hp = HostPipe();
    cudaSetDevice(prev);
}
}  // namespace
}  // extern "C++"

int dsk_release_host_pipeline(int device) {
    if (device < -1 || device >= 64) {
        set_error("dsk_release_host_pipeline: device must be -1 (all) or a device index");
        return DSK_ERR_INVALID;
    }
    std::lock_guard<std::mutex> lk(g_pipe_mu);
    for (int d = 0; d < 64; ++d)
        if (device < 0 || d == device) pipe_release(g_pipe[d]);
    return DSK_OK;
}

int dsk_minhash_bulk_host(const dsk_perm *perm, const void *h_tokens, int token_is_u64, const int64_t *h_offsets,
                          int64_t n_docs, const void *h_init, int64_t init_stride, int init_is_u64, void *h_out,
                          int out_is_u64, int flags) {
    if (!perm || !h_offsets || !h_out || n_docs < 0) {
        set_error("dsk_minhash_bulk_host: bad arguments");
        return DSK_ERR_INVALID;
    }
    if (n_docs == 0) return DSK_OK;
    const int64_t n_tokens = h_offsets[n_docs] - h_offsets[0];
    if (n_tokens < 0 || (n_tokens > 0 && !h_tokens)) {
        set_error("dsk_minhash_bulk_host: bad offsets / tokens");
        return DSK_ERR_INVALID;
    }
    int mode;
    int rc = pick_mode(perm, token_is_u64, flags, &mode);
    if (rc) return rc;
    DevInfo *dev;
    rc = get_dev(perm->device, &dev);
    if (rc) return rc;

    const size_t tsz = token_is_u64 ? 8 : 4, osz = out_is_u64 ? 8 : 4;
    const int K = perm->num_perm;
    // slice limits: ~16 Mi tokens and 128 Ki documents per slice keep each copy in the MB range
    // (DSK_SLICE_TOKENS overrides the token limit: a tuning knob for the copy/compute overlap, not a semantic one)
    int64_t max_tok = 16ll << 20;
    const int64_t max_docs = 128ll << 10;
    if (const char *e = getenv("DSK_SLICE_TOKENS")) {
        const long long v = atoll(e);
        if (v >= 4096) max_tok = v;
    }

    std::lock_guard<std::mutex> lk(g_pipe_mu);
    int prev = 0;
    cudaGetDevice(&prev);
    DSK_CUDA(cudaSetDevice(perm->device));
    HostPipe &hp = g_pipe[perm->device];

    // Long documents are cut into pieces so that many warps work on them (one warp per document otherwise);
    // the pieces' partial signatures are min-merged on the device (seg_min_kernel).
    auto piece_len = [](int64_t slice_tokens) -> int64_t { return slice_tokens < (2ll << 20) ? 2048 : 8192; };
    auto n_pieces = [](int64_t len, int64_t piece) -> int64_t { return len > 2 * piece ? (len + piece - 1) / piece : 1; };

    // first pass: slice boundaries (a single document larger than max_tok gets its own slice)
    std::vector<int64_t> cut;
    cut.push_back(0);
    int64_t biggest_tok = 0, biggest_docs = 0, biggest_ext = 0, biggest_split_docs = 0;
    {
        int64_t d0 = 0;
        while (d0 < n_docs) {
            int64_t d1 = d0;
            const int64_t t0 = h_offsets[d0];
            while (d1 < n_docs && d1 - d0 < max_docs && (h_offsets[d1 + 1] - t0 <= max_tok || d1 == d0)) ++d1;
            if (h_offsets[d1] < h_offsets[d0]) {
                cudaSetDevice(prev);
                set_error("dsk_minhash_bulk_host: offsets must be non-decreasing");
                return DSK_ERR_INVALID;
            }
            biggest_tok = biggest_tok > h_offsets[d1] - t0 ? biggest_tok : h_offsets[d1] - t0;
            biggest_docs = biggest_docs > d1 - d0 ? biggest_docs : d1 - d0;
            {
                const int64_t piece = piece_len(h_offsets[d1] - t0);
                int64_t ext = 0;
                bool decreasing = false;   // every interior offset is checked here, in the pass that reads them anyway
                for (int64_t i = d0; i < d1; ++i) {
                    const int64_t len = h_offsets[i + 1] - h_offsets[i];
                    decreasing |= len < 0;
                    ext += n_pieces(len, piece);
                }
                if (decreasing) {
                    cudaSetDevice(prev);
                    set_error("dsk_minhash_bulk_host: offsets must be non-decreasing");
                    return DSK_ERR_INVALID;
                }
                if (ext != d1 - d0) {
                    biggest_ext = biggest_ext > ext ? biggest_ext : ext;
                    biggest_split_docs = biggest_split_docs > d1 - d0 ? biggest_split_docs : d1 - d0;
                }
            }
            cut.push_back(d1);
            d0 = d1;
        }
    }
    const size_t isz = init_is_u64 ? 8 : 4;
    const size_t init_rows = !h_init ? 0 : (init_stride == 0 ? 1 : (size_t)biggest_docs);
    if (h_init && init_stride != 0 && init_stride < K) {
        cudaSetDevice(prev);
        set_error("dsk_minhash_bulk_host: init_stride must be 0 or >= num_perm");
        return DSK_ERR_INVALID;
    }
    rc = pipe_reserve(hp, perm->device, (size_t)biggest_tok * tsz,
                      (size_t)(biggest_docs > biggest_ext ? biggest_docs : biggest_ext), (size_t)biggest_docs * K * osz,
                      init_rows * (size_t)(init_stride ? init_stride : K) * isz, (size_t)biggest_ext * K * sizeof(uint32_t),
                      (size_t)biggest_split_docs);
    if (rc) {
        cudaSetDevice(prev);
        return rc;
    }

    BulkParams prm{};
    prm.a_lo = perm->d_tab;
    prm.a_hi = perm->d_tab + perm->kpad;
    prm.b_lo = perm->d_tab + 2 * perm->kpad;
    prm.b_hi = perm->d_tab + 3 * perm->kpad;
    prm.b_lo7 = perm->d_tab + 4 * perm->kpad;
    prm.b_lo8 = perm->d_tab + 5 * perm->kpad;
    prm.gen = token_is_u64 ? 2 : (perm->n_unsafe ? 1 : 0);
    prm.k = K;
    prm.init = nullptr;
    prm.init_stride = init_stride;
    prm.init_is_u64 = init_is_u64;
    prm.out_is_u64 = out_is_u64;

    cudaError_t e = cudaSuccess;
    for (size_t s = 0; s + 1 < cut.size() && e == cudaSuccess; ++s) {
        const int slot = (int)(s % kSlots);
        const int64_t d0 = cut[s], d1 = cut[s + 1], nd = d1 - d0;
        const int64_t t0 = h_offsets[d0], nt = h_offsets[d1] - t0;
        cudaStream_t st = hp.stream[slot];
        // the pinned offsets staging buffer of this slot is reused: wait for its previous slice
        if (s >= (size_t)kSlots) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) break;
        // offsets of this slice, rebased; documents above the split threshold become several pieces
        const int64_t piece = piece_len(nt);
        int64_t n_ext = 0;
        for (int64_t i = d0; i < d1; ++i) n_ext += n_pieces(h_offsets[i + 1] - h_offsets[i], piece);
        const bool split = n_ext != nd;
        if (!split) {
            for (int64_t i = 0; i <= nd; ++i) hp.h_off[slot][i] = h_offsets[d0 + i] - t0;
        } else {
            int64_t w = 0;
            for (int64_t i = d0; i < d1; ++i) {
                const int64_t b = h_offsets[i] - t0, len = h_offsets[i + 1] - h_offsets[i];
                const int64_t np = n_pieces(len, piece);
                hp.h_seg[slot][i - d0] = w;
                for (int64_t q = 0; q < np; ++q) hp.h_off[slot][w++] = b + (np == 1 ? 0 : q * piece);
            }
            hp.h_seg[slot][nd] = w;
            hp.h_off[slot][w] = nt;
        }
        if (nt > 0)
            e = cudaMemcpyAsync(hp.d_tok[slot], (const char *)h_tokens + (size_t)t0 * tsz, (size_t)nt * tsz,
                                cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(hp.d_off[slot], hp.h_off[slot], (size_t)(n_ext + 1) * sizeof(int64_t),
                                cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess && split)
            e = cudaMemcpyAsync(hp.d_seg[slot], hp.h_seg[slot], (size_t)(nd + 1) * sizeof(int64_t),
                                cudaMemcpyHostToDevice, st);
        const void *slice_init = nullptr;
        if (e == cudaSuccess && h_init) {
            const size_t rows = init_stride == 0 ? 1 : (size_t)nd;
            const size_t row_elems = (size_t)(init_stride ? init_stride : K);
            const char *src = (const char *)h_init + (init_stride == 0 ? 0 : (size_t)d0 * row_elems * isz);
            e = cudaMemcpyAsync(hp.d_init[slot], src, rows * row_elems * isz, cudaMemcpyHostToDevice, st);
            slice_init = hp.d_init[slot];
        }
        if (e != cudaSuccess) break;
        prm.tokens = hp.d_tok[slot];
        prm.offsets = hp.d_off[slot];
        prm.n_docs = n_ext;
        prm.n_tokens = nt;
        prm.docs_per_unit = 0;
        prm.n_peers = 0;
        prm.peer_row_offset = 0;
        CounterLease lease(perm, st);
        prm.work_counter = lease.ptr;
        if (!split) {
            prm.init = slice_init;
            prm.out = hp.d_out[slot];
            prm.out_is_u64 = out_is_u64;
            e = launch_minhash_bulk(prm, mode, token_is_u64, dev->sm_count, st);
        } else {
            prm.init = nullptr;
            prm.out = hp.d_part[slot];
            prm.out_is_u64 = 0;
            e = launch_minhash_bulk(prm, mode, token_is_u64, dev->sm_count, st);
            if (e == cudaSuccess)
                e = launch_seg_min(hp.d_part[slot], hp.d_seg[slot], nd, K, slice_init, init_stride, init_is_u64,
                                   hp.d_out[slot], out_is_u64, dev->sm_count, st);
        }
        if (e == cudaSuccess)
            e = cudaMemcpyAsync((char *)h_out + (size_t)d0 * K * osz, hp.d_out[slot], (size_t)nd * K * osz,
                                cudaMemcpyDeviceToHost, st);
    }
    for (int i = 0; i < kSlots; ++i) {
        cudaError_t e2 = cudaStreamSynchronize(hp.stream[i]);
        if (e == cudaSuccess) e = e2;
    }
    cudaSetDevice(prev);
    if (e != cudaSuccess) return cuda_fail(e, "dsk_minhash_bulk_host pipeline");
    return DSK_OK;
}

}  // extern "C"
