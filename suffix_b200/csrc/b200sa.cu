// b200sa.cu -- context, level driver and C-ABI of libb200sa.so (sm_90a).
//
// Host-side level driver for the device pipeline that replaces
// `sais_table` / `sais` (reference src/table.rs:378-574) and
// `lcp_lens_quadratic` (src/table.rs:348-361).  See DESIGN.md for the phase
// map.  No CPU fallback exists: every entry point launches CUDA kernels or
// fails with an error code.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <new>
#include <string>
#include <vector>

#include "../../include/b200sa.h"
#include "../../include/b200sa_internal.h"
#include "common.cuh"
#include "classify.cuh"
#include "classify2.cuh"
#include "classify_packed.cuh"
#include "induce.cuh"
#include "induce6.cuh"
#include "pipeline_kernels.cuh"
#include "lms_sort.cuh"
#include "shard.cuh"
#include "tree.cuh"
#include "docs.cuh"
#include "docs_tree.cuh"
#include "docs_list.cuh"
#include "docs_topk.cuh"
#include "match.cuh"
#include "repeats.cuh"
#include "lz.cuh"
#include "bwt.cuh"
#include "approx.cuh"
#include "edit.cuh"
#include "best.cuh"
#include "iupac.cuh"
#include "bulge.cuh"
#include "strand.cuh"
#include "approx_docs.cuh"
#include "align.cuh"
#include "loci.cuh"
#include "nccl_dyn.h"

using namespace b200sa;

// ---------------------------------------------------------------- context
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
};

struct b200sa_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr;
    cudaStream_t stream = nullptr;   // stream of the current call
    cudaStream_t copy_stream = nullptr;   // D2H of the SA overlapped with the LCP kernels
    cudaEvent_t ev_sa = nullptr;
    int sm_count = 0;
    int induce_blocks = 0;          // largest co-resident grid (workspace is sized for it)
    int induce_bps_max = 1;         // occupancy bound over both kernels, blocks per SM
    int induce_occ[3] = {1, 1, 1};  // occupancy bound per text packing (2, 4, 8 bits) of the default kernel
    int induce_occ_v[2][3] = {{1, 1, 1}, {1, 1, 1}};   // per kernel: [0] k_induce, [1] k_induce6 (k_induce for 4 / 8 bits)
    int induce_bps_env = 0;         // B200SA_INDUCE_BPS override (0 = adaptive)
    int cur_induce_blocks = 0;      // grid of the current build
    std::string last_error;
    bool timing = false;
    std::vector<std::pair<const char *, cudaEvent_t>> marks;
    std::vector<cudaEvent_t> event_pool;
    size_t events_used = 0;
    std::vector<const char *> phase_names;
    std::vector<float> phase_ms;
    b200sa_stats stats;
    uint32_t launches = 0;
    uint32_t *h_pin = nullptr;       // pinned read-back area (64 words)
    uint32_t *h_tab = nullptr;       // pinned copy of bstart[257] | Lcnt[256] (early SA copy-out)
    uint32_t *early_sa_out = nullptr;   // host SA buffer of the current host-API call (or null)
    bool early_done = false;
    size_t ws_bytes = 0;
    // ---- workspace
    DevBuf text, sa, lcp;                      // staging for the host API
    DevBuf pred, stype, lmsb, lmsrank, lmspos, lmslist, lmspred, sorted, flag, reduced, sa_r;
    DevBuf blkstate, carry, tables, small, scan_partial, radix_cnt, blkcnt;
    DevBuf os_hist, os_status, phik, phiv, runscr, plcp_samp;
    DevBuf k32b, k64a, k64b, v0, v1, p0, p1, g0, g1, rank, isa, qbuf;
    DevBuf packed, scan_state, cls_state, lmsdesc, steplog, hist_copies;
    DevBuf tree_out;                           // output staging of b200sa_suffix_tree
    DevBuf docs_starts, docs_out;              // doc_starts and output staging of b200sa_docs_build
    DevBuf icode;                              // approx positions with B200SA_APPROX_IUPAC: the canonical queries,
                                               // then with B200SA_APPROX_FIXED their marks
    DevBuf strand, sstage;                     // with B200SA_APPROX_BOTH_STRANDS: the doubled batch, the staged hits
    DevBuf adoff, adocs;                       // with B200SA_APPROX_DOCUMENTS: the hit offsets, the staged hits
    DevBuf aops;                               // with B200SA_APPROX_ALIGN: each hit's operations
    DevBuf abulge;                             // with B200SA_APPROX_ALIGN | _BULGES: the DP rows of a batch of hits
    DevBuf loci;                               // with B200SA_APPROX_LOCI: the locus keys, heads, marks and offsets
    uint32_t cls_calls = 0;
    // multi-GPU (SURVEY 8e): communicator owned or attached, NCCL resolved at run time
    ncclComm_t comm = nullptr;
    bool comm_owned = false;
    int nranks = 1, comm_rank = 0;
    DevBuf sh_a, sh_b, sh_c, sh_d, sh_e, sh_f, sh_small;
    bool lms_asc_ready = false;       // c->lmspos / c->lmsrank (text order) valid for the current text
    bool lms_keys_ready = false;      // k_classify_packed ran: window keys in c->reduced, their digit counts in c->os_hist
    uint32_t scan_epoch = 0, scan_tiles_cap = 0;
    uint32_t sigma = 256;            // distinct bytes of the current text
    int bits = 8;                    // bits per char of the packed text of the current call (2, 4 or 8 = raw)
    const void *ptext = nullptr;     // packed words, or the byte text when bits == 8
    uint64_t last_n = 0, last_m = 0;
};

// layout of the `tables` buffer (u32 words)
constexpr int T_BSTART = 0, T_LCNT = 257, T_SCNT = 513, T_LMSOFF = 769, T_HIST = 1026, T_CODE = 1794,
              T_ALPHA = 2050, T_END = 2306;

static const char *kVersion = "b200sa 0.1 (sm_90a)";

#define CU_TRY(ctx, expr)                                                                   \
    do {                                                                                    \
        cudaError_t e__ = (expr);                                                           \
        if (e__ != cudaSuccess) {                                                           \
            char buf__[512];                                                                \
            snprintf(buf__, sizeof buf__, "%s:%d: %s -> %s", __FILE__, __LINE__, #expr,     \
                     cudaGetErrorString(e__));                                              \
            (ctx)->last_error = buf__;                                                      \
            return (e__ == cudaErrorMemoryAllocation) ? B200SA_ERR_OOM : B200SA_ERR_CUDA;   \
        }                                                                                   \
    } while (0)

#define TRY(expr)                        \
    do {                                 \
        int rc__ = (expr);               \
        if (rc__ != B200SA_OK) return rc__; \
    } while (0)

static int ensure(b200sa_ctx *c, DevBuf &b, size_t bytes) {
    if (bytes == 0) bytes = 16;
    if (b.cap >= bytes) return B200SA_OK;
    if (b.p) { CU_TRY(c, cudaFree(b.p)); c->ws_bytes -= b.cap; b.p = nullptr; b.cap = 0; }
    size_t want = bytes + bytes / 16 + 256;    // a little slack against regrowth
    want = (want + 255) & ~(size_t)255;
    CU_TRY(c, cudaMalloc(&b.p, want));
    b.cap = want;
    c->ws_bytes += want;
    return B200SA_OK;
}
template <class T>
static T *ptr(DevBuf &b) { return reinterpret_cast<T *>(b.p); }

static inline uint32_t cdiv(uint64_t a, uint64_t b) { return (uint32_t)((a + b - 1) / b); }

static int mark(b200sa_ctx *c, const char *name) {
    if (!c->timing) return B200SA_OK;
    if (c->events_used == c->event_pool.size()) {
        cudaEvent_t e;
        CU_TRY(c, cudaEventCreate(&e));
        c->event_pool.push_back(e);
    }
    cudaEvent_t e = c->event_pool[c->events_used++];
    CU_TRY(c, cudaEventRecord(e, c->stream));
    c->marks.push_back({name, e});
    return B200SA_OK;
}
// Every argument error of an entry point leaves its own message, so that b200sa_last_error never
// reports an earlier call's failure.
static int fail(b200sa_ctx *c, int code, const char *msg) {
    c->last_error = msg;
    return code;
}
static int null_ptr(b200sa_ctx *c) { return fail(c, B200SA_ERR_BAD_ARG, "null pointer"); }
static int too_long(b200sa_ctx *c) { return fail(c, B200SA_ERR_TOO_LARGE, "text longer than 2^32-4096 bytes"); }
static int no_docs(b200sa_ctx *c) { return fail(c, B200SA_ERR_BAD_ARG, "doc_starts rejected: ndocs == 0 with n > 0;"); }

// The start of every entry point once its arguments are checked; each one then returns through leave().
static int enter(b200sa_ctx *c, void *stream) {
    CU_TRY(c, cudaSetDevice(c->device));
    c->stream = stream ? (cudaStream_t)stream : c->own_stream;
    c->marks.clear();
    c->events_used = 0;
    c->launches = 0;
    c->last_error.clear();
    return B200SA_OK;
}
// On failure, work of the call may still be in flight on its stream, writing into the caller's
// buffers, which the caller is free to release as soon as we return: wait for it, and clear the
// sticky error.  On success nothing waits beyond what the call did itself.
static int leave(b200sa_ctx *c, int rc) {
    if (rc != B200SA_OK) {
        if (c->stream) cudaStreamSynchronize(c->stream);
        cudaGetLastError();
        return rc;
    }
    c->stats.kernel_launches = c->launches;
    c->stats.workspace_bytes = c->ws_bytes;
    c->phase_names.clear();
    c->phase_ms.clear();
    if (c->timing && c->marks.size() >= 2) {
        CU_TRY(c, cudaEventSynchronize(c->marks.back().second));
        for (size_t i = 0; i + 1 < c->marks.size(); i++) {
            float ms = 0;
            CU_TRY(c, cudaEventElapsedTime(&ms, c->marks[i].second, c->marks[i + 1].second));
            c->phase_names.push_back(c->marks[i].first);
            c->phase_ms.push_back(ms);
        }
    }
    return B200SA_OK;
}

template <class... KArgs, class... Args>
static inline void launch_k(b200sa_ctx *c, void (*kern)(KArgs...), uint32_t grid, Args... args) {
    kern<<<grid, BLK, 0, c->stream>>>(args...);
    c->launches++;
}
#define LAUNCH(ctx, kern, grid, ...) launch_k((ctx), kern, (grid), __VA_ARGS__)

static int read_words(b200sa_ctx *c, const uint32_t *dsrc, int count) {
    CU_TRY(c, cudaMemcpyAsync(c->h_pin, dsrc, sizeof(uint32_t) * count, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}
// Words i and i + 1 of the last read_words as one u64 (low word first).
static uint64_t pin_u64(const b200sa_ctx *c, int i) { return c->h_pin[i] | ((uint64_t)c->h_pin[i + 1] << 32); }

// ------------------------------------------------------- generic primitives
// Single-pass scan (k_scan_lb, common.cuh): one launch, the input functor is evaluated once
// per element.  The tile descriptors live in c->scan_state and are epoch-tagged, so nothing
// is cleared between scans; a (re)allocated buffer is zeroed once (epochs start at 2).
// Scan descriptors for a kernel that embeds tile_lookback (same buffer and epochs as dev_scan).
static int scan_state_for(b200sa_ctx *c, uint32_t nb, ScanState *S) {
    size_t need = (size_t)nb * 28 + 64;
    if (c->scan_state.cap < need) {
        TRY(ensure(c, c->scan_state, need * 2));
        CU_TRY(c, cudaMemsetAsync(c->scan_state.p, 0, c->scan_state.cap, c->stream));
        c->scan_tiles_cap = (uint32_t)((c->scan_state.cap - 64) / 28);
    }
    uint8_t *basep = ptr<uint8_t>(c->scan_state);
    S->ticket = reinterpret_cast<uint32_t *>(basep);
    S->agg = reinterpret_cast<unsigned long long *>(basep + 64);
    S->incl = S->agg + c->scan_tiles_cap;
    S->pk = S->incl + c->scan_tiles_cap;
    S->flag = reinterpret_cast<uint32_t *>(S->pk + c->scan_tiles_cap);
    c->scan_epoch += 2;
    S->epoch = c->scan_epoch;
    return B200SA_OK;
}

template <class Op, class InF, class OutF>
static int dev_scan(b200sa_ctx *c, InF in, OutF out, uint64_t n, typename Op::T *d_total) {
    typedef typename Op::T T;
    if (n == 0) {
        if (d_total) CU_TRY(c, cudaMemsetAsync(d_total, 0, sizeof(T), c->stream));
        return B200SA_OK;
    }
    uint32_t nb = cdiv(n, SCAN_CHUNK);
    ScanState S;
    TRY(scan_state_for(c, nb, &S));
    LAUNCH(c, (k_scan_lb<Op, InF, OutF>), nb, in, out, n, nb, S, d_total);
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

// Grid cap of the grid-stride histogram / radix kernels: 8 blocks per SM.
static inline uint32_t grid_cap(const b200sa_ctx *c) { return (uint32_t)c->sm_count * 8u; }

template <class DigF, class MoveF>
static int radix_pass(b200sa_ctx *c, DigF dig, MoveF mv, uint64_t n) {
    if (n == 0) return B200SA_OK;
    uint32_t tiles = cdiv(n, TILE);
    uint32_t nb = tiles < grid_cap(c) ? tiles : grid_cap(c);
    uint32_t tpb = cdiv(tiles, nb);
    nb = cdiv(tiles, tpb);
    TRY(ensure(c, c->radix_cnt, (size_t)256 * nb * 4));
    uint32_t *cnt = ptr<uint32_t>(c->radix_cnt);
    LAUNCH(c, (k_radix_hist<DigF>), nb, dig, n, tpb, cnt);
    TRY((dev_scan<OpSum>(c, InArray{cnt}, OutStoreExcl{cnt}, (uint64_t)256 * nb, nullptr)));
    LAUNCH(c, (k_radix_scatter<DigF, MoveF>), nb, dig, mv, n, tpb, cnt);
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

// Keys per thread of the one-sweep passes.  From 2^20 items the tiles are wide (32 keys per thread for 32-bit
// keys, 16 for 64-bit keys, at two CTAs per SM): a fourth or half of the tiles, look-backs and per-tile scans per key.
// B200SA_SORT_ITEMS=8 forces the narrow tiles and any other value the wide ones; B200SA_SORT_NARROW the narrow.
static bool os_wide(uint64_t n) {
    if (const char *e = getenv("B200SA_SORT_ITEMS")) return atoi(e) != ITEMS;
    return n >= (1u << 20) && !getenv("B200SA_SORT_NARROW");
}

// Where the first pass of a one-sweep sort reads its keys.  IN_PLACE: from ka; a sort of no bits leaves (ka, va)
// as they are.  FROM_FUNCTORS: the histogram kernel gathers them from the key functor into kb (free until the
// second pass writes it) and the first pass writes (ka, va); at least one pass runs, so the result always lands
// in a buffer pair.  FROM_KEYS: as FROM_FUNCTORS, but a kernel before the sort has already written the keys to kb
// and the digit counts of every pass to c->os_hist (zeroed, tickets included, before that kernel): no histogram
// kernel, and keyf is not called.
enum OsFirst { IN_PLACE, FROM_FUNCTORS, FROM_KEYS };

// One one-sweep pass over `tiles` tiles of OSI * BLK items; the tile is staged in dynamic shared memory.
template <int OSI, class K, class KeyF, class ValF>
static int os_pass(b200sa_ctx *c, uint32_t tiles, KeyF keyf, ValF valf, K *kout, uint32_t *vout, uint64_t n,
                   uint32_t shift, const uint32_t *gbase, volatile unsigned long long *status, uint32_t *ticket) {
    auto kern = k_os_pass<K, KeyF, ValF, OSI>;
    constexpr size_t shm = os_stage_bytes<K, OSI>();
    CU_TRY(c, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)shm));
    kern<<<tiles, BLK, shm, c->stream>>>(keyf, valf, kout, vout, n, shift, gbase, status, ticket);
    c->launches++;
    return B200SA_OK;
}

// Sorts n items by key bits [shift0, shift0 + bits) with the one-sweep passes of common.cuh, OSI keys per
// thread.  The histogram reads the keys through keyf and the first pass the values through valf; *kout/*vout
// point at the buffer pair holding the result.
template <OsFirst FIRST, int OSI, class K, class KeyF, class ValF>
static int os_sort_items(b200sa_ctx *c, KeyF keyf, ValF valf, K *ka, uint32_t *va, K *kb, uint32_t *vb, uint64_t n,
                         int bits, uint32_t shift0, K **kout, uint32_t **vout) {
    *kout = ka;
    *vout = va;
    if (n == 0 || (FIRST == IN_PLACE && bits <= 0)) return B200SA_OK;
    int npass = (bits + 7) / 8;
    if (npass < 1) npass = 1;
    if (npass > OS_MAX_PASSES) npass = OS_MAX_PASSES;
    uint32_t tiles = cdiv(n, OSI * BLK);
    size_t status_bytes = (size_t)tiles * 256 * 8;
    TRY(ensure(c, c->os_hist, OS_MAX_PASSES * 256 * 4 + 64));
    TRY(ensure(c, c->os_status, status_bytes));
    uint32_t *ghist = ptr<uint32_t>(c->os_hist);
    uint32_t *ticket = ghist + OS_MAX_PASSES * 256;
    uint32_t hb = cdiv(n, TILE) < grid_cap(c) ? cdiv(n, TILE) : grid_cap(c);
    if (FIRST != FROM_KEYS) {
        CU_TRY(c, cudaMemsetAsync(ghist, 0, OS_MAX_PASSES * 256 * 4 + 64, c->stream));
        size_t shm = (size_t)NWARP * npass * 256 * 4;
        auto kfn = k_os_hist<K, KeyF>;
        CU_TRY(c, cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(NWARP * OS_MAX_PASSES * 256 * 4)));
        kfn<<<hb, BLK, shm, c->stream>>>(keyf, n, npass, shift0, ghist, FIRST == FROM_FUNCTORS ? kb : (K *)nullptr);
        c->launches++;
    }
    LAUNCH(c, k_os_scan, (uint32_t)npass, ghist);
    volatile unsigned long long *status = reinterpret_cast<volatile unsigned long long *>(c->os_status.p);
    if (FIRST != IN_PLACE) {            // the first pass reads the gathered keys in kb and writes (ka, va)
        std::swap(ka, kb);
        std::swap(va, vb);
    }
    for (int p = 0; p < npass; p++) {
        CU_TRY(c, cudaMemsetAsync(c->os_status.p, 0, status_bytes, c->stream));
        const uint32_t shift = shift0 + (uint32_t)(8 * p);
        if (p == 0)
            TRY(os_pass<OSI>(c, tiles, LoadArr<K>{ka}, valf, kb, vb, n, shift, ghist, status, ticket));
        else
            TRY(os_pass<OSI>(c, tiles, LoadArr<K>{ka}, LoadArr<uint32_t>{va}, kb, vb, n, shift, ghist + p * 256, status,
                             ticket + p));
        std::swap(ka, kb);
        std::swap(va, vb);
    }
    CU_TRY(c, cudaGetLastError());
    *kout = ka;
    *vout = va;
    return B200SA_OK;
}

template <OsFirst FIRST, class K, class KeyF, class ValF>
static int os_sort(b200sa_ctx *c, KeyF keyf, ValF valf, K *ka, uint32_t *va, K *kb, uint32_t *vb, uint64_t n, int bits,
                   uint32_t shift0, K **kout, uint32_t **vout) {
    if (os_wide(n))
        return os_sort_items<FIRST, sizeof(K) == 4 ? 32 : 16>(c, keyf, valf, ka, va, kb, vb, n, bits, shift0, kout, vout);
    return os_sort_items<FIRST, ITEMS>(c, keyf, valf, ka, va, kb, vb, n, bits, shift0, kout, vout);
}

// Sorts (ka, va) by the low `bits` of the key.
template <class K>
static int sort_pairs(b200sa_ctx *c, K *ka, uint32_t *va, K *kb, uint32_t *vb, uint64_t n, int bits,
                      K **kout, uint32_t **vout) {
    return os_sort<IN_PLACE>(c, LoadArr<K>{ka}, LoadArr<uint32_t>{va}, ka, va, kb, vb, n, bits, 0u, kout, vout);
}

// Sorts the items (keyf(i), valf(i)) by key bits [shift0, shift0 + bits), with (ka, va) and (kb, vb) as the
// buffer pairs.
template <class K, class KeyF, class ValF>
static int sort_pairs_from(b200sa_ctx *c, KeyF keyf, ValF valf, K *ka, uint32_t *va, K *kb, uint32_t *vb, uint64_t n,
                           int bits, K **kout, uint32_t **vout, uint32_t shift0 = 0) {
    return os_sort<FROM_FUNCTORS>(c, keyf, valf, ka, va, kb, vb, n, bits, shift0, kout, vout);
}

static int bit_length(uint64_t x) {
    int b = 0;
    while (x) { b++; x >>= 1; }
    return b;
}

// ------------------------------------------------------- reduced problem
// Refinement rounds shared by both entry paths.  On entry the na active
// suffixes (members of non-singleton groups) are listed in asuf with their SA
// slots in c->p0 and group starts in c->g0; rank[] and sa_r hold the order by
// the first h symbols.
static int doubling_rounds(b200sa_ctx *c, uint32_t m, uint32_t na, uint32_t *asuf, uint32_t *ascratch, uint64_t h,
                           uint32_t *rounds_io, const uint32_t *names_arr = nullptr, uint32_t kgram = 0,
                           uint32_t bw = 0) {
    uint32_t *sa_r = ptr<uint32_t>(c->sa_r), *rank = ptr<uint32_t>(c->rank);
    uint32_t *apos = ptr<uint32_t>(c->p0), *apos_next = ptr<uint32_t>(c->p1);
    uint32_t *G0 = ptr<uint32_t>(c->g0), *G1 = ptr<uint32_t>(c->g1), *agrp = G0;
    uint32_t *d_na = ptr<uint32_t>(c->small);
    uint32_t rounds = *rounds_io;
    if (na > 0) {
        TRY(ensure(c, c->k64a, (size_t)na * 8));
        TRY(ensure(c, c->k64b, (size_t)na * 8));
    }
    int b2 = bit_length(m);
    bool try_local = getenv("B200SA_NO_LOCAL_SORT") == nullptr;
    static const char *kSortNames[] = {"rsa_sort1", "rsa_sort2", "rsa_sort3", "rsa_sort4", "rsa_sort5", "rsa_sortN"};
    static const char *kScanNames[] = {"rsa_scan1", "rsa_scan2", "rsa_scan3", "rsa_scan4", "rsa_scan5", "rsa_scanN"};
    while (na > 0) {
        rounds++;
        { uint32_t ri = rounds - *rounds_io; TRY(mark(c, kSortNames[ri <= 5 ? ri - 1 : 5])); }
        if (rounds > 40) { c->last_error = "doubling did not converge"; return B200SA_ERR_INTERNAL; }
        uint64_t *KA = ptr<uint64_t>(c->k64a), *KB = ptr<uint64_t>(c->k64b), *K2;
        uint32_t hh = h > 0xffffffffull ? 0xffffffffu : (uint32_t)h;
        bool first = (names_arr != nullptr) && rounds == *rounds_io + 1 && kgram >= 2;
        int bits = 2 * b2;
        if (first) {     // depth 1 -> depth kgram in one sort of kgram dense names
            LAUNCH(c, (k_multi_key_list<uint64_t>), cdiv(na, BLK), names_arr, m, asuf, na, kgram, bw, KA);
            bits = (int)(kgram * bw);
        } else {
            LAUNCH(c, k_pair_keys, cdiv(na, BLK), agrp, asuf, rank, na, m, hh, (uint32_t)b2, KA);
        }
        uint32_t *Vsorted = nullptr;
        bool sorted_locally = false;
        bool use_local = !first && try_local;
        const char *how = first ? "radix(kgram)" : (try_local ? "local" : "radix(off)");   // for B200SA_TRACE
        if (use_local) {                        // probe ~4096 elements: are large groups common?
            CU_TRY(c, cudaMemsetAsync(d_na + 24, 0, 16, c->stream));   // [24] overflow, [25] large count, [26] max size
            uint32_t stride = na / 4096u; if (stride < 1) stride = 1;
            uint32_t samples = cdiv(na, stride);
            LAUNCH(c, k_group_probe, cdiv(samples, BLK), KA, na, (uint32_t)b2, stride, d_na + 25);
            TRY(read_words(c, d_na + 25, 2));
            if (c->h_pin[0] * 20u > samples) { use_local = false; how = "radix(probe)"; }   // > 5 % in big groups: this round only
        }
        if (use_local) {                        // tiny groups: rank inside the group by counting
            LAUNCH(c, k_group_local_sort, cdiv(na, BLK), KA, asuf, na, (uint32_t)b2, KB, ascratch, d_na + 24);
            TRY(read_words(c, d_na + 24, 1));
            if (c->h_pin[0] == 0) { K2 = KB; Vsorted = ascratch; sorted_locally = true; }
            else { try_local = false; how = "radix(overflow)"; }   // some group is large: radix sort from now on
        }
        if (!sorted_locally) TRY(sort_pairs<uint64_t>(c, KA, asuf, KB, ascratch, na, bits, &K2, &Vsorted));
        uint32_t *Vother = (Vsorted == asuf) ? ascratch : asuf;
        { uint32_t ri = rounds - *rounds_io; TRY(mark(c, kScanNames[ri <= 5 ? ri - 1 : 5])); }
        TRY((dev_scan<OpMaxSum>(c, InGroupActive<uint64_t>{K2, apos, na},
                                OutGroupRankCompact{Vsorted, apos, rank, sa_r, apos_next, Vother, G0}, na,
                                reinterpret_cast<unsigned long long *>(d_na + 16))));
        TRY(read_words(c, d_na + 16, 1));          // low word of the pair total = number of ambiguous suffixes
        na = c->h_pin[0];
        if (getenv("B200SA_TRACE")) fprintf(stderr, "[b200sa] doubling round %u: h=%llu -> active %u of %u, %s\n", rounds, (unsigned long long)h, na, m, how);
        asuf = Vother; ascratch = Vsorted;
        uint32_t *t = apos; apos = apos_next; apos_next = t;
        agrp = G0;
        if (first) h = kgram; else h *= 2;
    }
    *rounds_io = rounds;
    return B200SA_OK;
}


// SA of the u32 string R[0..m) (all symbols < names) -> ctx->sa_r.
// Stands in for the reference's recursion (src/table.rs:494-500): sort by
// name, then refine (group, rank[i+h]) pairs, doubling h, keeping only
// suffixes whose group is not yet a singleton.
static int reduced_sa(b200sa_ctx *c, uint32_t *R, uint32_t m, uint32_t names, uint32_t *rounds_out) {
    TRY(ensure(c, c->sa_r, (size_t)m * 4));
    TRY(ensure(c, c->k32b, (size_t)m * 4));
    TRY(ensure(c, c->v0, (size_t)m * 4));
    TRY(ensure(c, c->v1, (size_t)m * 4));
    TRY(ensure(c, c->p0, (size_t)m * 4));
    TRY(ensure(c, c->p1, (size_t)m * 4));
    TRY(ensure(c, c->g0, (size_t)m * 4));
    TRY(ensure(c, c->g1, (size_t)m * 4));
    TRY(ensure(c, c->rank, (size_t)m * 4));
    TRY(ensure(c, c->small, 256));
    uint32_t *sa_r = ptr<uint32_t>(c->sa_r), *rank = ptr<uint32_t>(c->rank);
    uint32_t *V0 = ptr<uint32_t>(c->v0), *V1 = ptr<uint32_t>(c->v1);
    uint32_t *P0 = ptr<uint32_t>(c->p0), *P1 = ptr<uint32_t>(c->p1);
    uint32_t *G0 = ptr<uint32_t>(c->g0), *G1 = ptr<uint32_t>(c->g1);
    uint32_t *d_na = ptr<uint32_t>(c->small);
    uint32_t rounds = 0;

    // round 0: sort suffixes by their first k symbols (k chosen so that the
    // key has about bit_length(m)+2 bits: random-like inputs become almost all
    // singletons after one sort; k = 1 when the alphabet is already ~m).
    LAUNCH(c, k_iota, cdiv(m, BLK), V0, m);
    int bm = bit_length(m);
    int bw = bit_length(names);               // symbols are stored +1 (0 = past the end)
    if (bw < 1) bw = 1;
    uint32_t k0 = 1;
    if (bw + 3 < bm) {
        k0 = (uint32_t)((bm + 2 + bw - 1) / bw);
        if ((int)k0 * bw > 64) k0 = 64 / bw;
    }
    if (const char *e = getenv("B200SA_K0")) { int v = atoi(e); if (v >= 1 && v * bw <= 64) k0 = (uint32_t)v; }
    if (getenv("B200SA_TRACE")) fprintf(stderr, "[b200sa] reduced_sa: m=%u names=%u k0=%u bw=%d: %s round-0 keys\n", m, names, k0, bw,
                                        (int)k0 * bw <= 32 ? "32-bit" : "64-bit");
    uint32_t *Vs;
    uint32_t na = 0;
    if ((int)k0 * bw <= 32) {
        uint32_t *KA = ptr<uint32_t>(c->k32b), *Ks;
        LAUNCH(c, (k_multi_key<uint32_t>), cdiv(m, BLK), R, m, k0, (uint32_t)bw, KA);
        // R itself is the ping-pong partner (it is dead once the keys exist)
        TRY(sort_pairs<uint32_t>(c, KA, V0, R, V1, m, (int)k0 * bw, &Ks, &Vs));
        TRY((dev_scan<OpMax>(c, InGroupStart<uint32_t>{Ks, nullptr}, OutGroupRank{Vs, nullptr, G1, rank, sa_r}, m, nullptr)));
        uint32_t *Vf = (Vs == V0) ? V1 : V0;
        TRY((dev_scan<OpSum>(c, InActive<uint32_t>{Ks, m}, OutCompactActive{nullptr, Vs, G1, P0, Vf, G0}, m, d_na)));
    } else {
        TRY(ensure(c, c->k64a, (size_t)m * 8));
        TRY(ensure(c, c->k64b, (size_t)m * 8));
        uint64_t *KA = ptr<uint64_t>(c->k64a), *KB = ptr<uint64_t>(c->k64b), *Ks;
        LAUNCH(c, (k_multi_key<uint64_t>), cdiv(m, BLK), R, m, k0, (uint32_t)bw, KA);
        TRY(sort_pairs<uint64_t>(c, KA, V0, KB, V1, m, (int)k0 * bw, &Ks, &Vs));
        TRY((dev_scan<OpMax>(c, InGroupStart<uint64_t>{Ks, nullptr}, OutGroupRank{Vs, nullptr, G1, rank, sa_r}, m, nullptr)));
        uint32_t *Vf = (Vs == V0) ? V1 : V0;
        TRY((dev_scan<OpSum>(c, InActive<uint64_t>{Ks, m}, OutCompactActive{nullptr, Vs, G1, P0, Vf, G0}, m, d_na)));
    }
    uint32_t *Vfree = (Vs == V0) ? V1 : V0;
    TRY(read_words(c, d_na, 1));
    na = c->h_pin[0];
    TRY(doubling_rounds(c, m, na, Vfree, Vs, k0, &rounds));
    if (rounds_out) *rounds_out = rounds;
    return B200SA_OK;
}

// ------------------------------------------------------- packed text
// Chooses 2 / 4 bits per char when the alphabet allows it and packs the text;
// code_of/alpha live in the tables buffer.  packed2: the classification already packed a 2-bit text.
static int pack_text(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t sigma, bool packed2 = false) {
    uint32_t *tab = ptr<uint32_t>(c->tables);
    c->bits = 8;
    c->ptext = text;
    c->sigma = sigma;
    if (getenv("B200SA_NOPACK")) return B200SA_OK;
    if (sigma <= 4) c->bits = 2; else if (sigma <= 16) c->bits = 4; else return B200SA_OK;
    uint32_t cpw = 32 / c->bits;
    uint64_t words = (n + cpw - 1) / cpw;
    TRY(ensure(c, c->packed, words * 4 + 32));  // + padding for text_bits()
    if (c->bits == 2 && !packed2)
        LAUNCH(c, (k_pack<2>), cdiv(words, BLK), text, n, tab + T_CODE, ptr<uint32_t>(c->packed), (const uint32_t *)nullptr,
               (const uint32_t *)nullptr, (const uint32_t *)nullptr, (uint32_t *)nullptr);
    else if (c->bits == 4)
        LAUNCH(c, (k_pack<4>), cdiv(words, BLK), text, n, tab + T_CODE, ptr<uint32_t>(c->packed), (const uint32_t *)nullptr,
               (const uint32_t *)nullptr, (const uint32_t *)nullptr, (uint32_t *)nullptr);
    CU_TRY(c, cudaGetLastError());
    c->ptext = c->packed.p;
    return B200SA_OK;
}

// ------------------------------------------------------- direct LMS-suffix sort
// lms_sort.cuh: radix sort of the LMS suffixes by character windows + refinement of the
// tied groups.  On success *list_out points at the LMS suffixes in suffix order (the
// seed of the final induce).  *done = false: the text has long repeats (groups stay tied);
// the caller takes the robust path (stage-1 induce, naming, rank doubling).
static uint32_t window_chars(uint32_t sigma, int bits, uint64_t *range_out) {
    if (bits == 2) { *range_out = 1ull << 32; return 16; }
    if (sigma < 2) sigma = 2;
    uint32_t cap = bits == 4 ? 13u : 8u, k = 0;
    uint64_t r = 1;
    while (k < cap && r * sigma <= (1ull << 32)) { r *= sigma; k++; }
    *range_out = r;
    return k;
}

// *done stays false: the caller takes the robust path.  B200SA_TRACE names the reason.
static int direct_hand_over(const char *why) {
    if (getenv("B200SA_TRACE")) fprintf(stderr, "[b200sa] direct LMS sort: hand over to the robust path: %s\n", why);
    return B200SA_OK;
}

template <int BITS>
static int lms_direct_sort_t(b200sa_ctx *c, uint32_t n, uint32_t m, uint32_t **list_out, bool *done) {
    *done = false;
    uint64_t range = 0;
    LmsWin W;
    W.ptext = c->ptext; W.code_of = ptr<uint32_t>(c->tables) + T_CODE; W.n = n;
    W.sigma = BITS == 2 ? 4u : c->sigma;
    W.kc = window_chars(c->sigma, BITS, &range);
    const uint32_t kc = W.kc;
    TRY(ensure(c, c->k32b, (size_t)m * 4));
    TRY(ensure(c, c->reduced, (size_t)m * 4));
    TRY(ensure(c, c->v0, (size_t)m * 4));
    TRY(ensure(c, c->v1, (size_t)m * 4));
    TRY(ensure(c, c->small, 4096));
    uint32_t *sm = ptr<uint32_t>(c->small);
    uint32_t *Ks, *Ps;
    TRY(ensure(c, c->p0, (size_t)m * 4));
    TRY(ensure(c, c->p1, (size_t)m * 4));
    TRY(ensure(c, c->g0, (size_t)m * 4));
    TRY(ensure(c, c->g1, (size_t)m * 4));
    TRY(ensure(c, c->sa_r, (size_t)m * 4));
    TRY(ensure(c, c->rank, (size_t)m * 4));
    uint32_t *slotA = ptr<uint32_t>(c->p0), *slotB = ptr<uint32_t>(c->p1);
    uint32_t *grpA = ptr<uint32_t>(c->g0), *grpB = ptr<uint32_t>(c->g1);
    uint32_t *posA = ptr<uint32_t>(c->sa_r), *posB = ptr<uint32_t>(c->rank);
    unsigned long long *d_tot = reinterpret_cast<unsigned long long *>(sm + 16);
    LmsKeyDesc<BITS> kf{W, ptr<uint32_t>(c->lmsdesc)};
    LmsValDesc vf{ptr<uint32_t>(c->lmsdesc)};
    // 2-bit text: two passes on the top 16 key bits (the first 8 characters), then k_lms_bucket_sort sorts every
    // bucket by the low 16 bits in shared memory and finds the round-1 ties with the group ids.  A bucket longer
    // than BS_CAP sends the sort back to the four full passes below.  B200SA_LMS_SORT4=1 forces those (cross-check).
    bool bucketed = false;
    if (BITS == 2 && !getenv("B200SA_LMS_SORT4")) {
        TRY(mark(c, "lms_sort"));
        // k_classify_packed wrote the keys to c->reduced and their digit counts (2-bit text is always classified
        // from its packed words here: c->lms_keys_ready)
        TRY((os_sort<FROM_KEYS>(c, kf, vf, ptr<uint32_t>(c->k32b), ptr<uint32_t>(c->v0), ptr<uint32_t>(c->reduced),
                                ptr<uint32_t>(c->v1), (uint64_t)m, 16, 16u, &Ks, &Ps)));
        TRY(mark(c, "lms_groups"));
        uint32_t *Pout = ptr<uint32_t>(c->k32b);                    // keys of the first pass: dead after the second
        CU_TRY(c, cudaMemsetAsync(sm + 16, 0, 12, c->stream));      // [16] tied count, [18] bucket overflow
        uint32_t nt = cdiv(m, BS_T);
        ScanState S;
        TRY(scan_state_for(c, nt, &S));
        CU_TRY(c, cudaFuncSetAttribute(k_lms_bucket_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BS_SMEM));
        // all of the unified L1 as shared memory: three CTAs per SM (the default carveout may leave room for one)
        CU_TRY(c, cudaFuncSetAttribute(k_lms_bucket_sort, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
        if (getenv("B200SA_TRACE")) {
            int occ = 0;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_lms_bucket_sort, BLK, BS_SMEM);
            fprintf(stderr, "[b200sa] k_lms_bucket_sort: %u CTAs, %d per SM\n", nt, occ);
        }
        k_lms_bucket_sort<<<nt, BLK, BS_SMEM, c->stream>>>(Ks, Ps, m, n, kc, nt, S, Pout, slotA, posA, grpA, sm + 16, sm + 18);
        c->launches++;
        CU_TRY(c, cudaGetLastError());
        TRY(read_words(c, sm + 16, 3));
        bucketed = c->h_pin[2] == 0;
        Ps = Pout;
        if (!bucketed && getenv("B200SA_TRACE"))
            fprintf(stderr, "[b200sa] direct LMS sort: a top-16 bucket holds more than %u suffixes: four-pass sort\n", BS_CAP);
    }
    if (!bucketed) {
        TRY(mark(c, "lms_sort"));
        TRY(sort_pairs_from(c, kf, vf, ptr<uint32_t>(c->k32b), ptr<uint32_t>(c->v0), ptr<uint32_t>(c->reduced),
                            ptr<uint32_t>(c->v1), m, bit_length(range - 1), &Ks, &Ps));
        // groups of equal windows; members of non-singleton groups -> active list
        TRY(mark(c, "lms_groups"));
        size_t fw = ((size_t)m + 31) / 32 + 1;
        TRY(ensure(c, c->flag, fw * 4));
        uint32_t *forced = ptr<uint32_t>(c->flag);
        CU_TRY(c, cudaMemsetAsync(forced, 0, fw * 4, c->stream));
        CU_TRY(c, cudaMemsetAsync(sm + 16, 0, 8, c->stream));
        LAUNCH(c, (k_lms_mark_trunc<BITS>), 1u, W, ptr<uint32_t>(c->lmsdesc), m, Ks, Ps, kc, forced);
        uint32_t nt = cdiv(m, LG_TILE);
        ScanState S;
        TRY(scan_state_for(c, nt, &S));
        LAUNCH(c, k_lms_groups1, nt, Ks, Ps, forced, m, nt, S, slotA, posA, grpA, sm + 16);
        CU_TRY(c, cudaGetLastError());
        TRY(read_words(c, sm + 16, 1));
    }
    uint32_t na = c->h_pin[0];
    c->stats.names = m - na;                       // LMS suffixes settled by the first window
    uint32_t rounds = 1;
    uint32_t max_rounds = BITS == 8 ? 16u : 8u;    // byte windows hold 4-8 chars: natural text needs ~10 of them
    if (const char *e = getenv("B200SA_DIRECT_ROUNDS")) { int v = atoi(e); if (v >= 1) max_rounds = (uint32_t)v; }
    if (getenv("B200SA_TRACE")) fprintf(stderr, "[b200sa] direct LMS sort: kc=%u, round 1 leaves %u of %u tied%s\n", kc, na, m,
                                        bucketed ? " (bucket sort)" : "");
    // the window tells (almost) nothing apart: every suffix has a twin for kc characters -- repeats, not
    // a skewed alphabet (English leaves 99.5 % tied after 5 bytes and still converges in ~10 rounds)
    if ((uint64_t)na * 1000 > (uint64_t)m * 999 && m > 64) return direct_hand_over("round1-tied");
    if (na > 0 && !bucketed)     // group id of every tied element = slot of its group's head (the bucket sort writes it)
        TRY((dev_scan<OpMax>(c, InArray{grpA}, OutMaxInPlace{grpA}, na, nullptr)));
    uint64_t h = kc;
    const bool allow_local = getenv("B200SA_NO_LOCAL_SORT") == nullptr;
    const int gbits = 32 + bit_length(m);
    while (na > 0) {
        if (rounds >= max_rounds) return direct_hand_over("round-limit");   // still tied: robust path
        rounds++;
        {
            static const char *kNames[] = {"lms_refine2", "lms_refine3", "lms_refine4", "lms_refine5", "lms_refineN"};
            TRY(mark(c, kNames[rounds - 2 < 4 ? rounds - 2 : 4]));
        }
        TRY(ensure(c, c->k64a, (size_t)na * 8));
        TRY(ensure(c, c->k64b, (size_t)na * 8));
        TRY(ensure(c, c->sorted, (size_t)m * 4));
        uint64_t *KA = ptr<uint64_t>(c->k64a), *KB = ptr<uint64_t>(c->k64b), *K2 = nullptr;
        uint32_t *scratch = ptr<uint32_t>(c->sorted), *P2 = nullptr;
        LAUNCH(c, (k_lms_refine_keys<BITS>), cdiv(na, BLK), W, posA, grpA, na, (uint32_t)h, KA);
        const uint32_t span = (uint32_t)(h + kc > 0xffffffffull ? 0xffffffffull : h + kc);
        bool local_ok = false;
        bool try_local = allow_local;
        const char *how = allow_local ? "local" : "radix(off)";      // for B200SA_TRACE
        if (try_local && na >= (1u << 20)) {    // probe ~4096 elements: counting inside a group is quadratic in its size
                                                // (a short list is cheap either way: no probe, no extra host round trip)
            CU_TRY(c, cudaMemsetAsync(sm + 24, 0, 16, c->stream));   // [24] overflow, [25] members of big groups, [26] max size
            uint32_t stride = na / 4096u; if (stride < 1) stride = 1;
            uint32_t samples = cdiv(na, stride);
            LAUNCH(c, k_group_probe, cdiv(samples, BLK), KA, na, 32u, stride, sm + 25);
            TRY(read_words(c, sm + 25, 2));
            if (c->h_pin[0] * 20u > samples) { try_local = false; how = "radix(probe)"; }   // > 5 % sit in groups of >= 128
        }
        if (try_local) {                         // tiny groups: rank inside the group by counting
            CU_TRY(c, cudaMemsetAsync(sm + 24, 0, 4, c->stream));
            LAUNCH(c, k_group_local_sort, cdiv(na, BLK), KA, posA, na, 32u, KB, scratch, sm + 24);
            TRY((dev_scan<OpMaxSum>(c, InLmsGroupR{KB, scratch, slotA, na, n, span},
                                    OutLmsCompactR{scratch, slotA, Ps, slotB, posB, grpB}, na, d_tot)));
            TRY(read_words(c, sm + 16, 9));          // [0] tied count ... [8] = sm[24] overflow flag
            local_ok = c->h_pin[8] == 0;             // some group larger than the limit: radix sort this round
            if (!local_ok) how = "radix(overflow)";
        }
        if (!local_ok) {
            TRY(sort_pairs<uint64_t>(c, KA, posA, KB, scratch, na, gbits, &K2, &P2));
            // (posA may now hold sorted values; the compaction below writes posB)
            TRY((dev_scan<OpMaxSum>(c, InLmsGroupR{K2, P2, slotA, na, n, span},
                                    OutLmsCompactR{P2, slotA, Ps, slotB, posB, grpB}, na, d_tot)));
            TRY(read_words(c, sm + 16, 1));
        }
        uint32_t na_next = c->h_pin[0];
        if (getenv("B200SA_TRACE")) fprintf(stderr, "[b200sa] direct LMS sort: round %u (h=%llu): %u -> %u tied, %s\n", rounds, (unsigned long long)h, na, na_next, how);
        // slow convergence on a large residue means long repeats: stop early
        if ((uint64_t)na_next * 100 > (uint64_t)na * 85 && (uint64_t)na_next * 64 > m) return direct_hand_over("no-convergence");
        na = na_next;
        uint32_t *t;
        t = slotA; slotA = slotB; slotB = t;
        t = posA; posA = posB; posB = t;
        t = grpA; grpA = grpB; grpB = t;
        h += kc;
    }
    c->stats.doubling_rounds = rounds;
    *list_out = Ps;
    *done = true;
    return B200SA_OK;
}
static int lms_direct_sort(b200sa_ctx *c, uint32_t n, uint32_t m, uint32_t **list_out, bool *done) {
    if (c->bits == 2) return lms_direct_sort_t<2>(c, n, m, list_out, done);
    if (c->bits == 4) return lms_direct_sort_t<4>(c, n, m, list_out, done);
    return lms_direct_sort_t<8>(c, n, m, list_out, done);
}

// ------------------------------------------------------- induce launcher
// Kernel variants of the induce passes:
//   1  k_induce: one-round steps with MATCH ranking (any packing; the default for 4-bit and byte text)
//   6  k_induce6: packed-counter ranking on physically aligned tiles + 16-bit carried chars + cascade steps for
//      short chain lists (2-bit text; default there; B200SA_NO_CASCADE / B200SA_CASCADE_MAX=<entries> switch the
//      cascade steps off / limit them)
// B200SA_INDUCE=1 forces variant 1 on 2-bit text, which also runs there when sa or lms is not 16-byte aligned.
static int induce_variant(int bits) {
    const char *e = getenv("B200SA_INDUCE");       // read per call: tests switch variants inside one process
    return (bits == 2 && !(e && atoi(e) == 1)) ? 6 : 1;
}
static const void *induce_fn_v(bool spass, int bits, int variant) {
    if (variant == 6 && bits == 2) return spass ? (const void *)k_induce6<true> : (const void *)k_induce6<false>;
    if (bits == 2) return spass ? (const void *)k_induce<true, 2> : (const void *)k_induce<false, 2>;
    if (bits == 4) return spass ? (const void *)k_induce<true, 4> : (const void *)k_induce<false, 4>;
    return spass ? (const void *)k_induce<true, 8> : (const void *)k_induce<false, 8>;
}
static int launch_induce(b200sa_ctx *c, bool spass, const uint8_t *text, uint32_t n, uint32_t *sa,
                         const uint32_t *lms, uint32_t m) {
    (void)m;
    uint32_t *tab = ptr<uint32_t>(c->tables);
    InduceArgs A;
    A.text = text; A.ptext = c->ptext; A.alpha = tab + T_ALPHA;
    A.n = n; A.sa = sa; A.pred = ptr<uint8_t>(c->pred);
    A.lms = lms; A.lms_pred = ptr<uint8_t>(c->lmspred);
    A.bstart = tab + T_BSTART; A.Lcnt = tab + T_LCNT; A.Scnt = tab + T_SCNT; A.lms_off = tab + T_LMSOFF;
    A.blk_cnt = ptr<uint32_t>(c->blkcnt);
    uint32_t *sm = ptr<uint32_t>(c->small);
    A.g_fill = sm + 64; A.g_state = reinterpret_cast<int32_t *>(sm + 320); A.err = sm + 32;
    A.run_scratch = ptr<uint32_t>(c->runscr);
    A.run_alive = A.run_scratch + TILE;
    A.cmd = sm + 336;
    A.steplog = nullptr;
    A.blocklog_step = 0;
    A.carry = 0;
    { static int rs = -1; if (rs < 0) { const char *e = getenv("B200SA_RUN_STREAK"); rs = e ? atoi(e) : 0; } A.run_streak = (uint32_t)rs; }
    if (getenv("B200SA_STEPLOG")) {
        if (ensure(c, c->steplog, 8192 * 8) == B200SA_OK) {
            A.steplog = ptr<unsigned long long>(c->steplog);
            if (const char *e = getenv("B200SA_BLOCKLOG")) {          // "<pass 0|1>:<big step index>"
                int ps = 0, st = 0;
                if (sscanf(e, "%d:%d", &ps, &st) == 2 && ps == (spass ? 1 : 0)) A.blocklog_step = (uint32_t)st + 1u;
            }
            if (!spass) cudaMemsetAsync(c->steplog.p, 0, 8, c->stream);
        }
    }
    void *args[] = {&A};
    int variant = induce_variant(c->bits);
    if (variant == 6 && (((uintptr_t)sa | (uintptr_t)lms) & 15) != 0) variant = 1;      // 16-byte loads need aligned arrays
    A.carry = variant == 6 ? 2 : 0;
    int bi = c->bits == 2 ? 0 : (c->bits == 4 ? 1 : 2);
    int blocks = c->cur_induce_blocks, cap = c->sm_count * c->induce_occ_v[variant == 6][bi];
    if (blocks > cap) blocks = cap;
    A.cascade = 0;
    if (variant == 6 && !getenv("B200SA_NO_CASCADE")) {          // multi-round steps for the short lists of every bucket's cascade
        A.cascade = (uint32_t)blocks * (uint32_t)TILE;
        if (const char *e = getenv("B200SA_CASCADE_MAX")) { long v = atol(e); if (v >= 0 && (uint64_t)v < A.cascade) A.cascade = (uint32_t)v; }
    }
    CU_TRY(c, cudaLaunchCooperativeKernel(induce_fn_v(spass, c->bits, variant), dim3(blocks), dim3(BLK), args, 0, c->stream));
    c->launches++;
    return B200SA_OK;
}

// ------------------------------------------------------- the level driver
// After the histogram is known: packed text and the grid of the persistent induce kernels.
static int post_classify(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t sigma, bool packed2 = false) {
    TRY(pack_text(c, text, n, sigma, packed2));
    // few buckets -> long lists, latency bound -> more blocks per SM; many buckets -> grid-sync bound -> one per SM
    int bps = sigma <= 16 ? 3 : (sigma <= 64 ? 2 : 1);
    if (c->induce_bps_env) bps = c->induce_bps_env;
    int occ_here = c->induce_occ[c->bits == 2 ? 0 : (c->bits == 4 ? 1 : 2)];
    if (bps > occ_here) bps = occ_here;
    if (bps < 1) bps = 1;
    c->cur_induce_blocks = c->sm_count * bps;
    return B200SA_OK;
}

// K1 fused (classify2.cuh): one pass -> type / LMS bitmaps, (byte, type) histogram, bucket
// tables, LMS positions in descending text order (c->lmsdesc), packed text.
// packed_first: the alphabet is found first (k_byte_hist -> k_alpha_from_hist, sigma on the device; see the
// sampled packing below) and a
// text of at most 4 distinct bytes is packed at 2 bits and classified from its packed words by
// k_classify_packed, which also writes the LMS sort's window keys (c->lms_keys_ready); for a larger
// alphabet those kernels return at once and k_classify_fused classifies the bytes.  The one host read after
// the classification stays the only one.  B200SA_NOPACK keeps the byte classifier on every text.
static int classify_fused_dev(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t *m_out,
                              ShardEdge edge = ShardEdge{-1, -1, ST_L}, bool pack = true, bool packed_first = false) {
    const bool try2 = packed_first && pack && !getenv("B200SA_NOPACK");
    uint64_t nw = (n + 31) / 32;
    uint32_t nbc = cdiv(nw, CLS_WORDS);
    TRY(ensure(c, c->stype, nw * 4));
    TRY(ensure(c, c->lmsb, nw * 4));
    TRY(ensure(c, c->tables, T_END * 4));
    TRY(ensure(c, c->small, 4096));
    TRY(ensure(c, c->lmsdesc, (size_t)(n / 2 + 2) * 4));
    if (c->cls_state.cap < (size_t)nbc * 4) {
        TRY(ensure(c, c->cls_state, (size_t)nbc * 8));
        CU_TRY(c, cudaMemsetAsync(c->cls_state.p, 0, c->cls_state.cap, c->stream));
    }
    uint32_t *tab = ptr<uint32_t>(c->tables), *hist = tab + T_HIST, *sm = ptr<uint32_t>(c->small);
    TRY(ensure(c, c->hist_copies, (size_t)HIST_COPIES * 768 * 4));
    CU_TRY(c, cudaMemsetAsync(c->hist_copies.p, 0, (size_t)HIST_COPIES * 768 * 4, c->stream));
    CU_TRY(c, cudaMemsetAsync(sm, 0, 4096, c->stream));
    ScanState S;
    TRY(scan_state_for(c, nbc, &S));
    Cls2State CS{ptr<uint32_t>(c->cls_state), (++c->cls_calls) * 8u};
    const uint32_t *d_sigma2 = nullptr;
    if (try2) {
        // The alphabet of the first 1 MiB codes the packing; a byte outside it sets sm[4] (d_miss), and only
        // then do the alphabet of the whole text and a second packing run, so that a text whose sample holds
        // its whole alphabet (the usual case) is read once before the classification instead of twice.
        CU_TRY(c, cudaMemsetAsync(hist, 0, 256 * 4, c->stream));
        const uint64_t ns = n < (1u << 20) ? n : (1u << 20);
        uint32_t *d_miss = sm + 4;
        d_sigma2 = sm + 3;
        auto byte_grid = [&](uint64_t len) { uint32_t g = cdiv(len, BLK * 64); return g > grid_cap(c) ? grid_cap(c) : g; };
        uint64_t pw = (n + 15) / 16;
        TRY(ensure(c, c->packed, pw * 4 + 32));
        LAUNCH(c, k_byte_hist, byte_grid(ns), text, ns, hist, (const uint32_t *)nullptr);
        LAUNCH(c, k_alpha_from_hist, 1, hist, tab + T_CODE, tab + T_ALPHA, sm + 3, (const uint32_t *)nullptr);
        LAUNCH(c, (k_pack<2>), cdiv(pw, BLK), text, n, tab + T_CODE, ptr<uint32_t>(c->packed), d_sigma2,
               (const uint32_t *)nullptr, (const uint32_t *)hist, d_miss);
        if (n > ns) {
            LAUNCH(c, k_byte_hist, byte_grid(n), text, n, hist, (const uint32_t *)d_miss);
            LAUNCH(c, k_alpha_from_hist, 1, hist, tab + T_CODE, tab + T_ALPHA, sm + 3, (const uint32_t *)d_miss);
            LAUNCH(c, (k_pack<2>), cdiv(pw, BLK), text, n, tab + T_CODE, ptr<uint32_t>(c->packed), d_sigma2,
                   (const uint32_t *)d_miss, (const uint32_t *)nullptr, (uint32_t *)nullptr);
        }
        // the window keys go where the LMS sort's key gathering would put them; the digit counts of its two
        // passes (and their tickets) are zeroed here instead of there
        TRY(ensure(c, c->reduced, (size_t)(n / 2 + 2) * 4));
        TRY(ensure(c, c->os_hist, OS_MAX_PASSES * 256 * 4 + 64));
        CU_TRY(c, cudaMemsetAsync(c->os_hist.p, 0, OS_MAX_PASSES * 256 * 4 + 64, c->stream));
        uint32_t nt2 = (uint32_t)cdiv(n, (uint64_t)CP_TILE_CHARS);
        LAUNCH(c, k_classify_packed, nt2, ptr<uint32_t>(c->packed), n, nt2, d_sigma2, tab + T_ALPHA, S, CS,
               ptr<uint32_t>(c->stype), ptr<uint32_t>(c->lmsb), ptr<uint32_t>(c->hist_copies), ptr<uint32_t>(c->lmsdesc),
               ptr<uint32_t>(c->reduced), ptr<uint32_t>(c->os_hist), sm);
    }
    LAUNCH(c, k_classify_fused, nbc, text, n, nbc, S, CS, ptr<uint32_t>(c->stype), ptr<uint32_t>(c->lmsb),
           ptr<uint32_t>(c->hist_copies), ptr<uint32_t>(c->lmsdesc), sm, edge, d_sigma2);
    LAUNCH(c, k_hist_fold, 1u, ptr<uint32_t>(c->hist_copies), hist);
    LAUNCH(c, k_bucket_tables, 1, hist, tab + T_BSTART, tab + T_LCNT, tab + T_SCNT, tab + T_LMSOFF, tab + T_CODE,
           tab + T_ALPHA, sm + 3);
    CU_TRY(c, cudaGetLastError());
    if (c->early_sa_out)
        CU_TRY(c, cudaMemcpyAsync(c->h_tab, tab + T_BSTART, 513 * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    TRY(read_words(c, sm, 4));
    uint32_t m = c->h_pin[0], sigma = c->h_pin[3];
    c->lms_keys_ready = try2 && sigma <= 4;
    if (getenv("B200SA_TRACE"))
        fprintf(stderr, "[b200sa] classify: sigma=%u, %s\n", sigma, c->lms_keys_ready ? "packed 2-bit words" : "bytes");
    if (pack) TRY(post_classify(c, text, n, sigma, c->lms_keys_ready));
    c->lms_asc_ready = false;
    *m_out = m;
    return B200SA_OK;
}

// Text-order LMS positions + per-word LMS ranks (robust path, k_unrename): derived on demand.
static int lms_ascending(b200sa_ctx *c, uint64_t n, uint32_t m) {
    if (c->lms_asc_ready) return B200SA_OK;
    uint64_t nw = (n + 31) / 32;
    TRY(ensure(c, c->lmsrank, nw * 4));
    TRY(ensure(c, c->lmspos, (size_t)m * 4));
    TRY((dev_scan<OpSum>(c, InPopcWords{ptr<uint32_t>(c->lmsb)}, OutStoreExcl{ptr<uint32_t>(c->lmsrank)}, nw, nullptr)));
    if (m > 0) LAUNCH(c, k_reverse_u32, cdiv(m, BLK), ptr<uint32_t>(c->lmsdesc), m, ptr<uint32_t>(c->lmspos));
    CU_TRY(c, cudaGetLastError());
    c->lms_asc_ready = true;
    return B200SA_OK;
}


// Host API only: the L parts of all buckets are final after the last L pass and the
// S parts after the last S pass, so the SA can start leaving over PCIe one S-pass
// early (few buckets only: one memcpy per bucket part).
static int early_copy_parts(b200sa_ctx *c, const uint32_t *d_sa, bool s_parts) {
    if (!c->early_sa_out || c->sigma > 16) return B200SA_OK;
    CU_TRY(c, cudaEventRecord(c->ev_sa, c->stream));
    CU_TRY(c, cudaStreamWaitEvent(c->copy_stream, c->ev_sa, 0));
    const uint32_t *bstart = c->h_tab, *Lcnt = c->h_tab + 257;
    for (int b = 0; b < 256; b++) {
        uint32_t lo = bstart[b] + (s_parts ? Lcnt[b] : 0u);
        uint32_t hi = s_parts ? bstart[b + 1] : bstart[b] + Lcnt[b];
        if (hi > lo)
            CU_TRY(c, cudaMemcpyAsync(c->early_sa_out + lo, d_sa + lo, (size_t)(hi - lo) * 4, cudaMemcpyDeviceToHost, c->copy_stream));
    }
    if (s_parts) c->early_done = true;
    return B200SA_OK;
}

static int build_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, uint32_t *d_sa) {
    memset(&c->stats, 0, sizeof c->stats);
    c->stats.n = n;
    c->stats.sm_count = c->sm_count;
    c->stats.induce_blocks = c->induce_blocks;   // updated after classification
    c->last_n = n; c->last_m = 0;
    if (n > B200SA_MAX_N) return too_long(c);
    if (n == 0) return B200SA_OK;
    if (n == 1) { CU_TRY(c, cudaMemsetAsync(d_sa, 0, 4, c->stream)); return B200SA_OK; }
    const uint8_t *text = d_text;
    if (((uintptr_t)d_text & 15) != 0) {       // vector loads need 16-byte alignment
        TRY(ensure(c, c->text, n));
        CU_TRY(c, cudaMemcpyAsync(c->text.p, d_text, n, cudaMemcpyDeviceToDevice, c->stream));
        text = ptr<uint8_t>(c->text);
    }
    uint32_t n32 = (uint32_t)n;
    TRY(mark(c, "classify"));
    uint32_t m = 0;
    TRY(classify_fused_dev(c, text, n, &m, ShardEdge{-1, -1, ST_L}, true, true));
    c->stats.m = m; c->last_m = m;
    c->stats.induce_blocks = c->cur_induce_blocks;
    TRY(ensure(c, c->pred, 2 * n + 64));          // bytes (variant 1) or 16-bit carried words (variant 6)
    TRY(ensure(c, c->lmslist, (size_t)m * 4));
    TRY(ensure(c, c->lmspred, 2 * (size_t)m + 64));
    TRY(ensure(c, c->blkcnt, (size_t)2 * c->induce_blocks * 256 * 4));
    TRY(ensure(c, c->runscr, (size_t)2 * TILE * 4));
    uint32_t *lmslist = ptr<uint32_t>(c->lmslist);
    bool direct_done = false;
    if (m > 0 && !getenv("B200SA_NO_DIRECT")) {
        uint32_t *lst = nullptr;
        TRY(lms_direct_sort(c, n32, m, &lst, &direct_done));
        if (direct_done) lmslist = lst;
    }
    c->stats.direct_sort = direct_done ? 1u : 0u;
    if (m > 0 && !direct_done) {
        c->stats.doubling_rounds = 0;
        TRY(lms_ascending(c, n, m));              // text-order positions + per-word ranks for the robust path
        TRY(ensure(c, c->sorted, (size_t)m * 4));
        TRY(ensure(c, c->flag, m));
        TRY(ensure(c, c->reduced, (size_t)m * 4));
        uint32_t *sm = ptr<uint32_t>(c->small);
        // K3: LMS suffixes grouped by first byte (stable, text order inside a group)
        TRY(mark(c, "lms_group"));
        TRY(radix_pass(c, DigTextAtPos{text, ptr<uint32_t>(c->lmspos)}, MoveU32{ptr<uint32_t>(c->lmspos), lmslist}, m));
        // stage 1: induced sort of the LMS substrings
        TRY(mark(c, "induce1_L"));
        TRY(launch_induce(c, false, text, n32, d_sa, lmslist, m));
        TRY(mark(c, "induce1_S"));
        TRY(launch_induce(c, true, text, n32, d_sa, lmslist, m));
        // K6: sorted LMS substrings
        TRY(mark(c, "compact_lms"));
        TRY((dev_scan<OpSum>(c, InIsLmsEntry{d_sa, ptr<uint32_t>(c->lmsb)}, OutCompactSa{d_sa, ptr<uint32_t>(c->sorted)}, n, sm + 1)));
        // K7/K8: names, reduced string
        TRY(mark(c, "name"));
        if (c->bits == 2)
            LAUNCH(c, (k_name_flags<2>), cdiv(m, BLK), c->ptext, n32, ptr<uint32_t>(c->lmsb),
                   ptr<uint32_t>(c->sorted), m, ptr<uint8_t>(c->flag));
        else if (c->bits == 4)
            LAUNCH(c, (k_name_flags<4>), cdiv(m, BLK), c->ptext, n32, ptr<uint32_t>(c->lmsb),
                   ptr<uint32_t>(c->sorted), m, ptr<uint8_t>(c->flag));
        else
            LAUNCH(c, (k_name_flags<8>), cdiv(m, BLK), c->ptext, n32, ptr<uint32_t>(c->lmsb),
                   ptr<uint32_t>(c->sorted), m, ptr<uint8_t>(c->flag));
        TRY((dev_scan<OpSum>(c, InFlagU8{ptr<uint8_t>(c->flag)},
                             OutReduced{ptr<uint32_t>(c->sorted), ptr<uint32_t>(c->lmsb), ptr<uint32_t>(c->lmsrank), ptr<uint32_t>(c->reduced)},
                             m, sm + 2)));
        TRY(read_words(c, sm + 1, 2));
        uint32_t cnt_lms = c->h_pin[0], names = c->h_pin[1];
        if (cnt_lms != m) {
            char b[160]; snprintf(b, sizeof b, "stage-1 induce lost LMS entries: %u of %u", cnt_lms, m);
            c->last_error = b; return B200SA_ERR_INTERNAL;
        }
        c->stats.names = names;
        // K8/K9 + recursion stand-in: the sorted LMS substrings already give the
        // reduced suffixes ordered by their first symbol, so doubling starts at
        // h = 1 without sorting the names again.
        TRY(mark(c, "reduced_sa"));
        TRY(ensure(c, c->sa_r, (size_t)m * 4));
        TRY(ensure(c, c->rank, (size_t)m * 4));
        TRY(ensure(c, c->g1, (size_t)m * 4));
        // first refinement: k-gram of dense names (reduced string), k = as many as fit 64 bits
        uint32_t bw = (uint32_t)bit_length(names);
        uint32_t kgram = bw ? 64u / bw : 0u;
        if (kgram > 8) kgram = 8;
        if (const char *e = getenv("B200SA_KGRAM")) { int v = atoi(e); if (v >= 0 && (uint32_t)v * bw <= 64) kgram = (uint32_t)v; }
        TRY((dev_scan<OpMax>(c, InFlagPos{ptr<uint8_t>(c->flag)},
                             OutInitFromSorted{ptr<uint32_t>(c->sorted), ptr<uint32_t>(c->lmsb), ptr<uint32_t>(c->lmsrank),
                                               ptr<uint8_t>(c->flag), m, kgram >= 2 ? 0 : 1,
                                               ptr<uint32_t>(c->sa_r), ptr<uint32_t>(c->g1), ptr<uint32_t>(c->rank)},
                             m, nullptr)));
        if (names < m) {
            TRY(ensure(c, c->v0, (size_t)m * 4));
            TRY(ensure(c, c->v1, (size_t)m * 4));
            TRY(ensure(c, c->p0, (size_t)m * 4));
            TRY(ensure(c, c->p1, (size_t)m * 4));
            TRY(ensure(c, c->g0, (size_t)m * 4));
            TRY((dev_scan<OpSum>(c, InActive<uint32_t>{ptr<uint32_t>(c->g1), m},
                                 OutCompactActive{nullptr, ptr<uint32_t>(c->sa_r), ptr<uint32_t>(c->g1),
                                                  ptr<uint32_t>(c->p0), ptr<uint32_t>(c->v0), ptr<uint32_t>(c->g0)},
                                 m, sm)));
            TRY(read_words(c, sm, 1));
            uint32_t na = c->h_pin[0], rounds = 0;
            TRY(doubling_rounds(c, m, na, ptr<uint32_t>(c->v0), ptr<uint32_t>(c->v1), 1, &rounds,
                                ptr<uint32_t>(c->reduced), kgram, bw));
            c->stats.doubling_rounds = rounds;
        }
        // K10: ranks -> text positions; the list is grouped by first byte by construction
        TRY(mark(c, "unrename"));
        LAUNCH(c, k_unrename, cdiv(m, BLK), ptr<uint32_t>(c->sa_r), ptr<uint32_t>(c->lmspos), m, lmslist);
        CU_TRY(c, cudaGetLastError());
    }
    // stage 2: final induce from the sorted LMS suffixes
    TRY(mark(c, "induce2_L"));
    TRY(launch_induce(c, false, text, n32, d_sa, lmslist, m));
    TRY(early_copy_parts(c, d_sa, false));
    TRY(mark(c, "induce2_S"));
    TRY(launch_induce(c, true, text, n32, d_sa, lmslist, m));
    TRY(early_copy_parts(c, d_sa, true));
    TRY(mark(c, "end"));
    TRY(read_words(c, ptr<uint32_t>(c->small) + 32, 4));
    if (c->h_pin[0] != 0) {
        char b[200];
        snprintf(b, sizeof b, "induce invariant violated: bucket %u filled %u, expected %u", c->h_pin[1], c->h_pin[2], c->h_pin[3]);
        c->last_error = b;
        return B200SA_ERR_INTERNAL;
    }
    return B200SA_OK;
}

static int lcp_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_sa, uint32_t *d_lcp,
                   bool reuse_pack) {
    if (n > B200SA_MAX_N) return B200SA_ERR_TOO_LARGE;
    if (n == 0) return B200SA_OK;
    uint32_t n32 = (uint32_t)n;
    TRY(ensure(c, c->isa, (size_t)n * 4));
    if (!reuse_pack) {
        // stand-alone call: the table comes from the caller (from_parts accepts anything,
        // src/table.rs:111-119, and the reference would merely panic on a bad index), and
        // every LCP kernel indexes text and phi with sa[r]: check that it is a permutation
        // of 0..n-1 before trusting it
        TRY(mark(c, "lcp_validate"));
        TRY(ensure(c, c->small, 4096));
        uint64_t nwv = (n + 31) / 32;
        uint32_t *seen = ptr<uint32_t>(c->isa);             // free until the Phi path needs it
        uint32_t *bad = ptr<uint32_t>(c->small) + 12;
        CU_TRY(c, cudaMemsetAsync(seen, 0, nwv * 4, c->stream));
        CU_TRY(c, cudaMemsetAsync(bad, 0, 4, c->stream));
        CU_TRY(c, cudaMemsetAsync(bad + 1, 0, 4, c->stream));
        LAUNCH(c, k_sa_validate, cdiv(cdiv(n, 4), BLK), d_sa, n32, seen, bad);
        LAUNCH(c, k_sa_validate_count, (uint32_t)c->sm_count * 4u, seen, n32, bad + 1);
        LAUNCH(c, k_sa_validate_verdict, 1u, bad + 1, n32, bad);
        TRY(read_words(c, bad, 1));
        if (c->h_pin[0] != 0)
            return fail(c, B200SA_ERR_BAD_ARG, "table is not a permutation of 0..n-1 (index out of range or repeated)");
    }
    if (!reuse_pack) {
        // stand-alone call: byte histogram -> alphabet -> packed text
        TRY(mark(c, "lcp_pack"));
        const uint8_t *text = d_text;
        if (((uintptr_t)d_text & 15) != 0) {
            TRY(ensure(c, c->text, n));
            CU_TRY(c, cudaMemcpyAsync(c->text.p, d_text, n, cudaMemcpyDeviceToDevice, c->stream));
            text = ptr<uint8_t>(c->text);
        }
        TRY(ensure(c, c->tables, T_END * 4));
        TRY(ensure(c, c->small, 4096));
        uint32_t *tab = ptr<uint32_t>(c->tables), *sm = ptr<uint32_t>(c->small);
        CU_TRY(c, cudaMemsetAsync(tab + T_HIST, 0, 256 * 4, c->stream));
        uint32_t hb = cdiv(n, BLK * 64);
        if (hb > grid_cap(c)) hb = grid_cap(c);
        LAUNCH(c, k_byte_hist, hb, text, n, tab + T_HIST, (const uint32_t *)nullptr);
        LAUNCH(c, k_alpha_from_hist, 1, tab + T_HIST, tab + T_CODE, tab + T_ALPHA, sm + 3, (const uint32_t *)nullptr);
        TRY(read_words(c, sm + 3, 1));
        TRY(pack_text(c, text, n, c->h_pin[0]));
    }
    // fast path: direct adjacent-pair compare when the text is L2-resident
    // (packed, or small); falls through to the linear path if any pair hits the cap
    if ((c->bits < 8 || n <= (32u << 20)) && !getenv("B200SA_LCP_LINEAR")) {
        TRY(mark(c, "lcp_direct"));
        uint32_t *sm = ptr<uint32_t>(c->small);
        TRY(ensure(c, c->small, 4096));
        sm = ptr<uint32_t>(c->small);
        CU_TRY(c, cudaMemsetAsync(sm + 8, 0, 4, c->stream));
        const uint32_t cap = 256;
        if (c->bits == 2) LAUNCH(c, k_lcp_direct<2>, cdiv(n, BLK), c->ptext, n32, d_sa, d_lcp, cap, sm + 8);
        else if (c->bits == 4) LAUNCH(c, k_lcp_direct<4>, cdiv(n, BLK), c->ptext, n32, d_sa, d_lcp, cap, sm + 8);
        else LAUNCH(c, k_lcp_direct<8>, cdiv(n, BLK), c->ptext, n32, d_sa, d_lcp, cap, sm + 8);
        TRY(read_words(c, sm + 8, 1));
        if (c->h_pin[0] == 0) {
            TRY(mark(c, "end"));
            CU_TRY(c, cudaGetLastError());
            return B200SA_OK;
        }
    }
    TRY(mark(c, "lcp_phi"));
    if (n >= (1u << 22) && !getenv("B200SA_PHI_DIRECT")) {
        // partition (sa[r], sa[r-1]) by the top byte of sa[r], then scatter window by window
        TRY(ensure(c, c->phik, (size_t)n * 4));
        TRY(ensure(c, c->phiv, (size_t)n * 4));
        TRY(ensure(c, c->os_hist, OS_MAX_PASSES * 256 * 4 + 64));
        uint32_t tiles = cdiv(n, TILE);
        size_t status_bytes = (size_t)tiles * 256 * 8;
        TRY(ensure(c, c->os_status, status_bytes));
        uint32_t *ghist = ptr<uint32_t>(c->os_hist), *ticket = ghist + OS_MAX_PASSES * 256;
        int nbits = bit_length(n - 1);
        uint32_t shift = nbits > 8 ? (uint32_t)(nbits - 8) : 0u;
        CU_TRY(c, cudaMemsetAsync(ghist, 0, OS_MAX_PASSES * 256 * 4 + 64, c->stream));
        CU_TRY(c, cudaMemsetAsync(c->os_status.p, 0, status_bytes, c->stream));
        // sa is a permutation: the digit bases are known without a histogram pass
        LAUNCH(c, k_os_perm_base, 1u, ghist, shift, n32);
        TRY(os_pass<ITEMS>(c, tiles, LoadArr<uint32_t>{d_sa}, LoadPhiPrev{d_sa}, ptr<uint32_t>(c->phik),
                           ptr<uint32_t>(c->phiv), n, shift, ghist,
                           reinterpret_cast<volatile unsigned long long *>(c->os_status.p), ticket));
        LAUNCH(c, k_phi_apply, cdiv(n, BLK), ptr<uint32_t>(c->phik), ptr<uint32_t>(c->phiv), n32, ptr<uint32_t>(c->isa));
    } else {
        LAUNCH(c, k_phi, cdiv(n, BLK), d_sa, n32, ptr<uint32_t>(c->isa));
    }
    TRY(mark(c, "lcp_plcp"));
    uint32_t nchunk = cdiv(n, LCP_CHUNK);
    uint32_t pg = cdiv(nchunk, BLK), sg = cdiv(cdiv(nchunk, 32), BLK);
    TRY(ensure(c, c->plcp_samp, (size_t)nchunk * 4));
    uint32_t *samp = ptr<uint32_t>(c->plcp_samp), *phi = ptr<uint32_t>(c->isa);
    if (c->bits == 2) LAUNCH(c, (k_plcp_samples<2>), sg, c->ptext, n32, phi, samp, (uint64_t)0, ~(uint64_t)0);
    else if (c->bits == 4) LAUNCH(c, (k_plcp_samples<4>), sg, c->ptext, n32, phi, samp, (uint64_t)0, ~(uint64_t)0);
    else LAUNCH(c, (k_plcp_samples<8>), sg, c->ptext, n32, phi, samp, (uint64_t)0, ~(uint64_t)0);
    TRY(mark(c, "lcp_plcp_fill"));
    if (c->bits == 2) LAUNCH(c, (k_plcp<2>), pg, c->ptext, n32, phi, samp, (uint64_t)0, ~(uint64_t)0);
    else if (c->bits == 4) LAUNCH(c, (k_plcp<4>), pg, c->ptext, n32, phi, samp, (uint64_t)0, ~(uint64_t)0);
    else LAUNCH(c, (k_plcp<8>), pg, c->ptext, n32, phi, samp, (uint64_t)0, ~(uint64_t)0);
    TRY(mark(c, "lcp_gather"));
    LAUNCH(c, k_lcp_gather, cdiv(n, BLK), d_sa, ptr<uint32_t>(c->isa), n32, d_lcp);
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

template <class K>
static int test_sort_core(b200sa_ctx *c, K *keys, uint32_t *vals, uint64_t n, int bits) {
    TRY(ensure(c, c->k64a, n * sizeof(K)));
    TRY(ensure(c, c->k64b, n * sizeof(K)));
    TRY(ensure(c, c->v0, n * 4));
    TRY(ensure(c, c->v1, n * 4));
    CU_TRY(c, cudaMemcpyAsync(c->k64a.p, keys, n * sizeof(K), cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(c->v0.p, vals, n * 4, cudaMemcpyHostToDevice, c->stream));
    K *ko; uint32_t *vo;
    TRY(sort_pairs<K>(c, ptr<K>(c->k64a), ptr<uint32_t>(c->v0), ptr<K>(c->k64b), ptr<uint32_t>(c->v1), n, bits, &ko, &vo));
    if (n) {
        CU_TRY(c, cudaMemcpyAsync(keys, ko, n * sizeof(K), cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaMemcpyAsync(vals, vo, n * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

template <class K>
static int test_sort(b200sa_ctx *c, K *keys, uint32_t *vals, uint64_t n, int bits) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!keys || !vals)) return null_ptr(c);
    TRY(enter(c, nullptr));
    return leave(c, test_sort_core(c, keys, vals, n, bits));
}

// SA + LCP of one text, device-resident (b200sa_build_lcp_dev, and step 1 of b200sa_docs_build).
static int build_lcp_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, uint32_t *d_sa, uint32_t *d_lcp) {
    int rc = build_dev(c, d_text, n, d_sa);
    if (rc == B200SA_OK) {
        // build_dev may have classified an aligned copy of the text; the packed text (or that
        // copy) is still valid, so the LCP kernels reuse it (n >= 2 means classification ran)
        const uint8_t *t = (((uintptr_t)d_text & 15) != 0 && n >= 2) ? ptr<uint8_t>(c->text) : d_text;
        b200sa_stats st = c->stats;
        rc = lcp_dev(c, t, n, d_sa, d_lcp, n >= 2);
        c->stats = st;
    }
    return rc;
}

// ================================================================= C ABI
// include/b200sa.h and include/b200sa_internal.h give every entry point C linkage, which the
// definitions below keep.

const char *b200sa_version(void) { return kVersion; }

const char *b200sa_strerror(int code) {
    switch (code) {
        case B200SA_OK: return "ok";
        case B200SA_ERR_BAD_ARG: return "bad argument";
        case B200SA_ERR_TOO_LARGE: return "text longer than B200SA_MAX_N = 2^32-4096 bytes";
        case B200SA_ERR_NO_DEVICE: return "no usable CUDA device";
        case B200SA_ERR_OOM: return "out of device memory";
        case B200SA_ERR_CUDA: return "CUDA error";
        case B200SA_ERR_INTERNAL: return "internal invariant violated";
        default: return "unknown error";
    }
}

const char *b200sa_last_error(b200sa_ctx *ctx) { return ctx ? ctx->last_error.c_str() : "null context"; }

int b200sa_ctx_create(int device, b200sa_ctx **out) {
    if (!out) return B200SA_ERR_BAD_ARG;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return B200SA_ERR_NO_DEVICE;
    if (device < 0 || device >= count) return B200SA_ERR_BAD_ARG;
    if (cudaSetDevice(device) != cudaSuccess) return B200SA_ERR_NO_DEVICE;
    b200sa_ctx *c = new b200sa_ctx();
    c->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete c; return B200SA_ERR_CUDA; }
    if (prop.major != 9 || prop.minor != 0) { delete c; return B200SA_ERR_NO_DEVICE; }   // sm_90a code: H100 class only
    c->sm_count = prop.multiProcessorCount;
    if (!prop.cooperativeLaunch) { delete c; return B200SA_ERR_NO_DEVICE; }
    if (cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking) != cudaSuccess) { delete c; return B200SA_ERR_CUDA; }
    c->stream = c->own_stream;
    if (cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_sa, cudaEventDisableTiming) != cudaSuccess) { delete c; return B200SA_ERR_CUDA; }
    if (cudaMallocHost((void **)&c->h_pin, 64 * sizeof(uint32_t)) != cudaSuccess) { delete c; return B200SA_ERR_CUDA; }
    if (cudaMallocHost((void **)&c->h_tab, 513 * sizeof(uint32_t)) != cudaSuccess) { cudaFreeHost(c->h_pin); delete c; return B200SA_ERR_CUDA; }
    int occ = 0;
    {
        const int bb[3] = {2, 4, 8};
        for (int v = 0; v < 2; v++)
            for (int k = 0; k < 3; k++) {
                int ok = 1 << 30;
                for (int sp = 0; sp < 2; sp++) {
                    int o = 0;
                    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, induce_fn_v(sp != 0, bb[k], v ? 6 : 1), BLK, 0);
                    if (o < ok) ok = o;
                }
                c->induce_occ_v[v][k] = ok > 4 ? 4 : ok;
            }
        for (int k = 0; k < 3; k++) {
            c->induce_occ[k] = c->induce_occ_v[induce_variant(bb[k]) == 6][k];
            for (int v = 0; v < 2; v++) if (c->induce_occ_v[v][k] > occ) occ = c->induce_occ_v[v][k];
        }
    }
    if (occ < 1) { cudaFreeHost(c->h_pin); delete c; return B200SA_ERR_CUDA; }
    c->induce_bps_max = occ > 4 ? 4 : occ;
    if (const char *e = getenv("B200SA_INDUCE_BPS")) { int v = atoi(e); if (v >= 1) c->induce_bps_env = v > occ ? occ : v; }
    c->induce_blocks = c->sm_count * c->induce_bps_max;
    c->cur_induce_blocks = c->sm_count;
    memset(&c->stats, 0, sizeof c->stats);
    *out = c;
    return B200SA_OK;
}

void b200sa_ctx_destroy(b200sa_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->comm && c->comm_owned && nccl_api().ok) nccl_api().CommDestroy(c->comm);
    DevBuf *bufs[] = {&c->text, &c->sa, &c->lcp, &c->pred, &c->stype, &c->lmsb, &c->lmsrank, &c->lmspos, &c->lmslist,
                      &c->lmspred, &c->sorted, &c->flag, &c->reduced, &c->sa_r, &c->blkstate, &c->carry, &c->tables,
                      &c->small, &c->scan_partial, &c->radix_cnt, &c->blkcnt, &c->k32b, &c->k64a, &c->k64b, &c->v0,
                      &c->v1, &c->p0, &c->p1, &c->g0, &c->g1, &c->rank, &c->isa, &c->qbuf, &c->os_hist, &c->os_status, &c->packed, &c->phik, &c->phiv, &c->runscr, &c->plcp_samp, &c->scan_state, &c->cls_state, &c->lmsdesc, &c->steplog, &c->hist_copies, &c->tree_out, &c->docs_starts, &c->docs_out, &c->icode, &c->strand, &c->sstage, &c->adoff, &c->adocs, &c->aops, &c->abulge, &c->loci, &c->sh_a, &c->sh_b, &c->sh_c, &c->sh_d, &c->sh_e, &c->sh_f, &c->sh_small};
    for (DevBuf *b : bufs) if (b->p) cudaFree(b->p);
    for (cudaEvent_t e : c->event_pool) cudaEventDestroy(e);
    if (c->h_pin) cudaFreeHost(c->h_pin);
    if (c->h_tab) cudaFreeHost(c->h_tab);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    if (c->ev_sa) cudaEventDestroy(c->ev_sa);
    delete c;
}

int b200sa_set_timing(b200sa_ctx *c, int enabled) {
    if (!c) return B200SA_ERR_BAD_ARG;
    c->timing = enabled != 0;
    return B200SA_OK;
}

int b200sa_last_phase_times(b200sa_ctx *c, const char **names, float *ms, int cap) {
    if (!c) return B200SA_ERR_BAD_ARG;
    int k = (int)c->phase_names.size();
    for (int i = 0; i < k && i < cap; i++) {
        if (names) names[i] = c->phase_names[i];
        if (ms) ms[i] = c->phase_ms[i];
    }
    return k;
}

int b200sa_last_stats(b200sa_ctx *c, b200sa_stats *out) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!out) return null_ptr(c);
    *out = c->stats;
    out->workspace_bytes = c->ws_bytes;
    return B200SA_OK;
}

int b200sa_build_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, uint32_t *d_sa, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!d_text || !d_sa)) return null_ptr(c);
    TRY(enter(c, stream));
    return leave(c, build_dev(c, d_text, n, d_sa));
}

int b200sa_lcp_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_sa, uint32_t *d_lcp,
                   void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!d_text || !d_sa || !d_lcp)) return null_ptr(c);
    TRY(enter(c, stream));
    return leave(c, lcp_dev(c, d_text, n, d_sa, d_lcp, false));
}

int b200sa_build_lcp_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, uint32_t *d_sa, uint32_t *d_lcp,
                         void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!d_text || !d_sa || !d_lcp)) return null_ptr(c);
    TRY(enter(c, stream));
    return leave(c, build_lcp_dev(c, d_text, n, d_sa, d_lcp));
}

static int host_build_inner(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t *sa_out, uint32_t *lcp_out,
                            const uint32_t *sa_in) {
    memset(&c->stats, 0, sizeof c->stats);
    c->stats.n = n;
    if (n == 0) return B200SA_OK;
    TRY(ensure(c, c->text, n));
    TRY(ensure(c, c->sa, (size_t)n * 4));
    TRY(mark(c, "h2d"));
    CU_TRY(c, cudaMemcpyAsync(c->text.p, text, n, cudaMemcpyHostToDevice, c->stream));
    if (sa_in) CU_TRY(c, cudaMemcpyAsync(c->sa.p, sa_in, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    if (!sa_in) {
        // early copy-out only into pinned memory: a D2H into pageable memory blocks the host
        // thread, which would delay the launch of the last S pass
        bool pinned = false;
        if (sa_out) {
            cudaPointerAttributes pa;
            if (cudaPointerGetAttributes(&pa, sa_out) == cudaSuccess) pinned = (pa.type == cudaMemoryTypeHost);
            else cudaGetLastError();
        }
        c->early_sa_out = (pinned && n >= 2) ? sa_out : nullptr;
        c->early_done = false;
        int brc = build_dev(c, ptr<uint8_t>(c->text), n, ptr<uint32_t>(c->sa));
        c->early_sa_out = nullptr;
        if (brc != B200SA_OK) return brc;
        if (sa_out && c->early_done) {
            TRY(mark(c, "d2h_sa"));      // already on its way on the copy stream
        } else if (sa_out) {
            TRY(mark(c, "d2h_sa"));
            if (lcp_out) {      // the LCP kernels only read the SA: copy it out underneath them
                CU_TRY(c, cudaEventRecord(c->ev_sa, c->stream));
                CU_TRY(c, cudaStreamWaitEvent(c->copy_stream, c->ev_sa, 0));
                CU_TRY(c, cudaMemcpyAsync(sa_out, c->sa.p, (size_t)n * 4, cudaMemcpyDeviceToHost, c->copy_stream));
            } else {
                CU_TRY(c, cudaMemcpyAsync(sa_out, c->sa.p, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
            }
        }
    }
    if (lcp_out) {
        TRY(ensure(c, c->lcp, (size_t)n * 4));
        TRY(lcp_dev(c, ptr<uint8_t>(c->text), n, ptr<uint32_t>(c->sa), ptr<uint32_t>(c->lcp), sa_in == nullptr && n >= 2));
        TRY(mark(c, "d2h_lcp"));
        CU_TRY(c, cudaMemcpyAsync(lcp_out, c->lcp.p, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    TRY(mark(c, "end"));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->copy_stream));
    return B200SA_OK;
}

// The host API: a failed build may also have D2H copies into the caller's buffers in flight on
// the copy stream.
static int host_build(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t *sa_out, uint32_t *lcp_out,
                      const uint32_t *sa_in) {
    if (n > B200SA_MAX_N) return too_long(c);
    TRY(enter(c, nullptr));
    int rc = host_build_inner(c, text, n, sa_out, lcp_out, sa_in);
    if (rc != B200SA_OK) {
        c->early_sa_out = nullptr;
        if (c->copy_stream) cudaStreamSynchronize(c->copy_stream);
    }
    return leave(c, rc);
}

int b200sa_build(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t *sa_out) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!text || !sa_out)) return null_ptr(c);
    return host_build(c, text, n, sa_out, nullptr, nullptr);
}

int b200sa_lcp(b200sa_ctx *c, const uint8_t *text, uint64_t n, const uint32_t *sa, uint32_t *lcp_out) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!text || !sa || !lcp_out)) return null_ptr(c);
    return host_build(c, text, n, nullptr, lcp_out, sa);
}

int b200sa_build_lcp(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t *sa_out, uint32_t *lcp_out) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!text || !sa_out || !lcp_out)) return null_ptr(c);
    return host_build(c, text, n, sa_out, lcp_out, nullptr);
}

static int positions_core(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_sa,
                          const uint8_t *d_queries, const uint64_t *d_q_off, uint32_t nq, uint32_t *d_start,
                          uint32_t *d_end) {
    if (nq > 0) {
        LAUNCH(c, k_positions<TextEnd>, cdiv(nq, BLK), d_text, (uint32_t)n, d_sa, d_queries, d_q_off, nq, d_start, d_end,
               TextEnd{(uint32_t)n});
        CU_TRY(c, cudaGetLastError());
    }
    return B200SA_OK;
}

int b200sa_positions_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_sa,
                         const uint8_t *d_queries, const uint64_t *d_q_off, uint32_t nq, uint32_t *d_start,
                         uint32_t *d_end, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if ((nq > 0 && (!d_q_off || !d_start || !d_end)) || (n > 0 && (!d_text || !d_sa))) return null_ptr(c);
    if (n > B200SA_MAX_N) return too_long(c);
    TRY(enter(c, stream));
    return leave(c, positions_core(c, d_text, n, d_sa, d_queries, d_q_off, nq, d_start, d_end));
}

// ------------------------------------------------------------ multi-GPU shards (SURVEY 8e)
// The checks of both shard entry points on the shard and the next character.
static int shard_args(b200sa_ctx *c, const uint8_t *d_shard, uint64_t len, int next_char) {
    if (!d_shard) return null_ptr(c);
    if (len < 1 || len > B200SA_MAX_N) return fail(c, B200SA_ERR_BAD_ARG, "shard: len must be in [1, 2^32-4096]");
    if (next_char > 255) return fail(c, B200SA_ERR_BAD_ARG, "shard: next_char above 255");
    if (((uintptr_t)d_shard & 15) != 0) return fail(c, B200SA_ERR_BAD_ARG, "shard pointer must be 16-byte aligned");
    return B200SA_OK;
}

static int shard_summary_core(b200sa_ctx *c, const uint8_t *d_shard, uint64_t len, int next_char, int *state_out) {
    uint64_t nw = (len + 31) / 32;
    uint32_t nbc = cdiv(nw, CLS_WORDS);
    TRY(ensure(c, c->blkstate, nbc));
    TRY(ensure(c, c->carry, nbc));
    TRY(ensure(c, c->small, 4096));
    ShardEdge edge{next_char, -1, ST_P};
    LAUNCH(c, k_cls_block_state, nbc, d_shard, len, ptr<uint8_t>(c->blkstate), edge);
    LAUNCH(c, k_cls_carry, 1, ptr<uint8_t>(c->blkstate), nbc, ptr<uint8_t>(c->carry), (uint32_t)ST_P);
    CU_TRY(c, cudaGetLastError());
    uint8_t h[2];
    CU_TRY(c, cudaMemcpyAsync(&h[0], c->blkstate.p, 1, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaMemcpyAsync(&h[1], c->carry.p, 1, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    *state_out = (h[0] != ST_P) ? h[0] : h[1];
    return B200SA_OK;
}

int b200sa_shard_summary(b200sa_ctx *c, const uint8_t *d_shard, uint64_t len, int next_char, int *state_out, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!state_out) return null_ptr(c);
    TRY(shard_args(c, d_shard, len, next_char));
    TRY(enter(c, stream));
    return leave(c, shard_summary_core(c, d_shard, len, next_char, state_out));
}

static int shard_classify_core(b200sa_ctx *c, const uint8_t *d_shard, uint64_t len, int prev_char, int next_char,
                               int tail_carry, uint32_t *d_stype_words, uint32_t *d_lms_words, uint32_t *d_lmspos,
                               uint64_t cap_lms, uint64_t *hist768, uint64_t *m_out) {
    uint32_t m = 0;
    ShardEdge edge{next_char, prev_char, next_char >= 0 ? (uint32_t)tail_carry : ST_L};
    TRY(classify_fused_dev(c, d_shard, len, &m, edge, /*pack=*/false));
    TRY(lms_ascending(c, len, m));                // text-order LMS positions from the descending list
    uint64_t nw = (len + 31) / 32;
    if (d_stype_words) CU_TRY(c, cudaMemcpyAsync(d_stype_words, c->stype.p, nw * 4, cudaMemcpyDeviceToDevice, c->stream));
    if (d_lms_words) CU_TRY(c, cudaMemcpyAsync(d_lms_words, c->lmsb.p, nw * 4, cudaMemcpyDeviceToDevice, c->stream));
    if (d_lmspos && m > 0) {
        uint64_t k = m < cap_lms ? m : cap_lms;
        CU_TRY(c, cudaMemcpyAsync(d_lmspos, c->lmspos.p, k * 4, cudaMemcpyDeviceToDevice, c->stream));
    }
    if (hist768) {
        uint32_t h32[768];
        CU_TRY(c, cudaMemcpyAsync(h32, ptr<uint32_t>(c->tables) + T_HIST, sizeof h32, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaStreamSynchronize(c->stream));
        for (int i = 0; i < 768; i++) hist768[i] = h32[i];
    } else {
        CU_TRY(c, cudaStreamSynchronize(c->stream));
    }
    if (m_out) *m_out = m;
    return B200SA_OK;
}

int b200sa_shard_classify(b200sa_ctx *c, const uint8_t *d_shard, uint64_t len, int prev_char, int next_char,
                          int tail_carry, uint32_t *d_stype_words, uint32_t *d_lms_words, uint32_t *d_lmspos,
                          uint64_t cap_lms, uint64_t *hist768, uint64_t *m_out, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (prev_char > 255) return fail(c, B200SA_ERR_BAD_ARG, "shard: prev_char above 255");
    TRY(shard_args(c, d_shard, len, next_char));
    if (next_char >= 0 && tail_carry != (int)ST_L && tail_carry != (int)ST_S)
        return fail(c, B200SA_ERR_BAD_ARG, "shard: tail_carry must be L or S when next_char >= 0");
    TRY(enter(c, stream));
    return leave(c, shard_classify_core(c, d_shard, len, prev_char, next_char, tail_carry, d_stype_words, d_lms_words,
                                        d_lmspos, cap_lms, hist768, m_out));
}

// ------------------------------------------------------------ generalized SA / LCP intervals (SURVEY 8f-3, 8f-4)
static int doc_ids_core(b200sa_ctx *c, const uint32_t *d_pos, uint64_t count, const uint32_t *d_doc_starts,
                        uint32_t ndocs, uint32_t *d_doc, uint32_t *d_off) {
    if (count) LAUNCH(c, k_doc_ids, cdiv(count, BLK), d_pos, count, d_doc_starts, ndocs, d_doc, d_off);
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

int b200sa_doc_ids_dev(b200sa_ctx *c, const uint32_t *d_pos, uint64_t count, const uint32_t *d_doc_starts,
                       uint32_t ndocs, uint32_t *d_doc, uint32_t *d_off, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!d_doc_starts || (count > 0 && (!d_pos || !d_doc || !d_off))) return null_ptr(c);
    if (ndocs < 1) return fail(c, B200SA_ERR_BAD_ARG, "doc ids: ndocs must be at least 1");
    TRY(enter(c, stream));
    return leave(c, doc_ids_core(c, d_pos, count, d_doc_starts, ndocs, d_doc, d_off));
}

// Block minima of an array (the LCP array, or any other) over 32^k entries, in `buf`, for the ANSV searches.
static int ansv_levels(b200sa_ctx *c, const uint32_t *d_lcp, uint64_t n, AnsvLevels *L, DevBuf &buf) {
    memset(L, 0, sizeof *L);
    L->lv[0] = d_lcp; L->cnt[0] = n; L->nlev = 1;
    uint64_t total = 0;
    for (uint64_t k = (n + 31) / 32; ; k = (k + 31) / 32) { total += k; if (k <= 32) break; }
    TRY(ensure(c, buf, (total + 64) * 4));
    uint32_t *lvbuf = ptr<uint32_t>(buf);
    uint64_t cnt = n;
    while (cnt > 32 && L->nlev < 8) {
        uint64_t nxt = (cnt + 31) / 32;
        LAUNCH(c, k_min32, cdiv(nxt, BLK), L->lv[L->nlev - 1], cnt, lvbuf);
        L->lv[L->nlev] = lvbuf; L->cnt[L->nlev] = nxt; L->nlev++;
        lvbuf += nxt;
        cnt = nxt;
    }
    return B200SA_OK;
}

static int lcp_intervals_core(b200sa_ctx *c, const uint32_t *d_lcp, uint64_t n, uint32_t *d_psv, uint32_t *d_nsv) {
    if (n == 0) return B200SA_OK;
    AnsvLevels L;
    TRY(ansv_levels(c, d_lcp, n, &L, c->qbuf));
    LAUNCH(c, k_ansv, cdiv(n, BLK), L, n, d_psv, d_nsv);
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

int b200sa_lcp_intervals_dev(b200sa_ctx *c, const uint32_t *d_lcp, uint64_t n, uint32_t *d_psv, uint32_t *d_nsv,
                             void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!d_lcp || !d_psv || !d_nsv)) return null_ptr(c);
    if (n > B200SA_MAX_N) return too_long(c);
    TRY(enter(c, stream));
    return leave(c, lcp_intervals_core(c, d_lcp, n, d_psv, d_nsv));
}

// ------------------------------------------------------------ suffix tree from SA + LCP (SURVEY 8f-5)
static int tree_bad(b200sa_ctx *c, uint32_t bits) {
    std::string m = "suffix tree input rejected:";
    if (bits & TREE_BAD_SA) m += " sa[r] >= n;";
    if (bits & TREE_BAD_LCP0) m += " lcp[0] != 0;";
    if (bits & TREE_BAD_LCP) m += " lcp[r] longer than suffix sa[r-1] or sa[r];";
    if (bits & TREE_BAD_PARENT) m += " a parent node is missing (lcp is not the LCP array of sa);";
    if (bits & TREE_BAD_FIRST) m += " a rank starts no node (lcp is not the LCP array of sa);";
    if (bits & TREE_BAD_NODE) m += " the node of a document string is missing (glcp is not the LCP array of G);";
    c->last_error = m;
    return B200SA_ERR_BAD_ARG;
}

// n >= 1, device inputs and outputs (capacity >= 2n each).  Phases: tree_ansv, tree_emit, tree_sort,
// tree_first, tree_nodes.  len gives the suffix length of a rank (TextLen: one text; DocsLen: the
// generalized tree, whose sorted keys and first[] b200sa_docs_tree reads afterwards in k64a/k64b and g0).
template <class LenF>
static int suffix_tree_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_sa, const uint32_t *d_lcp, const TreeOut &o,
                            uint64_t *num_nodes, LenF len, uint64_t **keys_out = nullptr) {
    const uint64_t cap = 2 * (uint64_t)n;
    const int B = bit_length(n);                       // depth <= n and sa_lo < n both fit in B bits
    TRY(ensure(c, c->p0, (size_t)n * 4));
    TRY(ensure(c, c->p1, (size_t)n * 4));
    TRY(ensure(c, c->flag, n));
    TRY(ensure(c, c->g0, ((size_t)n + 1) * 4));
    TRY(ensure(c, c->k64a, cap * 8));
    TRY(ensure(c, c->k64b, cap * 8));
    TRY(ensure(c, c->v0, cap * 4));
    TRY(ensure(c, c->v1, cap * 4));
    TRY(ensure(c, c->small, 4096));
    uint32_t *psv = ptr<uint32_t>(c->p0), *nsv = ptr<uint32_t>(c->p1), *first = ptr<uint32_t>(c->g0);
    uint8_t *rep = ptr<uint8_t>(c->flag);
    uint32_t *words = ptr<uint32_t>(c->small);          // [0] nodes below the root, [1] check bits
    TRY(mark(c, "tree_ansv"));
    AnsvLevels L;
    TRY(ansv_levels(c, d_lcp, n, &L, c->qbuf));
    LAUNCH(c, k_tree_ansv, cdiv(n, BLK), L, (uint64_t)n, psv, nsv, rep);
    TRY(mark(c, "tree_emit"));
    CU_TRY(c, cudaMemsetAsync(words, 0, 8, c->stream));
    TreeCount<LenF> tin{len, d_sa, d_lcp, rep, n, words + 1};
    TreeEmit<LenF> tout{len, d_sa, d_lcp, psv, nsv, rep, n, B, ptr<uint64_t>(c->k64a), ptr<uint32_t>(c->v0)};
    TRY((dev_scan<OpSum>(c, tin, tout, n, words)));
    TRY(read_words(c, words, 2));
    if (c->h_pin[1]) return tree_bad(c, c->h_pin[1]);
    const uint32_t N = c->h_pin[0] + 1;
    TRY(mark(c, "tree_sort"));
    uint64_t *K;
    uint32_t *V;
    TRY(sort_pairs<uint64_t>(c, ptr<uint64_t>(c->k64a), ptr<uint32_t>(c->v0), ptr<uint64_t>(c->k64b),
                             ptr<uint32_t>(c->v1), N, 2 * B, &K, &V));
    TRY(mark(c, "tree_first"));
    if (LenF::DOCS) {
        CU_TRY(c, cudaMemsetAsync(first, 0, ((size_t)n + 1) * 4, c->stream));
        LAUNCH(c, k_tree_last, cdiv(N, BLK), K, N, B, first);
        TRY((dev_scan<OpMax>(c, InArray{first}, OutStoreExcl{first}, (uint64_t)n + 1, nullptr)));
    } else {
        CU_TRY(c, cudaMemsetAsync(first, 0xff, ((size_t)n + 1) * 4, c->stream));
        LAUNCH(c, k_tree_first, cdiv(N, BLK), K, N, B, n, first);
    }
    TRY(mark(c, "tree_nodes"));
    uint32_t grid_n = N > n + 1 ? N : n + 1;
    LAUNCH(c, k_tree_nodes, cdiv(grid_n, BLK), K, V, N, B, d_sa, d_lcp, psv, first, n, o, words + 1);
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    TRY(read_words(c, words + 1, 1));
    if (c->h_pin[0]) return tree_bad(c, c->h_pin[0]);
    *num_nodes = N;
    if (keys_out) *keys_out = K;
    return B200SA_OK;
}

static int tree_args(b200sa_ctx *c, uint64_t n, const void *sa, const void *lcp, const b200sa_tree *out,
                     uint64_t cap, uint64_t *num_nodes) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!out || !num_nodes || !out->parent || !out->depth || !out->sa_lo || !out->sa_hi || !out->label_start ||
        !out->subtree_end || (n > 0 && (!sa || !lcp)))
        return null_ptr(c);
    if (n > B200SA_TREE_MAX_N)
        return fail(c, B200SA_ERR_TOO_LARGE, "suffix tree: n >= 2^31 (node ids are u32 with 0xFFFFFFFF reserved)");
    if (cap < (n ? 2 * n : 1)) return fail(c, B200SA_ERR_BAD_ARG, "suffix tree: cap < max(1, 2n)");
    return B200SA_OK;
}

// The root alone, in the first entry of the device arrays dst[0, count): its values in root.
static int root_dev(b200sa_ctx *c, uint32_t *const *dst, const uint32_t *root, int count, uint64_t *num_nodes) {
    for (int k = 0; k < count; k++) {
        cudaError_t e = cudaMemcpyAsync(dst[k], &root[k], 4, cudaMemcpyHostToDevice, c->stream);
        if (e != cudaSuccess) return fail(c, B200SA_ERR_CUDA, cudaGetErrorString(e));
    }
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    *num_nodes = 1;
    return B200SA_OK;
}

static int suffix_tree_dev_core(b200sa_ctx *c, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp,
                                const b200sa_tree *out, uint64_t *num_nodes) {
    if (n == 0) {
        // the root alone: parent none, depth 0, range [0, 0), empty label, subtree [0, 1)
        const uint32_t root[6] = {TREE_NONE, 0, 0, 0, 0, 1};
        uint32_t *dst[6] = {out->parent, out->depth, out->sa_lo, out->sa_hi, out->label_start, out->subtree_end};
        return root_dev(c, dst, root, 6, num_nodes);
    }
    TreeOut o{out->parent, out->depth, out->sa_lo, out->sa_hi, out->label_start, out->subtree_end};
    return suffix_tree_core(c, (uint32_t)n, d_sa, d_lcp, o, num_nodes, TextLen{});
}

int b200sa_suffix_tree_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp,
                           const b200sa_tree *out, uint64_t cap, uint64_t *num_nodes, void *stream) {
    TRY(tree_args(c, n, d_sa, d_lcp, out, cap, num_nodes));
    TRY(enter(c, stream));
    *num_nodes = 0;
    return leave(c, suffix_tree_dev_core(c, n, d_sa, d_lcp, out, num_nodes));
}

static int suffix_tree_host(b200sa_ctx *c, uint64_t n, const uint32_t *sa, const uint32_t *lcp, const b200sa_tree *out,
                            uint64_t *num_nodes) {
    if (n == 0) {
        out->parent[0] = TREE_NONE;
        out->depth[0] = out->sa_lo[0] = out->sa_hi[0] = out->label_start[0] = 0;
        out->subtree_end[0] = 1;
        *num_nodes = 1;
        return B200SA_OK;
    }
    const uint64_t cap = 2 * n;
    TRY(ensure(c, c->sa, n * 4));
    TRY(ensure(c, c->lcp, n * 4));
    TRY(ensure(c, c->tree_out, cap * 4 * 6));
    TRY(mark(c, "h2d"));
    CU_TRY(c, cudaMemcpyAsync(c->sa.p, sa, n * 4, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(c->lcp.p, lcp, n * 4, cudaMemcpyHostToDevice, c->stream));
    uint32_t *dev[6];
    for (int k = 0; k < 6; k++) dev[k] = ptr<uint32_t>(c->tree_out) + k * cap;
    TreeOut o{dev[0], dev[1], dev[2], dev[3], dev[4], dev[5]};
    uint64_t N = 0;
    TRY(suffix_tree_core(c, (uint32_t)n, ptr<uint32_t>(c->sa), ptr<uint32_t>(c->lcp), o, &N, TextLen{}));
    if (!c->marks.empty()) c->marks.pop_back();        // the copy-out replaces the core's "end"
    TRY(mark(c, "d2h"));
    uint32_t *host[6] = {out->parent, out->depth, out->sa_lo, out->sa_hi, out->label_start, out->subtree_end};
    for (int k = 0; k < 6; k++)
        CU_TRY(c, cudaMemcpyAsync(host[k], dev[k], N * 4, cudaMemcpyDeviceToHost, c->stream));
    TRY(mark(c, "end"));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    *num_nodes = N;
    return B200SA_OK;
}

int b200sa_suffix_tree(b200sa_ctx *c, uint64_t n, const uint32_t *sa, const uint32_t *lcp, const b200sa_tree *out,
                       uint64_t cap, uint64_t *num_nodes) {
    TRY(tree_args(c, n, sa, lcp, out, cap, num_nodes));
    TRY(enter(c, nullptr));
    *num_nodes = 0;
    return leave(c, suffix_tree_host(c, n, sa, lcp, out, num_nodes));
}

// ------------------------------------------------------------ generalized suffix array without separators (SURVEY 8f-6)
static int docs_bad(b200sa_ctx *c, uint32_t bits) {
    std::string m = "doc_starts rejected:";
    if (bits & DOCS_BAD_FIRST) m += " doc_starts[0] != 0;";
    if (bits & DOCS_BAD_ORDER) m += " not ascending;";
    if (bits & DOCS_BAD_RANGE) m += " an entry above n;";
    c->last_error = m;
    return B200SA_ERR_BAD_ARG;
}

// k_docs_check on the device doc_starts (ndocs >= 1), one read-back; *maxlen gets the longest document.
static int docs_check_dev(b200sa_ctx *c, const uint32_t *d_starts, uint32_t ndocs, uint32_t n,
                          uint32_t *maxlen = nullptr) {
    TRY(ensure(c, c->small, 4096));
    uint32_t *words = ptr<uint32_t>(c->small);           // [0] check bits, [1] longest document
    CU_TRY(c, cudaMemsetAsync(words, 0, 8, c->stream));
    LAUNCH(c, k_docs_check, cdiv(ndocs, BLK), d_starts, ndocs, n, words);
    CU_TRY(c, cudaGetLastError());
    TRY(read_words(c, words, maxlen ? 2 : 1));
    if (c->h_pin[0]) return docs_bad(c, c->h_pin[0]);
    if (maxlen) *maxlen = c->h_pin[1];
    return B200SA_OK;
}

// The checks of k_docs_check on host entries doc_starts[first, first + count); *prev holds
// doc_starts[first - 1] on entry and the span's last entry on return.
static uint32_t docs_check_span(uint64_t n, const uint32_t *starts, uint64_t first, uint64_t count, uint64_t *prev) {
    uint32_t bad = 0;
    for (uint64_t k = 0; k < count; k++) {
        uint64_t v = starts[k], d = first + k;
        if (d == 0 && v != 0) bad |= DOCS_BAD_FIRST;
        if (v > n) bad |= DOCS_BAD_RANGE;
        if (d > 0 && *prev <= n && v < *prev) bad |= DOCS_BAD_ORDER;   // a start above n is flagged itself
        *prev = v;
    }
    return bad;
}

static int docs_check_host(b200sa_ctx *c, uint64_t n, const uint32_t *starts, uint32_t ndocs) {
    uint64_t prev = 0;
    uint32_t bad = docs_check_span(n, starts, 0, ndocs, &prev);
    return bad ? docs_bad(c, bad) : B200SA_OK;
}

// The same checks on device entries, copied back through a bounded host buffer (ndocs is not
// bounded by n: any number of documents may be empty).
static int docs_check_dev_copy(b200sa_ctx *c, uint64_t n, const uint32_t *d_starts, uint32_t ndocs) {
    const uint64_t chunk = 1u << 16;
    std::vector<uint32_t> buf;
    try {
        buf.resize(ndocs < chunk ? ndocs : chunk);
    } catch (const std::bad_alloc &) {
        c->last_error = "host buffer for the doc_starts check";
        return B200SA_ERR_OOM;
    }
    uint64_t prev = 0;
    uint32_t bad = 0;
    for (uint64_t first = 0; first < ndocs; first += chunk) {
        uint64_t cnt = ndocs - first < chunk ? ndocs - first : chunk;
        CU_TRY(c, cudaMemcpyAsync(buf.data(), d_starts + first, cnt * 4, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaStreamSynchronize(c->stream));
        bad |= docs_check_span(n, buf.data(), first, cnt, &prev);
    }
    return bad ? docs_bad(c, bad) : B200SA_OK;
}

static int docs_args(b200sa_ctx *c, uint64_t n, const void *text, const void *starts, uint32_t ndocs, const void *gsa) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if ((n > 0 && (!text || !gsa)) || (ndocs > 0 && !starts)) return null_ptr(c);
    if (n > B200SA_MAX_N) return too_long(c);
    if (ndocs == 0 && n > 0) return no_docs(c);
    return B200SA_OK;
}

// n >= 2, ndocs >= 1, device inputs and outputs (d_glcp may be null).  Phases: docs_check, the SA + LCP
// build's own, docs_split, docs_sort, docs_place, docs_fill, docs_out.
static int docs_core(b200sa_ctx *c, const uint8_t *d_text, uint32_t n, const uint32_t *d_starts, uint32_t ndocs,
                     uint32_t *d_gsa, uint32_t *d_glcp) {
    TRY(mark(c, "docs_check"));
    uint32_t maxlen;
    TRY(docs_check_dev(c, d_starts, ndocs, n, &maxlen));
    uint32_t *words = ptr<uint32_t>(c->small);           // [0] |A|

    // 1. SA and LCP of the concatenation
    TRY(ensure(c, c->sa, (size_t)n * 4));
    TRY(ensure(c, c->lcp, (size_t)n * 4));
    uint32_t *sa = ptr<uint32_t>(c->sa), *lcp = ptr<uint32_t>(c->lcp);
    TRY(build_lcp_dev(c, d_text, n, sa, lcp));
    if (!c->marks.empty()) c->marks.pop_back();          // docs_split follows instead of the build's "end"

    // 2-3. r per rank, U / A split, block minima of LCP_C
    TRY(mark(c, "docs_split"));
    TRY(ensure(c, c->isa, (size_t)n * 4));
    TRY(ensure(c, c->rank, (size_t)n * 4));
    TRY(ensure(c, c->p0, (size_t)n * 4));
    uint32_t *rem = ptr<uint32_t>(c->isa), *pre = ptr<uint32_t>(c->rank), *list = ptr<uint32_t>(c->p0);
    TRY((dev_scan<OpSum>(c, DocsSplitIn{sa, lcp, d_starts, ndocs, n, rem}, DocsSplitOut{pre, list, n}, n, words)));
    AnsvLevels L;
    TRY(ansv_levels(c, lcp, n, &L, c->qbuf));
    TRY(read_words(c, words, 1));
    const uint32_t na = c->h_pin[0];

    uint32_t *gr = nullptr, *glo = nullptr;
    if (na > 0) {
        // 4. sort A by (lo, r, d), place it, U fills the rest
        TRY(mark(c, "docs_sort"));
        TRY(ensure(c, c->k64a, (size_t)na * 8));
        TRY(ensure(c, c->k64b, (size_t)na * 8));
        TRY(ensure(c, c->v0, (size_t)na * 4));
        TRY(ensure(c, c->v1, (size_t)na * 4));
        const uint32_t *alist = list + (n - na);
        uint32_t *v0 = ptr<uint32_t>(c->v0), *v1 = ptr<uint32_t>(c->v1);
        const int lb = bit_length(n - 1), rb = bit_length(maxlen), db = bit_length(ndocs - 1);
        const char *e2 = getenv("B200SA_DOCS_SORT2");
        uint64_t *K;
        uint32_t *V;
        int shift;
        if (lb + rb + db <= 64 && !(e2 && atoi(e2) == 1)) {
            DocsKey kf{L, sa, rem, d_starts, alist, ndocs, rb, db, true};
            TRY(sort_pairs_from(c, kf, LoadArr<uint32_t>{alist}, ptr<uint64_t>(c->k64a), v0, ptr<uint64_t>(c->k64b), v1,
                                na, lb + rb + db, &K, &V));
            shift = rb + db;
        } else {
            // (lo, r, d) does not fit 64 bits: a stable sort by d, then one by (lo, r)
            uint32_t *K1, *V1;
            DocsDocKey kd{sa, d_starts, alist, ndocs};
            TRY(sort_pairs_from(c, kd, LoadArr<uint32_t>{alist}, ptr<uint32_t>(c->k64a), v0, ptr<uint32_t>(c->k64b), v1,
                                na, db, &K1, &V1));
            uint32_t *other = V1 == v0 ? v1 : v0;          // V1 is read only by the first pass of the second sort
            DocsKey kf{L, sa, rem, d_starts, V1, ndocs, rb, 0, false};
            TRY(sort_pairs_from(c, kf, LoadArr<uint32_t>{V1}, ptr<uint64_t>(c->k64a), other, ptr<uint64_t>(c->k64b), V1,
                                na, lb + rb, &K, &V));
            shift = rb;
        }
        TRY(mark(c, "docs_place"));
        TRY(ensure(c, c->p1, (size_t)n * 4));
        TRY(ensure(c, c->g0, (size_t)n * 4));
        gr = ptr<uint32_t>(c->p1);
        glo = ptr<uint32_t>(c->g0);
        CU_TRY(c, cudaMemsetAsync(glo, 0xff, (size_t)n * 4, c->stream));
        LAUNCH(c, k_docs_place, cdiv(na, BLK), K, V, na, shift, sa, lcp, rem, pre, gr, glo);
        TRY(mark(c, "docs_fill"));
        TRY((dev_scan<OpSum>(c, DocsFreeIn{glo}, DocsFreeOut{list, gr, glo}, n, nullptr)));
    }
    // 5. G and glcp
    TRY(mark(c, "docs_out"));
    LAUNCH(c, k_docs_out, cdiv(n, BLK), gr, glo, n, sa, rem, L, d_gsa, d_glcp);
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

static int docs_build_dev_core(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_doc_starts,
                               uint32_t ndocs, uint32_t *d_gsa, uint32_t *d_glcp) {
    if (n >= 2) return docs_core(c, d_text, (uint32_t)n, d_doc_starts, ndocs, d_gsa, d_glcp);
    // nothing to launch: doc_starts is checked from host copies, G = [0] and glcp = [0] for n = 1
    TRY(docs_check_dev_copy(c, n, d_doc_starts, ndocs));
    if (n == 1 && (cudaMemsetAsync(d_gsa, 0, 4, c->stream) != cudaSuccess ||
                   (d_glcp && cudaMemsetAsync(d_glcp, 0, 4, c->stream) != cudaSuccess)))
        return fail(c, B200SA_ERR_CUDA, "output write failed");
    return B200SA_OK;
}

int b200sa_docs_build_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_doc_starts,
                          uint32_t ndocs, uint32_t *d_gsa, uint32_t *d_glcp, void *stream) {
    TRY(docs_args(c, n, d_text, d_doc_starts, ndocs, d_gsa));
    TRY(enter(c, stream));
    return leave(c, docs_build_dev_core(c, d_text, n, d_doc_starts, ndocs, d_gsa, d_glcp));
}

static int docs_host(b200sa_ctx *c, const uint8_t *text, uint32_t n, const uint32_t *starts, uint32_t ndocs,
                     uint32_t *gsa_out, uint32_t *glcp_out) {
    if (n <= 1) {
        if (n == 1) {
            gsa_out[0] = 0;
            if (glcp_out) glcp_out[0] = 0;
        }
        return B200SA_OK;
    }
    TRY(ensure(c, c->text, n));
    TRY(ensure(c, c->docs_starts, (size_t)ndocs * 4));
    TRY(ensure(c, c->docs_out, (size_t)n * 4 * (glcp_out ? 2 : 1)));
    uint32_t *d_gsa = ptr<uint32_t>(c->docs_out), *d_glcp = glcp_out ? d_gsa + n : nullptr;
    TRY(mark(c, "h2d"));
    CU_TRY(c, cudaMemcpyAsync(c->text.p, text, n, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(c->docs_starts.p, starts, (size_t)ndocs * 4, cudaMemcpyHostToDevice, c->stream));
    TRY(docs_core(c, ptr<uint8_t>(c->text), n, ptr<uint32_t>(c->docs_starts), ndocs, d_gsa, d_glcp));
    if (!c->marks.empty()) c->marks.pop_back();          // the copy-out replaces the core's "end"
    TRY(mark(c, "d2h"));
    CU_TRY(c, cudaMemcpyAsync(gsa_out, d_gsa, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
    if (glcp_out) CU_TRY(c, cudaMemcpyAsync(glcp_out, d_glcp, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
    TRY(mark(c, "end"));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

int b200sa_docs_build(b200sa_ctx *c, const uint8_t *text, uint64_t n, const uint32_t *doc_starts, uint32_t ndocs,
                      uint32_t *gsa_out, uint32_t *glcp_out) {
    TRY(docs_args(c, n, text, doc_starts, ndocs, gsa_out));
    TRY(docs_check_host(c, n, doc_starts, ndocs));
    TRY(enter(c, nullptr));
    return leave(c, docs_host(c, text, (uint32_t)n, doc_starts, ndocs, gsa_out, glcp_out));
}

static int docs_positions_core(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_gsa,
                               const uint32_t *d_doc_starts, uint32_t ndocs, const uint8_t *d_queries,
                               const uint64_t *d_q_off, uint32_t nq, uint32_t *d_start, uint32_t *d_end) {
    if (nq > 0) {
        LAUNCH(c, k_positions<DocsEnd>, cdiv(nq, BLK), d_text, (uint32_t)n, d_gsa, d_queries, d_q_off, nq, d_start,
               d_end, DocsEnd{d_doc_starts, ndocs, (uint32_t)n});
        CU_TRY(c, cudaGetLastError());
    }
    return B200SA_OK;
}

int b200sa_docs_positions_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_gsa,
                              const uint32_t *d_doc_starts, uint32_t ndocs, const uint8_t *d_queries,
                              const uint64_t *d_q_off, uint32_t nq, uint32_t *d_start, uint32_t *d_end, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if ((nq > 0 && (!d_q_off || !d_start || !d_end)) || (n > 0 && (!d_text || !d_gsa || !d_doc_starts)))
        return null_ptr(c);
    if (ndocs == 0 && n > 0) return no_docs(c);
    if (n > B200SA_MAX_N) return too_long(c);
    TRY(enter(c, stream));
    return leave(c, docs_positions_core(c, d_text, n, d_gsa, d_doc_starts, ndocs, d_queries, d_q_off, nq, d_start,
                                        d_end));
}

// ------------------------------------------------------------ generalized suffix tree with document counts (SURVEY 8f-7)
static int docs_tree_args(b200sa_ctx *c, uint64_t n, const void *gsa, const void *glcp, const void *starts,
                          uint32_t ndocs, const b200sa_docs_tree_out *out, uint64_t cap, uint64_t *num_nodes) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!out) return null_ptr(c);
    TRY(tree_args(c, n, gsa, glcp, &out->tree, cap, num_nodes));
    if (!out->term_end || !out->doc_count || (ndocs > 0 && !starts)) return null_ptr(c);
    if (ndocs == 0 && n > 0) return no_docs(c);
    return B200SA_OK;
}

// The ranks stably by their document (the tree's document-sort key), in the buffers p0, p1, v0 and v1.
static int dtree_sort(b200sa_ctx *c, const uint32_t *doc, uint32_t n, int bits, uint32_t **kout, uint32_t **vout) {
    return sort_pairs_from(c, LoadArr<uint32_t>{doc}, LoadIndex{}, ptr<uint32_t>(c->p0), ptr<uint32_t>(c->p1),
                           ptr<uint32_t>(c->v0), ptr<uint32_t>(c->v1), n, bits, kout, vout);
}

// n >= 1, ndocs >= 1, device inputs and outputs (capacity >= 2n each).  Phases: docs_check (when
// check_starts), dtree_len, the tree's five, dtree_term, dtree_sort, dtree_pairs, dtree_count.
static int docs_tree_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_g, const uint32_t *d_glcp,
                          const uint32_t *d_starts, uint32_t ndocs, bool check_starts, const b200sa_docs_tree_out *out,
                          uint64_t *num_nodes) {
    TRY(ensure(c, c->small, 4096));
    uint32_t *words = ptr<uint32_t>(c->small);           // [0, 2) the tree's, [2] the check bits of the stages after it
    if (check_starts) {
        TRY(mark(c, "docs_check"));
        TRY(docs_check_dev(c, d_starts, ndocs, n));
    }
    // document and suffix length of every rank, then the tree with rule 3'
    TRY(mark(c, "dtree_len"));
    TRY(ensure(c, c->isa, (size_t)n * 4));
    TRY(ensure(c, c->rank, (size_t)n * 4));
    uint32_t *len = ptr<uint32_t>(c->isa), *doc = ptr<uint32_t>(c->rank);
    LAUNCH(c, k_dtree_len, cdiv(n, BLK), d_g, n, d_starts, ndocs, len, doc);
    const b200sa_tree &t = out->tree;
    TreeOut o{t.parent, t.depth, t.sa_lo, t.sa_hi, t.label_start, t.subtree_end};
    uint64_t N64 = 0, *K = nullptr;
    TRY(suffix_tree_core(c, n, d_g, d_glcp, o, &N64, DocsLen{len}, &K));
    if (!c->marks.empty()) c->marks.pop_back();          // dtree_term follows instead of the tree's "end"
    const uint32_t N = (uint32_t)N64, *first = ptr<uint32_t>(c->g0);
    const int B = bit_length(n);                         // as in suffix_tree_core

    // terminals
    TRY(mark(c, "dtree_term"));
    AnsvLevels L;
    TRY(ansv_levels(c, d_glcp, n, &L, c->qbuf));
    CU_TRY(c, cudaMemsetAsync(words + 2, 0, 4, c->stream));
    CU_TRY(c, cudaMemcpyAsync(out->term_end, t.sa_lo, (size_t)N * 4, cudaMemcpyDeviceToDevice, c->stream));
    LAUNCH(c, k_dtree_term, cdiv(n, BLK), L, len, n, K, first, N, B, out->term_end, words + 2);

    // Hui's counts: ranks stably by document, one add per pair at its lowest common ancestor, one scan
    TRY(mark(c, "dtree_sort"));
    TRY(ensure(c, c->p0, (size_t)n * 4));
    TRY(ensure(c, c->p1, (size_t)n * 4));
    uint32_t *dk, *rk;
    const int db = bit_length(ndocs - 1);
    TRY(dtree_sort(c, doc, n, db, &dk, &rk));
    TRY(mark(c, "dtree_pairs"));
    TRY(ensure(c, c->g1, ((size_t)N + 1) * 4));
    uint32_t *pairs = ptr<uint32_t>(c->g1);
    CU_TRY(c, cudaMemsetAsync(pairs, 0, ((size_t)N + 1) * 4, c->stream));
    LAUNCH(c, k_dtree_pairs, cdiv(n, BLK), L, dk, rk, len, n, K, first, N, B, pairs, words + 2);
    TRY(mark(c, "dtree_count"));
    TRY((dev_scan<OpSum>(c, InArray{pairs}, OutStoreExcl{pairs}, (uint64_t)N + 1, nullptr)));
    LAUNCH(c, k_dtree_count, cdiv(N, BLK), t.sa_lo, t.sa_hi, t.subtree_end, pairs, N, out->doc_count);
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    TRY(read_words(c, words + 2, 1));
    if (c->h_pin[0]) return tree_bad(c, c->h_pin[0]);
    *num_nodes = N;
    return B200SA_OK;
}

// n = 0: doc_starts checked from host copies; the root alone, without terminals or documents.
static int docs_tree_root_dev(b200sa_ctx *c, const uint32_t *d_starts, uint32_t ndocs, const b200sa_docs_tree_out *out,
                              uint64_t *num_nodes) {
    TRY(docs_check_dev_copy(c, 0, d_starts, ndocs));
    const uint32_t root[8] = {TREE_NONE, 0, 0, 0, 0, 1, 0, 0};
    const b200sa_tree &t = out->tree;
    uint32_t *dst[8] = {t.parent, t.depth, t.sa_lo, t.sa_hi, t.label_start, t.subtree_end, out->term_end,
                        out->doc_count};
    return root_dev(c, dst, root, 8, num_nodes);
}

int b200sa_docs_tree_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_gsa, const uint32_t *d_glcp,
                         const uint32_t *d_doc_starts, uint32_t ndocs, const b200sa_docs_tree_out *out, uint64_t cap,
                         uint64_t *num_nodes, void *stream) {
    TRY(docs_tree_args(c, n, d_gsa, d_glcp, d_doc_starts, ndocs, out, cap, num_nodes));
    TRY(enter(c, stream));
    *num_nodes = 0;
    if (n == 0) return leave(c, docs_tree_root_dev(c, d_doc_starts, ndocs, out, num_nodes));
    return leave(c, docs_tree_core(c, (uint32_t)n, d_gsa, d_glcp, d_doc_starts, ndocs, true, out, num_nodes));
}

static int docs_tree_host(b200sa_ctx *c, uint32_t n, const uint32_t *gsa, const uint32_t *glcp, const uint32_t *starts,
                          uint32_t ndocs, const b200sa_docs_tree_out *out, uint64_t *num_nodes) {
    if (n == 0) {
        const b200sa_tree &t = out->tree;
        t.parent[0] = TREE_NONE;
        t.depth[0] = t.sa_lo[0] = t.sa_hi[0] = t.label_start[0] = 0;
        t.subtree_end[0] = 1;
        out->term_end[0] = out->doc_count[0] = 0;
        *num_nodes = 1;
        return B200SA_OK;
    }
    const uint64_t cap = 2 * (uint64_t)n;
    TRY(ensure(c, c->sa, (size_t)n * 4));
    TRY(ensure(c, c->lcp, (size_t)n * 4));
    TRY(ensure(c, c->docs_starts, (size_t)ndocs * 4));
    TRY(ensure(c, c->tree_out, cap * 4 * 8));
    TRY(mark(c, "h2d"));
    CU_TRY(c, cudaMemcpyAsync(c->sa.p, gsa, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(c->lcp.p, glcp, (size_t)n * 4, cudaMemcpyHostToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(c->docs_starts.p, starts, (size_t)ndocs * 4, cudaMemcpyHostToDevice, c->stream));
    uint32_t *dev[8];
    for (int k = 0; k < 8; k++) dev[k] = ptr<uint32_t>(c->tree_out) + k * cap;
    b200sa_docs_tree_out o{{dev[0], dev[1], dev[2], dev[3], dev[4], dev[5]}, dev[6], dev[7]};
    uint64_t N = 0;
    TRY(docs_tree_core(c, n, ptr<uint32_t>(c->sa), ptr<uint32_t>(c->lcp), ptr<uint32_t>(c->docs_starts), ndocs, false,
                       &o, &N));
    if (!c->marks.empty()) c->marks.pop_back();          // the copy-out replaces the core's "end"
    TRY(mark(c, "d2h"));
    const b200sa_tree &t = out->tree;
    uint32_t *host[8] = {t.parent, t.depth, t.sa_lo, t.sa_hi, t.label_start, t.subtree_end, out->term_end,
                         out->doc_count};
    for (int k = 0; k < 8; k++)
        CU_TRY(c, cudaMemcpyAsync(host[k], dev[k], N * 4, cudaMemcpyDeviceToHost, c->stream));
    TRY(mark(c, "end"));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    *num_nodes = N;
    return B200SA_OK;
}

int b200sa_docs_tree(b200sa_ctx *c, uint64_t n, const uint32_t *gsa, const uint32_t *glcp, const uint32_t *doc_starts,
                     uint32_t ndocs, const b200sa_docs_tree_out *out, uint64_t cap, uint64_t *num_nodes) {
    TRY(docs_tree_args(c, n, gsa, glcp, doc_starts, ndocs, out, cap, num_nodes));
    TRY(docs_check_host(c, n, doc_starts, ndocs));
    TRY(enter(c, nullptr));
    *num_nodes = 0;
    return leave(c, docs_tree_host(c, (uint32_t)n, gsa, glcp, doc_starts, ndocs, out, num_nodes));
}

static int docs_tree_counts_core(b200sa_ctx *c, const uint32_t *d_sa_lo, const uint32_t *d_sa_hi,
                                 const uint32_t *d_doc_count, uint64_t num_nodes, const uint32_t *d_start,
                                 const uint32_t *d_end, uint32_t nq, uint32_t *d_count) {
    if (nq == 0) return B200SA_OK;
    TRY(ensure(c, c->small, 4096));
    uint32_t *flag = ptr<uint32_t>(c->small);
    CU_TRY(c, cudaMemsetAsync(flag, 0, 4, c->stream));
    LAUNCH(c, k_dtree_counts, cdiv(nq, BLK), d_sa_lo, d_sa_hi, d_doc_count, (uint32_t)num_nodes, d_start, d_end, nq,
           d_count, flag);
    CU_TRY(c, cudaGetLastError());
    TRY(read_words(c, flag, 1));
    if (c->h_pin[0]) return fail(c, B200SA_ERR_BAD_ARG, "docs tree counts: a range [start, end) is the range of no node");
    return B200SA_OK;
}

int b200sa_docs_tree_counts_dev(b200sa_ctx *c, const uint32_t *d_sa_lo, const uint32_t *d_sa_hi,
                                const uint32_t *d_doc_count, uint64_t num_nodes, const uint32_t *d_start,
                                const uint32_t *d_end, uint32_t nq, uint32_t *d_count, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (nq > 0 && (!d_sa_lo || !d_sa_hi || !d_doc_count || !d_start || !d_end || !d_count)) return null_ptr(c);
    if (nq > 0 && (num_nodes == 0 || num_nodes > 2 * B200SA_TREE_MAX_N))
        return fail(c, B200SA_ERR_BAD_ARG, "docs tree counts: num_nodes must be in [1, 2 * B200SA_TREE_MAX_N]");
    TRY(enter(c, stream));
    return leave(c, docs_tree_counts_core(c, d_sa_lo, d_sa_hi, d_doc_count, num_nodes, d_start, d_end, nq, d_count));
}

// ------------------------------------------------------------ document listing (SURVEY 8f-8)
// n >= 1, ndocs >= 1.  Phases: docs_check, dlist_len, dlist_sort, dlist_prev.
static int docs_list_index_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_g, const uint32_t *d_starts,
                                uint32_t ndocs, uint32_t *d_byd, uint32_t *d_prev) {
    TRY(mark(c, "docs_check"));
    TRY(docs_check_dev(c, d_starts, ndocs, n));
    TRY(mark(c, "dlist_len"));                          // the document of every rank (its length is not used)
    TRY(ensure(c, c->isa, (size_t)n * 4));
    TRY(ensure(c, c->rank, (size_t)n * 4));
    uint32_t *len = ptr<uint32_t>(c->isa), *doc = ptr<uint32_t>(c->rank);
    LAUNCH(c, k_dtree_len, cdiv(n, BLK), d_g, n, d_starts, ndocs, len, doc);
    TRY(mark(c, "dlist_sort"));
    TRY(ensure(c, c->p0, (size_t)n * 4));
    TRY(ensure(c, c->p1, (size_t)n * 4));
    TRY(ensure(c, c->v0, (size_t)n * 4));
    TRY(ensure(c, c->v1, (size_t)n * 4));
    uint32_t *dk, *rk;
    const int db = bit_length(ndocs - 1);
    TRY(dtree_sort(c, doc, n, db, &dk, &rk));
    TRY(mark(c, "dlist_prev"));
    LAUNCH(c, k_dlist_prev, cdiv(n, BLK), dk, rk, n, d_byd, d_prev);
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

int b200sa_docs_list_index_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_gsa, const uint32_t *d_doc_starts,
                               uint32_t ndocs, uint32_t *d_byd, uint32_t *d_prev, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if ((n > 0 && (!d_gsa || !d_byd || !d_prev)) || (ndocs > 0 && !d_doc_starts)) return null_ptr(c);
    if (ndocs == 0 && n > 0) return no_docs(c);
    if (n > B200SA_MAX_N) return too_long(c);
    TRY(enter(c, stream));
    if (n == 0) return leave(c, docs_check_dev_copy(c, 0, d_doc_starts, ndocs));
    return leave(c, docs_list_index_core(c, (uint32_t)n, d_gsa, d_doc_starts, ndocs, d_byd, d_prev));
}

// The listing's front half, shared by the listing and top-k: nq >= 1.  Writes the offsets (nq + 1) and
// *total, and leaves in *A and *item_off (c->k64a, c->k64b) what k_dlist<true> needs to emit.  Phases:
// dlist_levels, dlist_count, dlist_scan.
static int docs_list_front(b200sa_ctx *c, uint32_t n, const uint32_t *d_g, const uint32_t *d_starts, uint32_t ndocs,
                           const uint32_t *d_byd, const uint32_t *d_prev, const uint32_t *d_start,
                           const uint32_t *d_end, uint32_t nq, uint64_t *d_offsets, DListArgs *Aout,
                           unsigned long long **item_off_out, uint64_t *total) {
    typedef unsigned long long u64;
    TRY(ensure(c, c->small, 4096));
    uint32_t *words = ptr<uint32_t>(c->small);           // [0] check bits, [2, 4) items, [4, 6) total
    u64 *d_items = reinterpret_cast<u64 *>(words + 2), *d_total = reinterpret_cast<u64 *>(words + 4);
    TRY(mark(c, "dlist_levels"));
    DListArgs A;
    TRY(ansv_levels(c, d_prev, n, &A.L, c->qbuf));
    TRY(mark(c, "dlist_count"));
    CU_TRY(c, cudaMemsetAsync(words, 0, 24, c->stream));
    TRY(ensure(c, c->k64a, ((size_t)nq + 1) * 8));
    u64 *item_start = ptr<u64>(c->k64a);
    TRY((dev_scan<OpSum64>(c, DListChunks{d_start, d_end, nq, n, words}, OutStoreExcl64{item_start}, (uint64_t)nq + 1,
                           d_items)));
    TRY(read_words(c, words, 4));
    if (c->h_pin[0] & DLIST_BAD_RANGE)
        return fail(c, B200SA_ERR_BAD_ARG, "docs list: a range [start, end) has start > end or end > n");
    const uint64_t items = pin_u64(c, 2);
    if (items > (uint64_t)0x7fffffff * NWARP)
        return fail(c, B200SA_ERR_TOO_LARGE, "docs list: more than 2^31 * 8 chunks of 1024 ranks in one batch");
    A.qs = d_start; A.qe = d_end; A.item_start = item_start; A.nq = nq; A.items = items;
    TRY(ensure(c, c->p0, (size_t)items * 4));
    TRY(ensure(c, c->k64b, ((size_t)items + 1) * 8));
    uint32_t *cnt = ptr<uint32_t>(c->p0);
    u64 *item_off = ptr<u64>(c->k64b);
    const uint32_t grid = cdiv(items, NWARP);
    if (items) LAUNCH(c, k_dlist<false>, grid, A, cnt, (const u64 *)nullptr, d_g, d_starts, ndocs, n, d_byd,
                      (uint32_t *)nullptr, (uint32_t *)nullptr);
    TRY(mark(c, "dlist_scan"));
    TRY((dev_scan<OpSum64>(c, InCount64{cnt, items}, OutStoreExcl64{item_off}, items + 1, d_total)));
    LAUNCH(c, k_dlist_qoff, cdiv((uint64_t)nq + 1, BLK), item_start, item_off, nq, 1u,
           reinterpret_cast<u64 *>(d_offsets));
    TRY(read_words(c, words + 4, 2));
    *total = pin_u64(c, 0);
    *Aout = A;
    *item_off_out = item_off;
    return B200SA_OK;
}

// nq >= 1.  Phases: dlist_levels, dlist_count, dlist_scan, dlist_emit (when the listing fits in cap).
static int docs_list_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_g, const uint32_t *d_starts, uint32_t ndocs,
                          const uint32_t *d_byd, const uint32_t *d_prev, const uint32_t *d_start,
                          const uint32_t *d_end, uint32_t nq, uint64_t *d_offsets, uint32_t *d_docs, uint32_t *d_tf,
                          uint64_t cap, uint64_t *total) {
    typedef unsigned long long u64;
    DListArgs A;
    u64 *item_off;
    TRY(docs_list_front(c, n, d_g, d_starts, ndocs, d_byd, d_prev, d_start, d_end, nq, d_offsets, &A, &item_off, total));
    if (*total > 0 && *total <= cap) {
        TRY(mark(c, "dlist_emit"));
        LAUNCH(c, k_dlist<true>, cdiv(A.items, NWARP), A, ptr<uint32_t>(c->p0), item_off, d_g, d_starts, ndocs, n,
               d_byd, d_docs, d_tf);
    }
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

// The answer of the count-then-fetch entry points to a batch of no queries: offsets = [0] (the
// caller sets *total = 0).
static int empty_batch(b200sa_ctx *c, uint64_t *d_offsets) {
    CU_TRY(c, cudaMemsetAsync(d_offsets, 0, 8, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

int b200sa_docs_list_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_gsa, const uint32_t *d_doc_starts,
                         uint32_t ndocs, const uint32_t *d_byd, const uint32_t *d_prev, const uint32_t *d_start,
                         const uint32_t *d_end, uint32_t nq, uint64_t *d_offsets, uint32_t *d_docs, uint32_t *d_tf,
                         uint64_t cap, uint64_t *total, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!total || !d_offsets || (nq > 0 && (!d_start || !d_end)) || (cap > 0 && !d_docs) ||
        (n > 0 && (!d_gsa || !d_doc_starts || !d_byd || !d_prev)))
        return null_ptr(c);
    if (ndocs == 0 && n > 0) return no_docs(c);
    if (n > B200SA_MAX_N) return too_long(c);
    TRY(enter(c, stream));
    *total = 0;
    if (nq == 0) return leave(c, empty_batch(c, d_offsets));
    return leave(c, docs_list_core(c, (uint32_t)n, d_gsa, d_doc_starts, ndocs, d_byd, d_prev, d_start, d_end, nq,
                                   d_offsets, d_docs, d_tf, cap, total));
}

// ------------------------------------------------------------ top-k document retrieval (SURVEY 8f-9)
// Launches of k_topk_tile that a round needs when its largest query lists lmax entries (topk_tiles on the host).
static uint32_t topk_levels(uint64_t lmax, uint32_t k) {
    if (lmax <= TOPK_WARP) return 0;
    uint32_t lv = 1;
    for (uint64_t L = lmax; L > TOPK_TILE; lv++) {
        const uint64_t t1 = (L - 1) / TOPK_TILE, last = L - t1 * TOPK_TILE;
        L = t1 * k + (last < k ? last : k);
    }
    return lv;
}

// nq >= 1, 1 <= k <= B200SA_TOPK_MAX.  Phases: dlist_levels, dlist_count, dlist_scan, then per round
// topk_emit and topk_select.
static int docs_topk_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_g, const uint32_t *d_starts, uint32_t ndocs,
                          const uint32_t *d_byd, const uint32_t *d_prev, const uint32_t *d_start,
                          const uint32_t *d_end, uint32_t nq, uint32_t k, uint32_t *d_count, uint32_t *d_docs,
                          uint32_t *d_tf) {
    typedef unsigned long long u64;
    static_assert(TOPK_KMAX == B200SA_TOPK_MAX, "one block sorts the survivors of a tile");
    TRY(ensure(c, c->g0, ((size_t)nq + 1) * 8));
    u64 *off = ptr<u64>(c->g0);
    DListArgs A;
    u64 *item_off;
    uint64_t total;
    TRY(docs_list_front(c, n, d_g, d_starts, ndocs, d_byd, d_prev, d_start, d_end, nq,
                        reinterpret_cast<uint64_t *>(off), &A, &item_off, &total));
    LAUNCH(c, k_topk_count, cdiv(nq, BLK), off, nq, k, d_count);

    // Rounds: runs of consecutive queries whose listing fits the budget; a larger query is a round of its own.
    uint64_t budget = B200SA_TOPK_ROUND_ENTRIES;
    if (const char *e = getenv("B200SA_TOPK_ROUND")) { long long v = atoll(e); if (v >= 1) budget = (uint64_t)v; }
    struct Round { uint32_t q0, q1; uint64_t lmax; };
    std::vector<Round> rounds{{0, nq, total < ndocs ? total : (uint64_t)ndocs}};
    std::vector<u64> h_off, h_is;
    uint64_t rcap = total, max_items = 0;
    const bool multi = total > budget;
    if (multi) {                                         // cut the batch on the host
        h_off.resize((size_t)nq + 1);
        h_is.resize((size_t)nq + 1);
        CU_TRY(c, cudaMemcpyAsync(h_off.data(), off, ((size_t)nq + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaMemcpyAsync(h_is.data(), A.item_start, ((size_t)nq + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaStreamSynchronize(c->stream));
        rounds.clear();
        rcap = 0;
        for (uint32_t q0 = 0, q1; q0 < nq; q0 = q1) {
            uint64_t lmax = h_off[q0 + 1] - h_off[q0];
            for (q1 = q0 + 1; q1 < nq && h_off[q1 + 1] - h_off[q0] <= budget; q1++)
                lmax = std::max<uint64_t>(lmax, h_off[q1 + 1] - h_off[q1]);
            rounds.push_back({q0, q1, lmax});
            rcap = std::max<uint64_t>(rcap, h_off[q1] - h_off[q0]);
            max_items = std::max<uint64_t>(max_items, h_is[q1] - h_is[q0]);
        }
        TRY(ensure(c, c->p1, ((size_t)nq + 1) * 8));
        TRY(ensure(c, c->rank, (size_t)max_items * 8));
    }
    TRY(ensure(c, c->v0, (size_t)rcap * 8));             // X: the round's documents | tf, later keys
    TRY(ensure(c, c->v1, (size_t)rcap * 8));             // Y: keys
    TRY(ensure(c, c->g1, ((size_t)nq + 1) * 4));
    uint32_t *X = ptr<uint32_t>(c->v0), *tile_start = ptr<uint32_t>(c->g1);
    u64 *KX = ptr<u64>(c->v0), *KY = ptr<u64>(c->v1);
    uint32_t *d_ntiles = ptr<uint32_t>(c->small) + 8;
    const uint32_t tile_grid = (uint32_t)c->sm_count * 4;
    for (const Round &r : rounds) {
        const uint32_t nqr = r.q1 - r.q0;
        const uint64_t e0 = multi ? h_off[r.q0] : 0, entries = multi ? h_off[r.q1] - e0 : total;
        if (entries == 0) continue;                      // every count is 0
        TRY(mark(c, "topk_emit"));
        DListArgs Ar = A;
        const u64 *io = item_off;
        if (multi) {
            const uint64_t i0 = h_is[r.q0], items = h_is[r.q1] - i0;
            LAUNCH(c, k_topk_rebase, cdiv(std::max<uint64_t>((uint64_t)nqr + 1, items), BLK), A.item_start, item_off,
                   r.q0, nqr, i0, items, e0, ptr<u64>(c->p1), ptr<u64>(c->rank));
            Ar.qs = d_start + r.q0; Ar.qe = d_end + r.q0; Ar.item_start = ptr<u64>(c->p1); Ar.nq = nqr;
            Ar.items = items;
            io = ptr<u64>(c->rank);
        }
        LAUNCH(c, k_dlist<true>, cdiv(Ar.items, NWARP), Ar, ptr<uint32_t>(c->p0), io, d_g, d_starts, ndocs, n, d_byd,
               X, X + rcap);
        TRY(mark(c, "topk_select"));
        const TopkArgs P{off, e0, rcap, r.q0, nqr, k, ndocs, (uint32_t)bit_length(ndocs - 1), d_docs, d_tf};
        LAUNCH(c, k_topk_warp, cdiv(nqr, NWARP), P, (const uint32_t *)X);
        const uint32_t levels = topk_levels(r.lmax, k);
        for (uint32_t lv = 0; lv < levels; lv++) {
            TRY((dev_scan<OpSum>(c, TopkTileCount{off, r.q0, nqr, k, lv}, OutStoreExcl{tile_start}, nqr, d_ntiles)));
            if (lv == 0)
                LAUNCH(c, k_topk_tile<true>, tile_grid, P, lv, (const uint32_t *)tile_start, (const uint32_t *)d_ntiles,
                       (const uint32_t *)X, (const u64 *)nullptr, KY);
            else
                LAUNCH(c, k_topk_tile<false>, tile_grid, P, lv, (const uint32_t *)tile_start, (const uint32_t *)d_ntiles,
                       (const uint32_t *)nullptr, (const u64 *)(lv & 1 ? KY : KX), lv & 1 ? KX : KY);
        }
    }
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

int b200sa_docs_topk_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_gsa, const uint32_t *d_doc_starts,
                         uint32_t ndocs, const uint32_t *d_byd, const uint32_t *d_prev, const uint32_t *d_start,
                         const uint32_t *d_end, uint32_t nq, uint32_t k, uint32_t *d_count, uint32_t *d_docs,
                         uint32_t *d_tf, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!d_count || !d_docs || !d_tf || (nq > 0 && (!d_start || !d_end)) ||
        (n > 0 && (!d_gsa || !d_doc_starts || !d_byd || !d_prev)))
        return null_ptr(c);
    if (ndocs == 0 && n > 0) return no_docs(c);
    if (k == 0 || k > B200SA_TOPK_MAX) return fail(c, B200SA_ERR_BAD_ARG, "docs topk: k must be in 1 .. B200SA_TOPK_MAX");
    if (n > B200SA_MAX_N) return too_long(c);
    TRY(enter(c, stream));
    if (nq == 0) return leave(c, B200SA_OK);
    return leave(c, docs_topk_core(c, (uint32_t)n, d_gsa, d_doc_starts, ndocs, d_byd, d_prev, d_start, d_end, nq, k,
                                   d_count, d_docs, d_tf));
}

// ------------------------------------------------------------ matching statistics and SMEMs (DESIGN 6b f-10)
// q_off[0] = 0, ascending, q_off[nq] = q_bytes, checked on the device (one read-back).  nq >= 1.
static int match_check(b200sa_ctx *c, const uint64_t *d_q_off, uint32_t nq, uint64_t q_bytes) {
    TRY(ensure(c, c->small, 4096));
    uint32_t *word = ptr<uint32_t>(c->small);
    CU_TRY(c, cudaMemsetAsync(word, 0, 4, c->stream));
    LAUNCH(c, k_match_check, cdiv((uint64_t)nq + 1, BLK), d_q_off, nq, q_bytes, word);
    CU_TRY(c, cudaGetLastError());
    TRY(read_words(c, word, 1));
    if (const uint32_t bits = c->h_pin[0]) {
        std::string m = "q_off rejected:";
        if (bits & MATCH_BAD_FIRST) m += " q_off[0] != 0;";
        if (bits & MATCH_BAD_ORDER) m += " not ascending;";
        if (bits & MATCH_BAD_LAST) m += " q_off[nq] != q_bytes;";
        c->last_error = m;
        return B200SA_ERR_BAD_ARG;
    }
    return B200SA_OK;
}

static int match_args(b200sa_ctx *c, uint64_t n, const void *text, const void *sa, const void *queries,
                      const void *q_off, uint32_t nq, uint64_t q_bytes, const void *len, const void *start,
                      const void *end) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if ((n > 0 && (!text || !sa)) || (nq > 0 && !q_off) || (q_bytes > 0 && (!queries || !len))) return null_ptr(c);
    if ((start == nullptr) != (end == nullptr))
        return fail(c, B200SA_ERR_BAD_ARG, "match stats: d_start and d_end are both given or both NULL");
    if (n > B200SA_MAX_N || q_bytes > B200SA_MAX_N)
        return fail(c, B200SA_ERR_TOO_LARGE, "text or queries longer than 2^32-4096 bytes");
    return B200SA_OK;
}

// nq >= 1, q_bytes >= 1.  d_starts non-null (EndF = DocsEnd): doc_starts is verified with q_off.  Phases:
// match_check, match_levels (with ranges), match_search.
template <class EndF>
static int match_stats_core(b200sa_ctx *c, const uint8_t *d_text, uint32_t n, const uint32_t *d_sa,
                            const uint32_t *d_lcp, const uint8_t *d_queries, const uint64_t *d_q_off, uint32_t nq,
                            uint64_t q_bytes, uint32_t *d_len, uint32_t *d_start, uint32_t *d_end, EndF end,
                            const uint32_t *d_starts, uint32_t ndocs) {
    TRY(mark(c, "match_check"));
    TRY(match_check(c, d_q_off, nq, q_bytes));
    if (n > 0 && d_starts) TRY(docs_check_dev(c, d_starts, ndocs, n));
    if (n == 0) {                                        // nothing occurs
        CU_TRY(c, cudaMemsetAsync(d_len, 0, q_bytes * 4, c->stream));
        if (d_start) {
            CU_TRY(c, cudaMemsetAsync(d_start, 0, q_bytes * 4, c->stream));
            CU_TRY(c, cudaMemsetAsync(d_end, 0, q_bytes * 4, c->stream));
        }
        TRY(mark(c, "end"));
        return B200SA_OK;
    }
    const MatchBuf T(d_text, n), Q(d_queries, q_bytes);
    const uint32_t grid = cdiv(q_bytes, BLK);
    AnsvLevels L;
    memset(&L, 0, sizeof L);
    if (d_start) {
        TRY(mark(c, "match_levels"));
        TRY(ansv_levels(c, d_lcp, n, &L, c->qbuf));
        TRY(mark(c, "match_search"));
        LAUNCH(c, (k_match_stats<EndF, true>), grid, T, n, d_sa, L, Q, d_q_off, nq, q_bytes, d_len, d_start, d_end, end);
    } else {
        TRY(mark(c, "match_search"));
        LAUNCH(c, (k_match_stats<EndF, false>), grid, T, n, d_sa, L, Q, d_q_off, nq, q_bytes, d_len, d_start, d_end, end);
    }
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

int b200sa_match_stats_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_sa,
                           const uint32_t *d_lcp, const uint8_t *d_queries, const uint64_t *d_q_off, uint32_t nq,
                           uint64_t q_bytes, uint32_t *d_len, uint32_t *d_start, uint32_t *d_end, void *stream) {
    TRY(match_args(c, n, d_text, d_sa, d_queries, d_q_off, nq, q_bytes, d_len, d_start, d_end));
    if (n > 0 && d_start && !d_lcp) return null_ptr(c);
    TRY(enter(c, stream));
    if (nq == 0 || q_bytes == 0) return leave(c, B200SA_OK);
    return leave(c, match_stats_core(c, d_text, (uint32_t)n, d_sa, d_lcp, d_queries, d_q_off, nq, q_bytes, d_len,
                                     d_start, d_end, TextEnd{(uint32_t)n}, nullptr, 0));
}

int b200sa_docs_match_stats_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_gsa,
                                const uint32_t *d_glcp, const uint32_t *d_doc_starts, uint32_t ndocs,
                                const uint8_t *d_queries, const uint64_t *d_q_off, uint32_t nq, uint64_t q_bytes,
                                uint32_t *d_len, uint32_t *d_start, uint32_t *d_end, void *stream) {
    TRY(match_args(c, n, d_text, d_gsa, d_queries, d_q_off, nq, q_bytes, d_len, d_start, d_end));
    if (n > 0 && ((d_start && !d_glcp) || !d_doc_starts)) return null_ptr(c);
    if (ndocs == 0 && n > 0) return no_docs(c);
    TRY(enter(c, stream));
    if (nq == 0 || q_bytes == 0) return leave(c, B200SA_OK);
    return leave(c, match_stats_core(c, d_text, (uint32_t)n, d_gsa, d_glcp, d_queries, d_q_off, nq, q_bytes, d_len,
                                     d_start, d_end, DocsEnd{d_doc_starts, ndocs, (uint32_t)n}, d_doc_starts, ndocs));
}

// nq >= 1.  Phases: match_check, smem_flag, smem_scan, smem_emit.
static int smems_core(b200sa_ctx *c, const uint64_t *d_q_off, uint32_t nq, uint64_t q_bytes, const uint32_t *d_len,
                      uint32_t min_len, uint64_t *d_offsets, uint32_t *d_qpos, uint64_t cap, uint64_t *total) {
    TRY(mark(c, "match_check"));
    TRY(match_check(c, d_q_off, nq, q_bytes));
    TRY(mark(c, "smem_flag"));
    TRY(ensure(c, c->p0, (q_bytes + 1) * 4));
    TRY(ensure(c, c->p1, (q_bytes + 1) * 4));
    uint32_t *flag = ptr<uint32_t>(c->p0), *exc = ptr<uint32_t>(c->p1), *d_total = ptr<uint32_t>(c->small) + 2;
    LAUNCH(c, k_smem_flag, cdiv(q_bytes + 1, BLK), d_len, d_q_off, nq, q_bytes, min_len, flag);
    TRY(mark(c, "smem_scan"));                          // q_bytes <= B200SA_MAX_N: a u32 sum
    TRY((dev_scan<OpSum>(c, SmemIn{flag}, SmemOut{exc}, q_bytes + 1, d_total)));
    TRY(read_words(c, d_total, 1));
    *total = c->h_pin[0];
    TRY(mark(c, "smem_emit"));
    const uint64_t items = std::max<uint64_t>(q_bytes, (uint64_t)nq + 1);
    LAUNCH(c, k_smem_emit, cdiv(items, BLK), flag, exc, d_q_off, nq, q_bytes,
           reinterpret_cast<unsigned long long *>(d_offsets), *total <= cap ? d_qpos : (uint32_t *)nullptr);
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

int b200sa_smems_dev(b200sa_ctx *c, const uint64_t *d_q_off, uint32_t nq, uint64_t q_bytes, const uint32_t *d_len,
                     uint32_t min_len, uint64_t *d_offsets, uint32_t *d_qpos, uint64_t cap, uint64_t *total,
                     void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!total || !d_offsets || (nq > 0 && !d_q_off) || (q_bytes > 0 && !d_len) || (cap > 0 && !d_qpos))
        return null_ptr(c);
    if (min_len == 0) return fail(c, B200SA_ERR_BAD_ARG, "smems: min_len must be at least 1");
    if (q_bytes > B200SA_MAX_N) return fail(c, B200SA_ERR_TOO_LARGE, "queries longer than 2^32-4096 bytes");
    TRY(enter(c, stream));
    *total = 0;
    if (nq == 0) return leave(c, empty_batch(c, d_offsets));
    return leave(c, smems_core(c, d_q_off, nq, q_bytes, d_len, min_len, d_offsets, d_qpos, cap, total));
}

// ------------------------------------------------------------ repeats (DESIGN 6b f-11)
static int repeat_args(b200sa_ctx *c, uint64_t n, const void *sa, const void *lcp) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!sa || !lcp)) return null_ptr(c);
    if (n > B200SA_MAX_N) return too_long(c);
    return B200SA_OK;
}

// n >= 1.  Phases: rep_lens.
static int repeat_lens_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t *d_rl) {
    TRY(mark(c, "rep_lens"));
    LAUNCH(c, k_rep_lens, cdiv(n, BLK), d_sa, d_lcp, n, d_rl);
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

int b200sa_repeat_lens_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t *d_rl,
                           void *stream) {
    TRY(repeat_args(c, n, d_sa, d_lcp));
    if (n > 0 && !d_rl) return null_ptr(c);
    TRY(enter(c, stream));
    if (n == 0) return leave(c, B200SA_OK);
    return leave(c, repeat_lens_core(c, (uint32_t)n, d_sa, d_lcp, d_rl));
}

// seg (p0) and, on request, the smallest (p1) and largest (g0) position of every segment, at its head's slot
static int repeat_segments(b200sa_ctx *c, uint32_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t L,
                           bool want_first, bool want_last) {
    TRY(ensure(c, c->p0, (size_t)n * 4));
    uint32_t *seg = ptr<uint32_t>(c->p0);
    TRY((dev_scan<OpMax>(c, RepSegIn{d_lcp, L}, RepSegOut{seg}, n, nullptr)));
    if (want_first) {
        TRY(ensure(c, c->p1, (size_t)n * 4));
        TRY((dev_scan<OpMax64>(c, RepExtIn<true>{d_sa, seg}, RepExtOut<true>{d_lcp, n, L, ptr<uint32_t>(c->p1)}, n,
                               nullptr)));
    }
    if (want_last) {
        TRY(ensure(c, c->g0, (size_t)n * 4));
        TRY((dev_scan<OpMax64>(c, RepExtIn<false>{d_sa, seg}, RepExtOut<false>{d_lcp, n, L, ptr<uint32_t>(c->g0)}, n,
                               nullptr)));
    }
    return B200SA_OK;
}

// n >= 1.  Phases: rep_count, rep_segments (with first / last), rep_emit.
static int repeat_runs_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t L,
                            uint32_t *d_start, uint32_t *d_end, uint32_t *d_first, uint32_t *d_last, uint64_t cap,
                            uint64_t *total) {
    TRY(ensure(c, c->small, 4096));
    uint32_t *d_total = ptr<uint32_t>(c->small) + 2;
    TRY(mark(c, "rep_count"));
    TRY((dev_scan<OpSum>(c, RepRunIn{d_lcp, n, L}, RepNoOut{}, n, d_total)));
    TRY(read_words(c, d_total, 1));
    *total = c->h_pin[0];
    if (*total > 0 && *total <= cap) {
        if (d_first || d_last) {
            TRY(mark(c, "rep_segments"));
            TRY(repeat_segments(c, n, d_sa, d_lcp, L, d_first != nullptr, d_last != nullptr));
        }
        TRY(mark(c, "rep_emit"));
        TRY((dev_scan<OpSum>(c, RepRunIn{d_lcp, n, L},
                             RepRunOut{d_lcp, n, L, d_start, d_end, d_first, d_last, ptr<uint32_t>(c->p1),
                                       ptr<uint32_t>(c->g0)},
                             n, nullptr)));
    }
    TRY(mark(c, "end"));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

int b200sa_repeat_runs_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t min_len,
                           uint32_t *d_start, uint32_t *d_end, uint32_t *d_first, uint32_t *d_last, uint64_t cap,
                           uint64_t *total, void *stream) {
    TRY(repeat_args(c, n, d_sa, d_lcp));
    if (!total || (cap > 0 && (!d_start || !d_end))) return null_ptr(c);
    if (min_len == 0) return fail(c, B200SA_ERR_BAD_ARG, "repeat runs: min_len must be at least 1");
    TRY(enter(c, stream));
    *total = 0;
    if (n == 0) return leave(c, B200SA_OK);
    return leave(c, repeat_runs_core(c, (uint32_t)n, d_sa, d_lcp, min_len, d_start, d_end, d_first, d_last, cap, total));
}

// n >= 1.  Phases: rep_check (with documents), rep_segments (every mode but ANY), rep_flag, rep_cover,
// rep_count, rep_emit.
static int duplicate_spans_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_sa, const uint32_t *d_lcp,
                                const uint32_t *d_starts, uint32_t ndocs, uint32_t L, int mode, uint32_t *d_begin,
                                uint32_t *d_end, uint64_t cap, uint64_t *total, uint64_t *covered) {
    TRY(ensure(c, c->small, 4096));
    uint32_t *words = ptr<uint32_t>(c->small);
    unsigned long long *d_total = reinterpret_cast<unsigned long long *>(words + 4);
    if (d_starts) {
        TRY(mark(c, "rep_check"));
        TRY(docs_check_dev(c, d_starts, ndocs, n));
    }
    // two bitmaps of n bits, padded to whole words: flagged positions, document starts
    const size_t bm_words = ((size_t)n + 31) / 32;
    TRY(ensure(c, c->g1, bm_words * 8));
    uint32_t *flagged = ptr<uint32_t>(c->g1), *doc_bits = flagged + bm_words;
    CU_TRY(c, cudaMemsetAsync(flagged, 0, bm_words * 8, c->stream));
    if (mode != REP_ANY) {
        TRY(mark(c, "rep_segments"));
        TRY(repeat_segments(c, n, d_sa, d_lcp, L, true, mode == REP_OTHER_DOC));
    }
    TRY(mark(c, "rep_flag"));
    const uint32_t *seg = ptr<uint32_t>(c->p0), *sf = ptr<uint32_t>(c->p1), *sl = ptr<uint32_t>(c->g0);
    const uint32_t grid = cdiv(n, BLK);
    switch (mode) {
        case REP_ANY: LAUNCH(c, k_rep_flag<REP_ANY>, grid, d_sa, d_lcp, n, L, seg, sf, sl, d_starts, ndocs, flagged); break;
        case REP_EARLIER: LAUNCH(c, k_rep_flag<REP_EARLIER>, grid, d_sa, d_lcp, n, L, seg, sf, sl, d_starts, ndocs, flagged); break;
        case REP_OTHER_DOC: LAUNCH(c, k_rep_flag<REP_OTHER_DOC>, grid, d_sa, d_lcp, n, L, seg, sf, sl, d_starts, ndocs, flagged); break;
        default: LAUNCH(c, k_rep_flag<REP_EARLIER_DOC>, grid, d_sa, d_lcp, n, L, seg, sf, sl, d_starts, ndocs, flagged); break;
    }
    if (d_starts) LAUNCH(c, k_rep_doc_bits, cdiv(ndocs, BLK), d_starts, ndocs, n, doc_bits);
    TRY(mark(c, "rep_cover"));                           // seg is dead: its buffer takes near
    TRY(ensure(c, c->p0, (size_t)n * 4));
    uint32_t *near = ptr<uint32_t>(c->p0);
    TRY((dev_scan<OpMax>(c, RepNearIn{flagged}, RepNearOut{near}, n, nullptr)));
    TRY(mark(c, "rep_count"));
    const RepCover C{near, doc_bits, n, L};
    TRY((dev_scan<OpSum64>(c, RepSpanIn{C}, RepSpanNoOut{}, n, d_total)));
    TRY(read_words(c, reinterpret_cast<const uint32_t *>(d_total), 2));
    *covered = c->h_pin[0];
    *total = c->h_pin[1];
    if (*total > 0 && *total <= cap) {
        TRY(mark(c, "rep_emit"));
        TRY((dev_scan<OpSum64>(c, RepSpanIn{C}, RepSpanOut{C, d_begin, d_end}, n, nullptr)));
    }
    TRY(mark(c, "end"));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

int b200sa_duplicate_spans_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp,
                               const uint32_t *d_doc_starts, uint32_t ndocs, uint32_t min_len, int mode,
                               uint32_t *d_begin, uint32_t *d_end, uint64_t cap, uint64_t *total, uint64_t *covered,
                               void *stream) {
    TRY(repeat_args(c, n, d_sa, d_lcp));
    if (!total || !covered || (cap > 0 && (!d_begin || !d_end)) || (ndocs > 0 && !d_doc_starts)) return null_ptr(c);
    if (min_len == 0) return fail(c, B200SA_ERR_BAD_ARG, "duplicate spans: min_len must be at least 1");
    if (mode < B200SA_REPEAT_ANY || mode > B200SA_REPEAT_EARLIER_DOC)
        return fail(c, B200SA_ERR_BAD_ARG, "duplicate spans: unknown mode");
    if (!d_doc_starts && mode >= B200SA_REPEAT_OTHER_DOC)
        return fail(c, B200SA_ERR_BAD_ARG, "duplicate spans: the document modes need doc_starts");
    if (d_doc_starts && ndocs == 0 && n > 0) return no_docs(c);
    TRY(enter(c, stream));
    *total = 0;
    *covered = 0;
    if (n == 0) return leave(c, B200SA_OK);
    return leave(c, duplicate_spans_core(c, (uint32_t)n, d_sa, d_lcp, d_doc_starts, ndocs, min_len, mode, d_begin, d_end,
                                         cap, total, covered));
}

// ------------------------------------------------------------ longest previous factor and LZ77 (DESIGN 6b f-12)
// n >= 1: the block minima of R (qbuf) and of lam (isa), then lpf / src.  Phases: lz_levels, lz_lpf.
static int lz_lpf_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t *d_lpf,
                       uint32_t *d_src) {
    AnsvLevels LR, LL;
    TRY(mark(c, "lz_levels"));
    TRY(ansv_levels(c, d_sa, n, &LR, c->qbuf));
    TRY(ansv_levels(c, d_lcp, n, &LL, c->isa));
    TRY(mark(c, "lz_lpf"));
    LAUNCH(c, k_lz_lpf, cdiv(n, BLK), LR, LL, n, d_lpf, d_src);
    CU_TRY(c, cudaGetLastError());
    return B200SA_OK;
}

int b200sa_lpf_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t *d_lpf,
                   uint32_t *d_src, void *stream) {
    TRY(repeat_args(c, n, d_sa, d_lcp));
    if (n > 0 && !d_lpf) return null_ptr(c);
    TRY(enter(c, stream));
    if (n == 0) return leave(c, B200SA_OK);
    int rc = lz_lpf_core(c, (uint32_t)n, d_sa, d_lcp, d_lpf, d_src);
    if (rc == B200SA_OK) rc = mark(c, "end");
    return leave(c, rc);
}

// n >= 1.  lpf (p0), src (p1), the jump arrays J (g0, g1: n + 1 each), the mark bitmap (v0).  Phases:
// lz_levels, lz_lpf, lz_parse, lz_count, lz_emit.
static int lz77_core(b200sa_ctx *c, uint32_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t *d_start,
                     uint32_t *d_len, uint32_t *d_src, uint64_t cap, uint64_t *total) {
    const uint32_t nwords = (uint32_t)(((uint64_t)n + 31) / 32);
    TRY(ensure(c, c->p0, (size_t)n * 4));
    TRY(ensure(c, c->p1, (size_t)n * 4));
    TRY(ensure(c, c->g0, ((size_t)n + 1) * 4));
    TRY(ensure(c, c->g1, ((size_t)n + 1) * 4));
    TRY(ensure(c, c->v0, (size_t)nwords * 4));
    TRY(ensure(c, c->small, 4096));
    uint32_t *lpf = ptr<uint32_t>(c->p0), *src = ptr<uint32_t>(c->p1), *marks = ptr<uint32_t>(c->v0);
    uint32_t *J[2] = {ptr<uint32_t>(c->g0), ptr<uint32_t>(c->g1)};
    uint32_t *state = ptr<uint32_t>(c->small) + 8, *d_total = state + 2;   // done, rounds, z
    TRY(lz_lpf_core(c, n, d_sa, d_lcp, lpf, src));
    TRY(mark(c, "lz_parse"));
    CU_TRY(c, cudaMemsetAsync(marks, 0, (size_t)nwords * 4, c->stream));
    CU_TRY(c, cudaMemsetAsync(state, 0, 8, c->stream));
    LAUNCH(c, k_lz_next, cdiv((uint64_t)n + 1, BLK), lpf, n, J[0], marks);
    int cur = 0;
    for (uint32_t b = n; b; b >>= 1, cur ^= 1) {         // bit_length(n) >= ceil(log2 z) rounds
        LAUNCH(c, k_lz_mark, cdiv(nwords, BLK), J[cur], n, marks, nwords, state);
        LAUNCH(c, k_lz_square, cdiv((uint64_t)n + 1, BLK), J[cur], n, J[cur ^ 1], state);
    }
    TRY(mark(c, "lz_count"));
    TRY((dev_scan<OpSum>(c, InPopcWords{marks}, LzNoOut{}, nwords, d_total)));
    CU_TRY(c, cudaGetLastError());
    TRY(read_words(c, state + 1, 2));
    c->stats.doubling_rounds = c->h_pin[0];
    *total = c->h_pin[1];
    if (*total > 0 && *total <= cap) {
        TRY(mark(c, "lz_emit"));
        TRY((dev_scan<OpSum>(c, InPopcWords{marks}, LzEmitOut{marks, lpf, src, d_start, d_len, d_src}, nwords,
                             nullptr)));
    }
    TRY(mark(c, "end"));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

int b200sa_lz77_dev(b200sa_ctx *c, uint64_t n, const uint32_t *d_sa, const uint32_t *d_lcp, uint32_t *d_start,
                    uint32_t *d_len, uint32_t *d_src, uint64_t cap, uint64_t *total, void *stream) {
    TRY(repeat_args(c, n, d_sa, d_lcp));
    if (!total || (cap > 0 && (!d_start || !d_len || !d_src))) return null_ptr(c);
    TRY(enter(c, stream));
    *total = 0;
    if (n == 0) return leave(c, B200SA_OK);
    return leave(c, lz77_core(c, (uint32_t)n, d_sa, d_lcp, d_start, d_len, d_src, cap, total));
}

// ------------------------------------------------------------ Burrows-Wheeler transform (DESIGN 6b f-13)
// nrows = n + k >= 1, k >= 1.  The gather (the L bytes in flag, the terminator bitmap in v0), then the
// compaction.  Phases: bwt_check (with documents), bwt_gather, bwt_compact (n > 0).
static int bwt_core(b200sa_ctx *c, uint32_t n, const uint8_t *d_text, const uint32_t *d_sa, const uint32_t *d_starts,
                    uint32_t k, uint8_t *d_bwt, uint32_t *d_term_rows, uint64_t *runs) {
    const uint32_t nrows = n + k, nwords = cdiv(nrows, 32);
    TRY(ensure(c, c->small, 4096));
    uint32_t *words = ptr<uint32_t>(c->small);
    unsigned long long *d_runs = reinterpret_cast<unsigned long long *>(words + 4);
    if (d_starts) {
        TRY(mark(c, "bwt_check"));
        TRY(docs_check_dev(c, d_starts, k, n));
    }
    TRY(ensure(c, c->flag, nrows));
    TRY(ensure(c, c->v0, (size_t)nwords * 4));
    uint8_t *lbyte = ptr<uint8_t>(c->flag);
    uint32_t *term_bm = ptr<uint32_t>(c->v0);
    TRY(mark(c, "bwt_gather"));
    if (runs) CU_TRY(c, cudaMemsetAsync(d_runs, 0, 8, c->stream));
    LAUNCH(c, k_bwt_gather, cdiv(nrows, BLK), BwtRows{d_text, d_sa, d_starts, n, k}, nrows, lbyte, term_bm, d_term_rows,
           runs ? d_runs : (unsigned long long *)nullptr);
    if (n > 0) {
        TRY(mark(c, "bwt_compact"));
        TRY((dev_scan<OpSum>(c, InPopcWords{term_bm}, BwtCompactOut{term_bm, lbyte, d_bwt, nrows}, nwords, nullptr)));
    }
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    if (runs) {
        TRY(read_words(c, reinterpret_cast<const uint32_t *>(d_runs), 2));
        *runs = pin_u64(c, 0);
    }
    return B200SA_OK;
}

int b200sa_bwt_dev(b200sa_ctx *c, uint64_t n, const uint8_t *d_text, const uint32_t *d_sa, const uint32_t *d_doc_starts,
                   uint32_t ndocs, uint8_t *d_bwt, uint32_t *d_term_rows, uint64_t *runs, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    const uint64_t k = d_doc_starts ? ndocs : 1;
    if ((n > 0 && (!d_text || !d_sa || !d_bwt)) || (k > 0 && !d_term_rows) || (ndocs > 0 && !d_doc_starts))
        return null_ptr(c);
    if (k == 0 && n > 0) return no_docs(c);
    if (n + k > B200SA_MAX_N) return fail(c, B200SA_ERR_TOO_LARGE, "bwt: text and terminators above 2^32-4096 rows");
    TRY(enter(c, stream));
    if (runs) *runs = 0;
    if (k == 0) return leave(c, B200SA_OK);              // no documents: no rows
    return leave(c, bwt_core(c, (uint32_t)n, d_text, d_sa, d_doc_starts, (uint32_t)k, d_bwt, d_term_rows, runs));
}

// The stable sorts of the inverse: the term rows (bits wide) or the bwt bytes (8 bits), by index.
template <class KeyF>
static int unbwt_sort(b200sa_ctx *c, KeyF kf, DevBuf &ka, DevBuf &va, DevBuf &kb, DevBuf &vb, uint32_t cnt, int bits,
                      uint32_t **kout, uint32_t **vout) {
    TRY(ensure(c, ka, (size_t)cnt * 4));
    TRY(ensure(c, va, (size_t)cnt * 4));
    TRY(ensure(c, kb, (size_t)cnt * 4));
    if (bits > 8) TRY(ensure(c, vb, (size_t)cnt * 4));    // one pass never writes vb
    uint32_t *a = ptr<uint32_t>(ka), *v = ptr<uint32_t>(va), *b = ptr<uint32_t>(kb), *w = ptr<uint32_t>(vb);
    return sort_pairs_from(c, kf, LoadIndex{}, a, v, b, w, cnt, bits, kout, vout);
}

constexpr uint32_t BWT_RULER_DEFAULT = 64;

// k >= 1.  Buffers: the sorted term rows (g0, g1, p1, rank: k entries), the sorted bytes (v0, v1, p0: n
// entries), psi / F (k64a: n + k u64), the ruler bitmap and its word prefix (isa), the ruler rows (qbuf),
// walk lengths (p0), the list (k64b, v0: two u64 per ruler), document starts (g1).  Phases: unbwt_sort,
// unbwt_walk, unbwt_rank, unbwt_emit.
static int unbwt_core(b200sa_ctx *c, uint32_t n, uint32_t k, const uint8_t *d_bwt, const uint32_t *d_term_rows,
                      uint8_t *d_text, uint32_t *d_starts_out) {
    const uint32_t nrows = n + k, nwords = cdiv(nrows, 32);
    TRY(ensure(c, c->small, 4096));
    // [0] check bits, [1] longest walk, [2, 4) rows covered (u64), [4] rulers, [8, 41) rounds that moved
    uint32_t *words = ptr<uint32_t>(c->small) + 16;
    CU_TRY(c, cudaMemsetAsync(words, 0, 48 * 4, c->stream));

    // 1. psi and F
    TRY(mark(c, "unbwt_sort"));
    uint32_t *ts, *tv, *fk = nullptr, *fu = nullptr;
    TRY(unbwt_sort(c, LoadArr<uint32_t>{d_term_rows}, c->g0, c->g1, c->p1, c->rank, k, bit_length(nrows - 1), &ts,
                   &tv));
    LAUNCH(c, k_bwt_terms_check, cdiv(k, BLK), ts, k, nrows, words);
    CU_TRY(c, cudaGetLastError());
    TRY(read_words(c, words, 1));
    if (c->h_pin[0]) return fail(c, B200SA_ERR_BAD_ARG, "unbwt: term_rows out of range or repeated");
    if (n > 0) TRY(unbwt_sort(c, BwtByteKey{d_bwt}, c->v0, c->v1, c->p0, c->p0, n, 8, &fk, &fu));
    TRY(ensure(c, c->k64a, (size_t)nrows * 8));
    unsigned long long *pf = ptr<unsigned long long>(c->k64a);
    LAUNCH(c, k_bwt_psi, cdiv(nrows, BLK), d_term_rows, ts, k, fk, fu, nrows, pf);

    // 2. rulers and their walks
    TRY(mark(c, "unbwt_walk"));
    uint32_t s = BWT_RULER_DEFAULT;
    if (const char *e = getenv("B200SA_BWT_RULER")) { long v = atol(e); if (v >= 1) s = v > 0xffffffffL ? 0xffffffffu : (uint32_t)v; }
    const BwtRuler isr{k, s, s <= n};
    TRY(ensure(c, c->isa, (size_t)nwords * 8));
    uint32_t *rbm = ptr<uint32_t>(c->isa), *wpre = rbm + nwords;
    LAUNCH(c, k_bwt_ruler_bits, cdiv(nrows, BLK), isr, nrows, rbm);
    TRY((dev_scan<OpSum>(c, InPopcWords{rbm}, OutStoreExcl{wpre}, nwords, words + 4)));
    TRY(read_words(c, words + 4, 1));
    const uint32_t m = c->h_pin[0];
    TRY(ensure(c, c->qbuf, (size_t)m * 4));
    TRY(ensure(c, c->p0, (size_t)m * 4));
    TRY(ensure(c, c->k64b, (size_t)m * 8));
    TRY(ensure(c, c->v0, (size_t)m * 8));
    uint32_t *rrow = ptr<uint32_t>(c->qbuf), *steps = ptr<uint32_t>(c->p0);
    unsigned long long *nv = ptr<unsigned long long>(c->k64b), *nv2 = ptr<unsigned long long>(c->v0);
    LAUNCH(c, k_bwt_ruler_list, cdiv(nwords, BLK), rbm, wpre, nwords, rrow);
    LAUNCH(c, k_bwt_walk, cdiv(m, BLK), pf, isr, rrow, rbm, wpre, m, nv, steps, words);

    // 3. ranking and the validity check
    TRY(mark(c, "unbwt_rank"));
    const int R = bit_length(m);                          // >= ceil(log2 m): every list of rulers is ranked
    for (int r = 0; r < R; r++) {
        LAUNCH(c, k_bwt_jump, cdiv(m, BLK), nv, m, k, nv2, words + 8, (uint32_t)r);
        std::swap(nv, nv2);
    }
    LAUNCH(c, k_bwt_valid, cdiv(m, BLK), nv, steps, m, k, reinterpret_cast<unsigned long long *>(words + 2), words);
    CU_TRY(c, cudaGetLastError());
    TRY(read_words(c, words, 8 + R));
    const uint64_t covered = pin_u64(c, 2);
    uint32_t rounds = 0;
    for (int r = 0; r < R; r++) rounds += c->h_pin[8 + r] ? 1u : 0u;
    c->stats.doubling_rounds = rounds;
    if (getenv("B200SA_TRACE"))
        fprintf(stderr, "[b200sa] unbwt: n=%u k=%u spacing=%u rulers=%u longest walk=%u rank rounds=%u\n", n, k, s, m,
                c->h_pin[1], rounds);
    if (c->h_pin[0] || covered != nrows)
        return fail(c, B200SA_ERR_BAD_ARG, "unbwt: (bwt, term_rows) is not the transform of any documents");

    // 4. document starts, then every ruler writes its segment
    TRY(mark(c, "unbwt_emit"));
    TRY(ensure(c, c->g1, (size_t)k * 4));
    uint32_t *starts = ptr<uint32_t>(c->g1);
    TRY((dev_scan<OpSum>(c, BwtLenIn{nv}, BwtStartsOut{starts, d_starts_out}, k, nullptr)));
    if (n > 0) LAUNCH(c, k_bwt_emit, cdiv(m, BLK), pf, rrow, steps, nv, starts, m, k, d_text);
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

int b200sa_unbwt_dev(b200sa_ctx *c, uint64_t n, uint32_t ndocs, const uint8_t *d_bwt, const uint32_t *d_term_rows,
                     uint8_t *d_text_out, uint32_t *d_doc_starts_out, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!d_term_rows || (n > 0 && (!d_bwt || !d_text_out))) return null_ptr(c);
    if (ndocs == 0) return fail(c, B200SA_ERR_BAD_ARG, "unbwt: ndocs must be at least 1");
    if (n + ndocs > B200SA_MAX_N) return fail(c, B200SA_ERR_TOO_LARGE, "unbwt: text and terminators above 2^32-4096 rows");
    TRY(enter(c, stream));
    return leave(c, unbwt_core(c, (uint32_t)n, ndocs, d_bwt, d_term_rows, d_text_out, d_doc_starts_out));
}

// ------------------------------------------------------------ approximate positions (DESIGN 6b f-14 .. f-22)
// B200SA_APPROX_BULGES: on, with t substitutions, d DNA bulges and r RNA bulges.
struct Bulges {
    bool on;
    uint32_t t, d, r;
};

// The k of a call as approx_args decodes it: the threshold (t + d + r with B200SA_APPROX_BULGES), B200SA_APPROX_BEST's
// slack, and the flags.
struct ApproxFlags {
    uint32_t k, s;
    bool edit, best, iupac, fixed, both, docs, align, loci;
    bool stage;                                          // docs || align || loci: the final lists go to staging
    Bulges bulges;
};

// The words of c->small through which the approximate search hands results from its kernels to the host; a u64
// takes two words, low word first.  [0] the range flag of DListChunks, [2, 4) the search's items, [4, 6) its total
// (the search clears [0, 6)); [8, 10) (batch size << 32) | batch bytes of best_batch, [10] the rounds where a query
// ended, [12, 14) the best rounds' total (the rounds clear [8, 14)); [16, 18) the least (offset << 8) | byte that
// iupac_canon rejects; [20, 22) the number of listed documents or alignment operations, [22] align_list's error
// word; [24] the longest query; [26, 28) the number of loci.
enum ApproxWord : uint32_t {
    AW_FLAG = 0, AW_ITEMS = 2, AW_TOTAL = 4, AW_BATCH = 8, AW_ENDED = 10, AW_BEST_TOTAL = 12, AW_IUPAC_BAD = 16,
    AW_LISTED = 20, AW_ALIGN_ERR = 22, AW_MMAX = 24, AW_LOCI = 26
};

// The checks of a call (nq >= 1, k its threshold): q_off on the device with q_off[nq] read back as *q_bytes,
// doc_starts (d_starts non-null for documents), and the sizes.  Phase approx_check.
static int approx_prep(b200sa_ctx *c, uint32_t n, const uint32_t *d_starts, uint32_t ndocs, const uint8_t *d_queries,
                       const uint64_t *d_q_off, uint32_t nq, uint32_t k, uint64_t *q_bytes) {
    TRY(mark(c, "approx_check"));
    TRY(ensure(c, c->small, 4096));
    CU_TRY(c, cudaMemcpyAsync(c->h_pin, d_q_off + nq, 8, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    *q_bytes = pin_u64(c, 0);
    TRY(match_check(c, d_q_off, nq, *q_bytes));          // q_off[0] = 0 and ascending
    if (d_starts && ndocs > 0) TRY(docs_check_dev(c, d_starts, ndocs, n));
    if (*q_bytes > B200SA_MAX_N) return fail(c, B200SA_ERR_TOO_LARGE, "queries longer than 2^32-4096 bytes");
    if (*q_bytes > 0 && !d_queries) return null_ptr(c);
    if ((uint64_t)nq * (k + 1) >= 0xFFFFFFFFull)
        return fail(c, B200SA_ERR_TOO_LARGE, "approx positions: nq * (k + 1) of 2^32 - 1 or more slots");
    return B200SA_OK;
}

// n = 0: every list is empty.
static int approx_nothing(b200sa_ctx *c, uint64_t *d_offsets, uint32_t nq) {
    CU_TRY(c, cudaMemsetAsync(d_offsets, 0, ((size_t)nq + 1) * 8, c->stream));
    TRY(mark(c, "end"));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

// B200SA_APPROX_IUPAC: the canonical copy of the q_bytes query bytes into c->icode (*out), or BAD_ARG naming the
// first byte that is not an IUPAC letter; with fixed (B200SA_APPROX_FIXED) the marks of the fixed bytes after it
// (*marks, k_iupac_marks).  Phase approx_check.
static int iupac_canon(b200sa_ctx *c, const uint8_t *d_queries, uint64_t q_bytes, bool fixed, const uint8_t **out,
                       const uint8_t **marks) {
    typedef unsigned long long u64;
    uint32_t *words = ptr<uint32_t>(c->small);
    TRY(ensure(c, c->icode, (size_t)q_bytes * (fixed ? 2 : 1)));
    CU_TRY(c, cudaMemsetAsync(words + AW_IUPAC_BAD, 0xFF, 8, c->stream));
    if (q_bytes > 0)
        LAUNCH(c, k_iupac_code, cdiv(q_bytes, BLK), d_queries, q_bytes, ptr<uint8_t>(c->icode),
               reinterpret_cast<u64 *>(words + AW_IUPAC_BAD));
    CU_TRY(c, cudaGetLastError());
    TRY(read_words(c, words + AW_IUPAC_BAD, 2));
    const uint64_t bad = pin_u64(c, 0);
    if (bad != ~0ull) {
        char m[200];
        snprintf(m, sizeof m,
                 "approx positions: with B200SA_APPROX_IUPAC, query byte 0x%02x at offset %llu of the queries is not "
                 "an IUPAC nucleotide code",
                 (unsigned)(bad & 0xFF), (unsigned long long)(bad >> 8));
        return fail(c, B200SA_ERR_BAD_ARG, m);
    }
    *out = ptr<uint8_t>(c->icode);
    if (fixed) {
        *marks = ptr<uint8_t>(c->icode) + q_bytes;
        if (q_bytes > 0)
            LAUNCH(c, k_iupac_marks, cdiv(q_bytes, BLK), d_queries, q_bytes, ptr<uint8_t>(c->icode) + q_bytes);
    }
    return B200SA_OK;
}

// The count (EMIT false) or emit pass of the search for the metric and the query alphabet (fixed: IUPAC queries
// with fixed symbols).
typedef void (*ApproxKernel)(ApproxArgs, uint32_t *, const unsigned long long *, int, unsigned long long *, uint32_t *);
template <bool EMIT>
static ApproxKernel approx_kernel(bool edit, bool iupac, bool fixed) {
    if (fixed) return edit ? k_approx_edit_iupac_fixed<EMIT> : k_approx_iupac_fixed<EMIT>;
    if (iupac) return edit ? k_approx_edit_iupac<EMIT> : k_approx_iupac<EMIT>;
    return edit ? k_approx_edit<EMIT> : k_approx<EMIT>;
}

// B200SA_APPROX_BULGES: the count (EMIT false) or emit pass of k_approx_bulge over the items, for the query alphabet.
template <bool EMIT>
static void launch_bulge(b200sa_ctx *c, bool iupac, bool fixed, uint64_t items, const BulgeArgs &B, uint32_t *cnt,
                         const unsigned long long *item_off, int pbits, unsigned long long *key, uint32_t *val) {
    typedef void (*Kernel)(BulgeArgs, uint32_t *, const unsigned long long *, int, unsigned long long *, uint32_t *);
    const Kernel kern = fixed   ? k_approx_bulge<EMIT, FixedIupacPieces>
                        : iupac ? k_approx_bulge<EMIT, IupacPieces>
                                : k_approx_bulge<EMIT, CutPieces>;
    kern<<<(uint32_t)cdiv(items, BULGE_WARPS), BULGE_BLK, 0, c->stream>>>(B, cnt, item_off, pbits, key, val);
    c->launches++;
}

// One search of nq >= 1 queries at threshold k on n >= 1 bytes: d_offsets (nq + 1) and *total, read back.  When
// 0 < total <= cap it also emits and sorts: *ko / *vo then hold the keys (q << *pbits) | p in (q, p) order and
// their distances.  Phases: approx_pieces, approx_scan, approx_count, and approx_emit, approx_sort when it
// emits.  B200SA_APPROX_EDIT picks k_approx_edit over k_approx; iupac (d_queries then the canonical copy) picks
// the pieces of k_iupac_pieces and the kernels' IUPAC instantiations; d_fixed, the marks of the queries' fixed
// symbols (B200SA_APPROX_FIXED, with iupac) or NULL, their fixed instantiations, with the pointer after the piece
// table (iupac_marks); bg.on (B200SA_APPROX_BULGES, k = t + d + r) the layered verification of k_approx_bulge in
// place of the metric's; everything else is shared.
template <class EndF>
static int approx_search(b200sa_ctx *c, const uint8_t *d_text, uint32_t n, const uint32_t *d_sa,
                         const uint32_t *d_starts, uint32_t ndocs, const uint8_t *d_queries, const uint64_t *d_q_off,
                         const uint8_t *d_fixed, uint32_t nq, uint32_t k, bool edit, bool iupac, uint64_t *d_offsets,
                         uint64_t cap,
                         uint64_t *total, EndF end, uint64_t **ko, uint32_t **vo, int *pbits_out,
                         Bulges bg = Bulges{}) {
    typedef unsigned long long u64;
    uint32_t *words = ptr<uint32_t>(c->small);
    const uint32_t P = k + 1;
    const uint64_t nslots = (uint64_t)nq * P;
    TRY(mark(c, "approx_pieces"));
    // with iupac the piece table follows pe, and with d_fixed the pointer to the marks follows the table
    TRY(ensure(c, c->p1, (size_t)nslots * (iupac ? 16 : 8) + (d_fixed ? 8 : 0)));
    uint32_t *ps = ptr<uint32_t>(c->p1), *pe = ps + nslots;
    if (iupac) {
        LAUNCH(c, (k_iupac_pieces<EndF>), cdiv(nq, BLK), d_text, n, d_sa, d_queries, d_q_off, nq, P, ps, pe,
               reinterpret_cast<uint2 *>(pe + nslots), end);
        if (d_fixed)
            CU_TRY(c, cudaMemcpyAsync(pe + 3 * nslots, &d_fixed, sizeof d_fixed, cudaMemcpyHostToDevice, c->stream));
    } else {
        LAUNCH(c, (k_approx_pieces<EndF>), cdiv(nslots, BLK), d_text, n, d_sa, d_queries, d_q_off, nq, P, ps, pe, end);
    }
    TRY(mark(c, "approx_scan"));
    CU_TRY(c, cudaMemsetAsync(words + AW_FLAG, 0, (AW_TOTAL + 2 - AW_FLAG) * 4, c->stream));
    TRY(ensure(c, c->k64a, ((size_t)nslots + 1) * 8));
    u64 *item_start = ptr<u64>(c->k64a), *d_items = reinterpret_cast<u64 *>(words + AW_ITEMS),
        *d_total = reinterpret_cast<u64 *>(words + AW_TOTAL);
    TRY((dev_scan<OpSum64>(c, DListChunks{ps, pe, (uint32_t)nslots, n, words + AW_FLAG}, OutStoreExcl64{item_start},
                           nslots + 1, d_items)));
    TRY(read_words(c, words + AW_ITEMS, 2));
    const uint64_t items = pin_u64(c, 0);
    if (items > (uint64_t)0x7fffffff * NWARP)
        return fail(c, B200SA_ERR_TOO_LARGE, "approx positions: more than 2^31 * 8 chunks of 1024 candidates in one batch");
    if (bg.on && items > (uint64_t)0x7fffffff * BULGE_WARPS)
        return fail(c, B200SA_ERR_TOO_LARGE, "approx positions: with B200SA_APPROX_BULGES, more than 2^31 * 4 chunks of "
                                             "1024 candidates in one batch");
    TRY(mark(c, "approx_count"));
    TRY(ensure(c, c->p0, (size_t)items * 4));
    TRY(ensure(c, c->k64b, ((size_t)items + 1) * 8));
    uint32_t *cnt = ptr<uint32_t>(c->p0);
    u64 *item_off = ptr<u64>(c->k64b);
    const bool fixed = d_fixed != nullptr;
    const ApproxArgs A{d_text, d_sa, d_starts, ndocs, n, d_queries, d_q_off, (uint32_t)nslots, P, k, ps, pe,
                       item_start, items};
    const int pbits = bit_length(n - 1);
    const BulgeArgs B{A, bg.t, bg.d, bg.r};
    if (items && bg.on)
        launch_bulge<false>(c, iupac, fixed, items, B, cnt, nullptr, pbits, nullptr, nullptr);
    else if (items)
        LAUNCH(c, approx_kernel<false>(edit, iupac, fixed), cdiv(items, NWARP), A, cnt, (const u64 *)nullptr, pbits,
               (u64 *)nullptr, (uint32_t *)nullptr);
    TRY((dev_scan<OpSum64>(c, InCount64{cnt, items}, OutStoreExcl64{item_off}, items + 1, d_total)));
    LAUNCH(c, k_dlist_qoff, cdiv((uint64_t)nq + 1, BLK), item_start, item_off, nq, P,
           reinterpret_cast<u64 *>(d_offsets));
    TRY(read_words(c, words + AW_TOTAL, 2));
    *total = pin_u64(c, 0);
    *pbits_out = pbits;
    if (*total > 0 && *total <= cap) {
        TRY(mark(c, "approx_emit"));
        TRY(ensure(c, c->g0, (size_t)*total * 8));
        TRY(ensure(c, c->g1, (size_t)*total * 8));
        TRY(ensure(c, c->v0, (size_t)*total * 4));
        TRY(ensure(c, c->v1, (size_t)*total * 4));
        if (bg.on)
            launch_bulge<true>(c, iupac, fixed, items, B, cnt, item_off, pbits, ptr<u64>(c->g0), ptr<uint32_t>(c->v0));
        else
            LAUNCH(c, approx_kernel<true>(edit, iupac, fixed), cdiv(items, NWARP), A, cnt, (const u64 *)item_off,
                   pbits, ptr<u64>(c->g0), ptr<uint32_t>(c->v0));
        TRY(mark(c, "approx_sort"));                     // by (q, p)
        TRY(sort_pairs<uint64_t>(c, ptr<uint64_t>(c->g0), ptr<uint32_t>(c->v0), ptr<uint64_t>(c->g1),
                                 ptr<uint32_t>(c->v1), *total, bit_length(nq - 1) + pbits, ko, vo));
    }
    return B200SA_OK;
}

// B200SA_APPROX_BOTH_STRANDS: the doubled batch of 2 nq queries and 2 q_bytes bytes must fit BestPick's scan word
// (bytes below 2^32) and the slot count.  Phase approx_check, before any kernel reads the queries.
static int strand_check(b200sa_ctx *c, uint64_t q_bytes, uint32_t nq, uint32_t k) {
    if (q_bytes > B200SA_MAX_N / 2)
        return fail(c, B200SA_ERR_TOO_LARGE,
                    "approx positions: with B200SA_APPROX_BOTH_STRANDS, queries longer than (2^32-4096) / 2 bytes");
    if (2ull * nq * (k + 1) >= 0xFFFFFFFFull)
        return fail(c, B200SA_ERR_TOO_LARGE,
                    "approx positions: with B200SA_APPROX_BOTH_STRANDS, 2 * nq * (k + 1) of 2^32 - 1 or more slots");
    return B200SA_OK;
}

// The doubled batch (strand.cuh) of the nq queries in c->strand: *eq / *eoff its 2 q_bytes bytes and 2 nq + 1
// offsets, *doff room for the 2 nq + 1 offsets of its search.  canon: d_queries is the IUPAC canonical copy.
// fixed (B200SA_APPROX_FIXED): the marks of d_queries, doubled after the bytes into *efx by the same kernel, whose
// complement leaves the bytes 0 and 1 as they are, so rc(q)'s marks are q's reversed.  Phase strand_queries.
static int strand_queries(b200sa_ctx *c, const uint8_t *d_queries, const uint64_t *d_q_off, uint32_t nq,
                          uint64_t q_bytes, bool canon, const uint8_t *fixed, const uint8_t **eq,
                          const uint64_t **eoff, uint64_t **doff, const uint8_t **efx) {
    TRY(mark(c, "strand_queries"));
    const size_t ne1 = (size_t)2 * nq + 1;
    TRY(ensure(c, c->strand, ne1 * 16 + (size_t)q_bytes * (fixed ? 4 : 2)));
    uint64_t *o2 = ptr<uint64_t>(c->strand);
    uint8_t *q2 = reinterpret_cast<uint8_t *>(o2 + 2 * ne1);
    LAUNCH(c, k_strand_queries, cdiv((uint64_t)nq * 32, BLK), d_queries, d_q_off, nq, canon, q2, o2);
    if (fixed) {                                         // writes the same offsets again
        LAUNCH(c, k_strand_queries, cdiv((uint64_t)nq * 32, BLK), fixed, d_q_off, nq, false, q2 + 2 * q_bytes, o2);
        *efx = q2 + 2 * q_bytes;
    }
    *eq = q2;
    *eoff = o2;
    *doff = o2 + ne1;
    return B200SA_OK;
}

// The caller's offsets (offsets[q] = doff[2q]) and, when emitted, the both-strand lists from the total hits of the
// doubled batch at its offsets doff (src: the sorted keys or the staged positions, val their distances).
// Phase strand_merge.
template <class Src>
static int strand_merge(b200sa_ctx *c, Src src, const uint32_t *val, uint64_t total, bool emitted,
                        const uint64_t *doff, uint32_t nq, uint64_t *d_offsets, uint32_t *d_pos, uint32_t *d_mis) {
    typedef unsigned long long u64;
    TRY(mark(c, "strand_merge"));
    LAUNCH(c, k_strand_offsets, cdiv((uint64_t)nq + 1, BLK), (const u64 *)doff, nq, reinterpret_cast<u64 *>(d_offsets));
    if (emitted)
        LAUNCH(c, k_strand_merge<Src>, cdiv(total, BLK), src, val, total, (const u64 *)doff, 2 * nq, d_pos, d_mis);
    return B200SA_OK;
}

// B200SA_APPROX_DOCUMENTS: the offsets of the final hit lists, which the search or the scan of the best rounds
// writes in place of the caller's.
static int adocs_offsets(b200sa_ctx *c, uint32_t nq, uint64_t **hoff) {
    TRY(ensure(c, c->adoff, ((size_t)nq + 1) * 8));
    *hoff = ptr<uint64_t>(c->adoff);
    return B200SA_OK;
}

// B200SA_APPROX_DOCUMENTS: the staging of htotal >= 1 final hits in c->adocs, laid out as the segment scan
// (htotal + 1 u64), then the positions *hpos, the distances *hmis and the marks (htotal u32 each).
static int adocs_stage(b200sa_ctx *c, uint64_t htotal, uint32_t **hpos, uint32_t **hmis) {
    TRY(ensure(c, c->adocs, ((size_t)htotal + 1) * 8 + (size_t)htotal * 12));
    *hpos = reinterpret_cast<uint32_t *>(ptr<uint64_t>(c->adocs) + htotal + 1);
    *hmis = *hpos + htotal;
    return B200SA_OK;
}

// B200SA_APPROX_DOCUMENTS: the staged final lists (*total hits at offsets hoff, from adocs_stage) reduced per
// (query, document) into the caller's offsets and, when the listing fits cap, d_pos and d_mis; *total becomes the
// number of listed documents.  Phases adocs_mark (marks, scan, offsets) and adocs_emit.
static int adocs_reduce(b200sa_ctx *c, const uint32_t *d_starts, uint32_t ndocs, uint32_t nq, const uint64_t *hoff,
                        uint64_t *d_offsets, uint32_t *d_pos, uint32_t *d_mis, uint64_t cap, uint64_t *total) {
    typedef unsigned long long u64;
    const uint64_t htotal = *total;
    TRY(mark(c, "adocs_mark"));
    if (htotal == 0) {
        CU_TRY(c, cudaMemsetAsync(d_offsets, 0, ((size_t)nq + 1) * 8, c->stream));
        return B200SA_OK;
    }
    u64 *seg = ptr<u64>(c->adocs);
    const uint32_t *hpos = reinterpret_cast<const uint32_t *>(seg + htotal + 1), *hmis = hpos + htotal;
    uint32_t *marks = reinterpret_cast<uint32_t *>(seg + htotal + 1) + 2 * htotal;
    uint32_t *words = ptr<uint32_t>(c->small);
    LAUNCH(c, k_adocs_mark, cdiv(htotal, BLK), hpos, htotal, (const u64 *)hoff, nq, d_starts, ndocs, marks);
    TRY((dev_scan<OpSum64>(c, InCount64{marks, htotal}, OutStoreExcl64{seg}, htotal + 1,
                           reinterpret_cast<u64 *>(words + AW_LISTED))));
    LAUNCH(c, k_adocs_offsets, cdiv((uint64_t)nq + 1, BLK), (const u64 *)hoff, (const u64 *)seg, nq,
           reinterpret_cast<u64 *>(d_offsets));
    TRY(read_words(c, words + AW_LISTED, 2));
    *total = pin_u64(c, 0);
    if (*total > cap) return B200SA_OK;
    TRY(mark(c, "adocs_emit"));
    uint32_t *least = d_mis ? marks : nullptr;           // the marks are spent; their room holds the least words
    if (least) CU_TRY(c, cudaMemsetAsync(least, 0xFF, (size_t)*total * 4, c->stream));
    LAUNCH(c, k_adocs_emit, cdiv(htotal, BLK), hpos, hmis, htotal, (const u64 *)seg, d_starts, ndocs, d_pos, least);
    if (least) LAUNCH(c, k_adocs_dist, cdiv(*total, BLK), (const uint32_t *)least, *total, d_mis);
    return B200SA_OK;
}

// B200SA_APPROX_ALIGN: the longest of the nq queries into *mmax, and the query-length limits.  Phase approx_check.
static int align_check(b200sa_ctx *c, const uint64_t *d_q_off, uint32_t nq, bool edit, uint32_t *mmax) {
    uint32_t *words = ptr<uint32_t>(c->small);
    CU_TRY(c, cudaMemsetAsync(words + AW_MMAX, 0, 4, c->stream));
    LAUNCH(c, k_align_mmax, cdiv((uint64_t)nq, BLK), d_q_off, nq, words + AW_MMAX);
    TRY(read_words(c, words + AW_MMAX, 1));
    *mmax = c->h_pin[0];
    if (*mmax > (1u << 27) - 1)
        return fail(c, B200SA_ERR_TOO_LARGE,
                    "approx positions: with B200SA_APPROX_ALIGN, a query longer than 2^27 - 1 bytes");
    if (edit && *mmax > B200SA_APPROX_ALIGN_MAX_M)
        return fail(c, B200SA_ERR_TOO_LARGE,
                    "approx positions: with B200SA_APPROX_ALIGN and B200SA_APPROX_EDIT, a query longer than "
                    "B200SA_APPROX_ALIGN_MAX_M bytes");
    return B200SA_OK;
}

// B200SA_APPROX_ALIGN: the staged final lists (*total hits at offsets hoff, from adocs_stage) aligned into the
// caller's offsets and, when the listing fits cap, d_pos and d_mis; *total becomes the number of operations.  qs:
// the queries (the canonical copy with iupac), k the threshold, mmax the longest query.  Phases align_count,
// align_scan and align_emit.  fixed: the marks of qs with B200SA_APPROX_FIXED (k_align_edit<true>), after qs in
// its buffer; else NULL.  bg.on (B200SA_APPROX_BULGES, k = t + d + r): k_align_bulge, over batches of hits whose
// DP rows fit ALIGN_BULGE_SCRATCH bytes.
constexpr size_t ALIGN_BULGE_SCRATCH = 64u << 20;
static int align_list(b200sa_ctx *c, const uint8_t *d_text, uint32_t n, const uint32_t *d_starts, uint32_t ndocs,
                      const uint8_t *qs, const uint64_t *d_q_off, const uint8_t *fixed, uint32_t nq, uint32_t k,
                      bool edit, bool iupac, uint32_t mmax, const uint64_t *hoff, uint64_t *d_offsets,
                      uint32_t *d_pos, uint32_t *d_mis, uint64_t cap, uint64_t *total, Bulges bg) {
    typedef unsigned long long u64;
    const uint64_t htotal = *total;
    TRY(mark(c, "align_count"));
    if (htotal == 0) {
        CU_TRY(c, cudaMemsetAsync(d_offsets, 0, ((size_t)nq + 1) * 8, c->stream));
        return B200SA_OK;
    }
    u64 *seg = ptr<u64>(c->adocs);
    uint32_t *hpos = reinterpret_cast<uint32_t *>(seg + htotal + 1), *hmis = hpos + htotal, *cnt = hmis + htotal;
    uint32_t *words = ptr<uint32_t>(c->small);
    const uint32_t stride = 2 * k + 1;
    TRY(ensure(c, c->aops, (size_t)htotal * stride * 4));
    CU_TRY(c, cudaMemsetAsync(words + AW_ALIGN_ERR, 0, 4, c->stream));
    const AlignArgs A{d_text, d_starts, ndocs, n, qs, d_q_off, nq, fixed ? (uint32_t)(fixed - qs) : 0u,
                      (const u64 *)hoff, hpos, hmis, htotal, iupac, stride, ptr<uint32_t>(c->aops), cnt,
                      words + AW_ALIGN_ERR};
    if (bg.on) {
        const uint32_t rows = mmax + 1;
        const size_t per_hit = (size_t)rows * (bg.d + bg.r + 1) * (bg.d + 1) * (bg.r + 1);
        const uint64_t batch = std::max<uint64_t>(1, ALIGN_BULGE_SCRATCH / per_hit);
        TRY(ensure(c, c->abulge, (size_t)std::min<uint64_t>(batch, htotal) * per_hit));
        for (uint64_t h0 = 0; h0 < htotal; h0 += batch) {
            const uint64_t h1 = std::min(htotal, h0 + batch);
            if (fixed)
                LAUNCH(c, k_align_bulge<true>, cdiv(h1 - h0, BLK), A, bg.t, bg.d, bg.r, h0, h1, rows,
                       ptr<uint8_t>(c->abulge));
            else
                LAUNCH(c, k_align_bulge<false>, cdiv(h1 - h0, BLK), A, bg.t, bg.d, bg.r, h0, h1, rows,
                       ptr<uint8_t>(c->abulge));
        }
    } else if (edit) {
        // 16 bytes of choices per query row and warp: as many warps per block (up to 8) as fit 48 KB, at least one
        const size_t per_warp = (size_t)max(mmax, 1u) * 16;
        const uint32_t aw = (uint32_t)std::max<size_t>(1, std::min<size_t>(NWARP, 49152 / per_warp));
        const size_t smem = per_warp * aw;
        void (*kernel)(AlignArgs, uint32_t) = fixed ? k_align_edit<true> : k_align_edit<false>;
        if (smem > 49152)
            CU_TRY(c, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kernel<<<(uint32_t)cdiv(htotal, aw), aw * 32, smem, c->stream>>>(A, max(mmax, 1u));
        c->launches++;
    } else {
        LAUNCH(c, k_align_hamming, cdiv(htotal, BLK), A);
    }
    TRY(mark(c, "align_scan"));
    TRY((dev_scan<OpSum64>(c, InCount64{cnt, htotal}, OutStoreExcl64{seg}, htotal + 1,
                           reinterpret_cast<u64 *>(words + AW_LISTED))));
    LAUNCH(c, k_adocs_offsets, cdiv((uint64_t)nq + 1, BLK), (const u64 *)hoff, (const u64 *)seg, nq,
           reinterpret_cast<u64 *>(d_offsets));
    TRY(read_words(c, words + AW_LISTED, AW_ALIGN_ERR + 1 - AW_LISTED));
    if (c->h_pin[AW_ALIGN_ERR - AW_LISTED])
        return fail(c, B200SA_ERR_INTERNAL, "approx positions: with B200SA_APPROX_ALIGN, an alignment's cost differs "
                                            "from its hit's distance");
    *total = pin_u64(c, 0);
    if (*total > cap) return B200SA_OK;
    TRY(mark(c, "align_emit"));
    LAUNCH(c, k_align_emit, cdiv(htotal, BLK), (const uint32_t *)hpos, (const uint32_t *)hmis, htotal,
           (const u64 *)seg, (const uint32_t *)cnt, (const uint32_t *)ptr<uint32_t>(c->aops), stride, d_pos, d_mis);
    return B200SA_OK;
}

// B200SA_APPROX_LOCI: the staged final lists (*total hits at offsets hoff, from adocs_stage) cut to one hit per
// locus (loci.cuh); q_off gives each query's length.  *total becomes the number of loci.  With align the
// representatives replace the staged lists, for align_list, at the offsets *loff; else they go to the caller's
// offsets and, when they fit cap, d_pos and d_mis.  c->loci holds the least keys (8 bytes per hit), the scan of the
// marks (8 per hit), the offsets with align (8 per query) and the marks, then heads (4 per hit).  Phases loci_mark
// (three scans and the offsets) and loci_emit.
static int loci_reduce(b200sa_ctx *c, const uint32_t *d_starts, uint32_t ndocs, const uint64_t *d_q_off, uint32_t nq,
                       const uint64_t *hoff, bool align, uint64_t *d_offsets, uint32_t *d_pos, uint32_t *d_mis,
                       uint64_t cap, uint64_t *total, const uint64_t **loff) {
    typedef unsigned long long u64;
    const uint64_t htotal = *total;
    *loff = hoff;
    TRY(mark(c, "loci_mark"));
    if (htotal == 0) {
        if (!align) CU_TRY(c, cudaMemsetAsync(d_offsets, 0, ((size_t)nq + 1) * 8, c->stream));
        return B200SA_OK;
    }
    if (htotal >= 0xFFFFFFFFull)
        return fail(c, B200SA_ERR_TOO_LARGE, "approx positions: with B200SA_APPROX_LOCI, 2^32 - 1 or more hits");
    const size_t noff = align ? (size_t)nq + 1 : 0;
    TRY(ensure(c, c->loci, (size_t)htotal * 20 + 8 + noff * 8));
    u64 *least = ptr<u64>(c->loci), *keep = least + htotal, *aoff = keep + htotal + 1;
    uint32_t *marks = reinterpret_cast<uint32_t *>(aoff + noff);
    const uint32_t *hpos = reinterpret_cast<const uint32_t *>(ptr<u64>(c->adocs) + htotal + 1), *hmis = hpos + htotal;
    uint32_t *words = ptr<uint32_t>(c->small);
    const u64 *ho = reinterpret_cast<const u64 *>(hoff);
    CU_TRY(c, cudaMemsetAsync(least, 0xFF, (size_t)htotal * 8, c->stream));
    TRY((dev_scan<OpMax2x32>(c, LociPrevIn{hmis},
                             LociPrevOut{hpos, hmis, ho, reinterpret_cast<const u64 *>(d_q_off), nq, d_starts, ndocs,
                                         marks},
                             htotal, nullptr)));
    TRY((dev_scan<OpMax2x32>(c, LociHeadIn{hmis, marks}, LociHeadOut{hpos, hmis, marks, least}, htotal, nullptr)));
    TRY((dev_scan<OpSum64>(c, LociKeepIn{hpos, hmis, marks, least, htotal}, OutStoreExcl64{keep}, htotal + 1,
                           reinterpret_cast<u64 *>(words + AW_LOCI))));
    u64 *off = align ? aoff : reinterpret_cast<u64 *>(d_offsets);
    LAUNCH(c, k_adocs_offsets, cdiv((uint64_t)nq + 1, BLK), ho, (const u64 *)keep, nq, off);
    TRY(read_words(c, words + AW_LOCI, 2));
    *total = pin_u64(c, 0);
    if (align) {                          // through the spent keys, then into the staging's layout for *total hits
        *loff = reinterpret_cast<const uint64_t *>(off);
        TRY(mark(c, "loci_emit"));
        uint32_t *kpos = reinterpret_cast<uint32_t *>(least), *kmis = kpos + *total;
        LAUNCH(c, k_loci_emit, cdiv(htotal, BLK), hpos, hmis, htotal, (const u64 *)keep, kpos, kmis);
        uint32_t *spos, *smis;
        TRY(adocs_stage(c, *total, &spos, &smis));
        CU_TRY(c, cudaMemcpyAsync(spos, kpos, (size_t)*total * 8, cudaMemcpyDeviceToDevice, c->stream));
        return B200SA_OK;
    }
    if (*total > cap) return B200SA_OK;
    TRY(mark(c, "loci_emit"));
    LAUNCH(c, k_loci_emit, cdiv(htotal, BLK), hpos, hmis, htotal, (const u64 *)keep, d_pos, d_mis);
    return B200SA_OK;
}

// The batch a BestPick selects: *nb queries, map[i] the query of entry i; their bytes and offsets at *bq / *boff,
// the call's own arrays when every query is picked, else gathered into c->qbuf and coff.  Pick: BestPick, or
// StrandPick over the entries of the doubled batch.  fx (B200SA_APPROX_FIXED, else NULL): the queries' marks,
// which *bfx gets in the same way, gathered into fx_out.
template <class Pick>
static int best_batch(b200sa_ctx *c, const uint8_t *d_queries, const uint64_t *d_q_off, const uint8_t *fx,
                      uint32_t nq, Pick pick, uint32_t *map, uint64_t *coff, uint8_t *fx_out, uint32_t *nb,
                      const uint8_t **bq, const uint64_t **boff, const uint8_t **bfx) {
    typedef unsigned long long u64;
    uint32_t *words = ptr<uint32_t>(c->small);
    TRY((dev_scan<OpSum64>(c, pick, BestPickOut{nq, map, coff}, (uint64_t)nq + 1,
                           reinterpret_cast<u64 *>(words + AW_BATCH))));
    TRY(read_words(c, words + AW_BATCH, 2));
    *nb = (uint32_t)(pin_u64(c, 0) >> 32);
    *bq = d_queries;
    *boff = d_q_off;
    *bfx = fx;
    if (*nb == nq || *nb == 0) return B200SA_OK;
    LAUNCH(c, k_best_gather, cdiv((uint64_t)*nb * 32, BLK), d_queries, d_q_off, (const uint32_t *)map,
           (const uint64_t *)coff, *nb, ptr<uint8_t>(c->qbuf));
    if (fx) {
        LAUNCH(c, k_best_gather, cdiv((uint64_t)*nb * 32, BLK), fx, d_q_off, (const uint32_t *)map,
               (const uint64_t *)coff, *nb, fx_out);
        *bfx = fx_out;
    }
    *bq = ptr<uint8_t>(c->qbuf);
    *boff = coff;
    return B200SA_OK;
}

// The ne entries the search runs on: the queries, or with B200SA_APPROX_BOTH_STRANDS the doubled batch of
// strand_queries; q their bytes, off their offsets, out the offsets of their lists, fx the marks of their fixed
// symbols with B200SA_APPROX_FIXED (else NULL).
struct ApproxEntries { const uint8_t *q; const uint64_t *off; uint64_t *out; uint32_t ne; const uint8_t *fx; };

// Where the final lists land: their offsets off, positions pos and distances mis, written when 0 < total <= cap.
// The caller's arrays and cap, or with B200SA_APPROX_DOCUMENTS or _ALIGN the offsets in c->adoff and every hit, even
// at cap = 0, in the staging of adocs_stage.
struct ApproxFinal { uint64_t *off; uint32_t *pos, *mis; uint64_t cap; };

// Without B200SA_APPROX_BEST: one search of the entries at the threshold, whose sorted keys k_approx_gather, or with
// B200SA_APPROX_BOTH_STRANDS k_strand_merge, writes as the final lists.  Phases: the search's; strand_merge with
// both strands.
template <class EndF>
static int approx_plain(b200sa_ctx *c, const uint8_t *d_text, uint32_t n, const uint32_t *d_sa,
                        const uint32_t *d_starts, uint32_t ndocs, EndF end, const ApproxFlags &f,
                        const ApproxEntries &e, uint32_t nq, ApproxFinal fin, uint64_t *total) {
    typedef unsigned long long u64;
    uint64_t *ko = nullptr;
    uint32_t *vo = nullptr;
    int pbits = 0;
    TRY(approx_search(c, d_text, n, d_sa, d_starts, ndocs, e.q, e.off, e.fx, e.ne, f.k, f.edit, f.iupac, e.out,
                      fin.cap, total, end, &ko, &vo, &pbits, f.bulges));
    const bool emitted = *total > 0 && *total <= fin.cap;
    if (f.stage && emitted) TRY(adocs_stage(c, *total, &fin.pos, &fin.mis));
    if (f.both)
        TRY(strand_merge(c, StrandKeys{(const u64 *)ko, pbits}, vo, *total, emitted, e.out, nq, fin.off, fin.pos,
                         fin.mis));
    else if (emitted)
        LAUNCH(c, k_approx_gather, cdiv(*total, BLK), (const u64 *)ko, (const uint32_t *)vo, *total,
               (u64)((1ull << pbits) - 1), fin.pos, fin.mis);
    return B200SA_OK;
}

// B200SA_APPROX_BEST: rounds t = 0 .. threshold over the live queries (best.cuh), then one emission per distinct
// final threshold, whose groups k_best_scatter moves to their entries' lists.  With B200SA_APPROX_BOTH_STRANDS a
// query and its reverse complement are live as a pair with one best (strand.cuh), the groups scatter into
// c->sstage and one k_strand_merge writes the final lists.  The batches are gathered from e.q, the IUPAC canonical
// copy with that flag, and their marks from e.fx with B200SA_APPROX_FIXED.  Phases: per round best_compact, the
// search's, best_update; per emitted group best_compact, the search's, best_scatter; strand_merge with both
// strands.
template <class EndF>
static int approx_best(b200sa_ctx *c, const uint8_t *d_text, uint32_t n, const uint32_t *d_sa,
                       const uint32_t *d_starts, uint32_t ndocs, EndF end, const ApproxFlags &f,
                       const ApproxEntries &e, uint32_t nq, uint64_t q_bytes, ApproxFinal fin, uint64_t *total) {
    typedef unsigned long long u64;
    const uint32_t ne = e.ne, k = f.k, s = f.s;
    TRY(ensure(c, c->k32b, (size_t)ne * 8 + nq));        // cnt, map (u32) per entry, best (u8) per query
    TRY(ensure(c, c->rank, ((size_t)ne + 1) * 16));      // the batch's q_off, the search's offsets
    const size_t eb = (size_t)q_bytes * (f.both ? 2 : 1);          // the bytes of the entries
    TRY(ensure(c, c->qbuf, eb * (e.fx ? 2 : 1)));                  // a gathered batch, then its marks
    uint8_t *bmk = ptr<uint8_t>(c->qbuf) + eb;
    uint32_t *cnt = ptr<uint32_t>(c->k32b), *map = cnt + ne;
    uint8_t *best = reinterpret_cast<uint8_t *>(map + ne);
    uint64_t *coff = ptr<uint64_t>(c->rank), *soff = coff + ne + 1;
    uint32_t *words = ptr<uint32_t>(c->small);
    CU_TRY(c, cudaMemsetAsync(cnt, 0, (size_t)ne * 4, c->stream));
    CU_TRY(c, cudaMemsetAsync(best, BEST_NONE, nq, c->stream));
    CU_TRY(c, cudaMemsetAsync(words + AW_BATCH, 0, (AW_BEST_TOTAL + 2 - AW_BATCH) * 4, c->stream));
    uint64_t *ko = nullptr, rtotal = 0;
    uint32_t *vo = nullptr, nb = 0, rounds = 0;
    int pbits = 0;
    const uint8_t *bq, *bfx;
    const uint64_t *boff;
    auto batch = [&](uint32_t t, bool group) {
        if (f.both)
            return best_batch(c, e.q, e.off, e.fx, ne, StrandPick{e.off, best, ne, t, s, k, group}, map, coff, bmk,
                              &nb, &bq, &boff, &bfx);
        return best_batch(c, e.q, e.off, e.fx, ne, BestPick{e.off, best, ne, t, s, k, group}, map, coff, bmk, &nb,
                          &bq, &boff, &bfx);
    };
    for (uint32_t t = 0; t <= k; t++) {
        TRY(mark(c, "best_compact"));
        TRY(batch(t, false));
        if (nb == 0) break;
        rounds++;
        TRY(approx_search(c, d_text, n, d_sa, d_starts, ndocs, bq, boff, bfx, nb, t, f.edit, f.iupac, soff, 0, &rtotal,
                          end, &ko, &vo, &pbits));
        TRY(mark(c, "best_update"));
        if (f.both)
            LAUNCH(c, k_strand_update, cdiv(nb / 2, BLK), (const uint32_t *)map, (const u64 *)soff, nb, t, s, k, best,
                   cnt, words + AW_ENDED);
        else
            LAUNCH(c, k_best_update, cdiv(nb, BLK), (const uint32_t *)map, (const u64 *)soff, nb, t, s, k, best, cnt,
                   words + AW_ENDED);
    }
    c->stats.doubling_rounds = rounds;
    TRY((dev_scan<OpSum64>(c, InCount64{cnt, ne}, OutStoreExcl64{reinterpret_cast<u64 *>(e.out)}, (uint64_t)ne + 1,
                           reinterpret_cast<u64 *>(words + AW_BEST_TOTAL))));
    TRY(read_words(c, words + AW_ENDED, AW_BEST_TOTAL + 2 - AW_ENDED));
    const uint32_t ended = c->h_pin[0];
    *total = pin_u64(c, AW_BEST_TOTAL - AW_ENDED);
    const bool emitted = *total > 0 && *total <= fin.cap;
    if (f.stage && emitted) TRY(adocs_stage(c, *total, &fin.pos, &fin.mis));
    uint32_t *gpos = fin.pos, *gmis = fin.mis;           // where the groups scatter
    if (f.both && emitted) {
        TRY(ensure(c, c->sstage, (size_t)*total * 8));
        gpos = ptr<uint32_t>(c->sstage);
        gmis = gpos + *total;
    }
    if (emitted) {
        for (uint32_t t = 0; t <= k; t++) {
            if (!(ended >> t & 1u)) continue;
            TRY(mark(c, "best_compact"));
            TRY(batch(t, true));
            TRY(approx_search(c, d_text, n, d_sa, d_starts, ndocs, bq, boff, bfx, nb, t, f.edit, f.iupac, soff, ~0ull,
                              &rtotal, end, &ko, &vo, &pbits));
            TRY(mark(c, "best_scatter"));
            LAUNCH(c, k_best_scatter, cdiv(rtotal, BLK), (const u64 *)ko, (const uint32_t *)vo, rtotal, pbits,
                   (const u64 *)soff, (const uint32_t *)map, (const u64 *)e.out, gpos, gmis);
        }
    }
    if (f.both) TRY(strand_merge(c, StrandStaged{gpos}, gmis, *total, emitted, e.out, nq, fin.off, fin.pos, fin.mis));
    return B200SA_OK;
}

// nq >= 1 queries as f asks.  The checks; the IUPAC canonical copy, which every later kernel reads, and with
// B200SA_APPROX_FIXED the marks that follow the queries through every batch; with B200SA_APPROX_BOTH_STRANDS the
// doubled batch; then approx_plain or approx_best writes each query's final list.
// With B200SA_APPROX_DOCUMENTS that list is staged and adocs_reduce writes the caller's arrays; with
// B200SA_APPROX_LOCI loci_reduce cuts it to one hit per locus first; with B200SA_APPROX_ALIGN align_list writes
// them.  `doubling_rounds` is set only with B200SA_APPROX_BEST.
// Phases: approx_check; strand_queries with both strands; the middle's; loci_mark, loci_emit with
// B200SA_APPROX_LOCI; adocs_mark, adocs_emit with B200SA_APPROX_DOCUMENTS or align_count, align_scan, align_emit
// with B200SA_APPROX_ALIGN.
template <class EndF>
static int approx_run(b200sa_ctx *c, const uint8_t *d_text, uint32_t n, const uint32_t *d_sa,
                      const uint32_t *d_starts, uint32_t ndocs, const uint8_t *d_queries, const uint64_t *d_q_off,
                      uint32_t nq, const ApproxFlags &f, uint64_t *d_offsets, uint32_t *d_pos, uint32_t *d_mis,
                      uint64_t cap, uint64_t *total, EndF end) {
    if (f.best) c->stats.doubling_rounds = 0;
    uint64_t q_bytes;
    TRY(approx_prep(c, n, d_starts, ndocs, d_queries, d_q_off, nq, f.k, &q_bytes));
    if (f.both) TRY(strand_check(c, q_bytes, nq, f.k));
    uint32_t mmax = 0;
    if (f.align) TRY(align_check(c, d_q_off, nq, f.edit, &mmax));
    const uint8_t *d_fixed = nullptr;
    if (f.iupac) TRY(iupac_canon(c, d_queries, q_bytes, f.fixed, &d_queries, &d_fixed));
    if (n == 0) return approx_nothing(c, d_offsets, nq);
    ApproxFinal fin{d_offsets, d_pos, d_mis, f.stage ? ~0ull : cap};
    if (f.stage) TRY(adocs_offsets(c, nq, &fin.off));
    ApproxEntries e{d_queries, d_q_off, fin.off, nq, d_fixed};
    if (f.both) {
        TRY(strand_queries(c, d_queries, d_q_off, nq, q_bytes, f.iupac, d_fixed, &e.q, &e.off, &e.out, &e.fx));
        e.ne = 2 * nq;
    }
    if (f.best)
        TRY(approx_best(c, d_text, n, d_sa, d_starts, ndocs, end, f, e, nq, q_bytes, fin, total));
    else
        TRY(approx_plain(c, d_text, n, d_sa, d_starts, ndocs, end, f, e, nq, fin, total));
    const uint64_t *hoff = fin.off;
    if (f.loci)
        TRY(loci_reduce(c, d_starts, ndocs, d_q_off, nq, fin.off, f.align, d_offsets, d_pos, d_mis, cap, total, &hoff));
    if (f.docs) TRY(adocs_reduce(c, d_starts, ndocs, nq, fin.off, d_offsets, d_pos, d_mis, cap, total));
    if (f.align)
        TRY(align_list(c, d_text, n, d_starts, ndocs, d_queries, d_q_off, d_fixed, nq, f.k, f.edit, f.iupac, mmax,
                       hoff, d_offsets, d_pos, d_mis, cap, total, f.bulges));
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

// The argument checks shared by both entry points, and k decoded into *f.  docs: the documents entry, the only one
// that takes B200SA_APPROX_DOCUMENTS, B200SA_APPROX_ALIGN, B200SA_APPROX_FIXED, B200SA_APPROX_BULGES (whose
// budget fields are known bits only beside it) and B200SA_APPROX_LOCI (bit 7, a threshold bit on the other entry).
static int approx_args(b200sa_ctx *c, uint64_t n, const void *text, const void *sa, const void *q_off, uint32_t nq,
                       uint32_t k, const void *offsets, const void *pos, uint64_t cap, const void *total, bool docs,
                       ApproxFlags *f) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!total || !offsets || (nq > 0 && !q_off) || (cap > 0 && !pos) || (n > 0 && (!text || !sa))) return null_ptr(c);
    const bool best = (k & B200SA_APPROX_BEST) != 0, bulges = (k & B200SA_APPROX_BULGES) != 0;
    const bool loci = docs && (k & B200SA_APPROX_LOCI) != 0;
    const uint32_t tk = docs ? k & ~B200SA_APPROX_LOCI : k;  // k without bit 7 where it is the flag
    const uint32_t accepted = 0xFFFFu | B200SA_APPROX_EDIT | B200SA_APPROX_IUPAC | B200SA_APPROX_BOTH_STRANDS |
                              (best ? B200SA_APPROX_BEST : 0u) |
                              (docs ? B200SA_APPROX_DOCUMENTS | B200SA_APPROX_ALIGN | B200SA_APPROX_FIXED : 0u) |
                              (docs && bulges ? B200SA_APPROX_BULGES | B200SA_APPROX_DNA_BULGES(3) |
                                                    B200SA_APPROX_RNA_BULGES(3)
                                              : 0u);
    // with B200SA_APPROX_BEST the threshold and the slack are a byte each, and either above the limit is a bad k
    if ((k & ~accepted) || (best && ((tk & 0xFFu) > B200SA_APPROX_MAX_K || ((k >> 8) & 0xFFu) > B200SA_APPROX_MAX_K))) {
        const std::string m =
            std::string("approx positions: ") + (best ? "with B200SA_APPROX_BEST, " : "") +
            "k must be a threshold up to B200SA_APPROX_MAX_K" +
            (best ? " | B200SA_APPROX_SLACK(s) with s up to B200SA_APPROX_MAX_K" : "") +
            ", optionally | B200SA_APPROX_EDIT, | B200SA_APPROX_IUPAC" +
            (docs ? ", | B200SA_APPROX_BOTH_STRANDS, | B200SA_APPROX_FIXED with B200SA_APPROX_IUPAC, "
                    "| B200SA_APPROX_LOCI and | B200SA_APPROX_DOCUMENTS, or | B200SA_APPROX_ALIGN"
                  : " and | B200SA_APPROX_BOTH_STRANDS") +
            (!docs && bulges ? "; B200SA_APPROX_BULGES is taken by b200sa_docs_approx_positions_dev only" : "");
        return fail(c, B200SA_ERR_BAD_ARG, m.c_str());
    }
    if ((k & B200SA_APPROX_FIXED) && !(k & B200SA_APPROX_IUPAC))
        return fail(c, B200SA_ERR_BAD_ARG, "approx positions: B200SA_APPROX_FIXED requires B200SA_APPROX_IUPAC");
    if (bulges && !(k & B200SA_APPROX_EDIT))
        return fail(c, B200SA_ERR_BAD_ARG, "approx positions: B200SA_APPROX_BULGES requires B200SA_APPROX_EDIT");
    if (bulges && best)
        return fail(c, B200SA_ERR_BAD_ARG,
                    "approx positions: B200SA_APPROX_BULGES and B200SA_APPROX_BEST do not combine");
    if (!best && (tk & 0xFFFFu) > B200SA_APPROX_MAX_K)
        return fail(c, B200SA_ERR_BAD_ARG, "approx positions: k above B200SA_APPROX_MAX_K");
    const Bulges bg{bulges, tk & 0xFFFFu, (k >> 17) & 3u, (k >> 22) & 3u};
    if (bulges && bg.t + bg.d + bg.r > B200SA_APPROX_MAX_K)
        return fail(c, B200SA_ERR_BAD_ARG, "approx positions: with B200SA_APPROX_BULGES, the threshold plus the DNA "
                                           "and RNA bulges above B200SA_APPROX_MAX_K");
    if (n > B200SA_MAX_N) return too_long(c);
    const bool listing = (k & B200SA_APPROX_DOCUMENTS) != 0, align = (k & B200SA_APPROX_ALIGN) != 0;
    *f = ApproxFlags{best ? tk & 0xFFu : bulges ? bg.t + bg.d + bg.r : tk & 0xFFFFu, best ? (k >> 8) & 0xFFu : 0u,
                     (k & B200SA_APPROX_EDIT) != 0, best, (k & B200SA_APPROX_IUPAC) != 0,
                     (k & B200SA_APPROX_FIXED) != 0, (k & B200SA_APPROX_BOTH_STRANDS) != 0, listing, align, loci,
                     listing || align || loci, bg};
    return B200SA_OK;
}

int b200sa_approx_positions_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_sa,
                                const uint8_t *d_queries, const uint64_t *d_q_off, uint32_t nq, uint32_t k,
                                uint64_t *d_offsets, uint32_t *d_pos, uint32_t *d_mismatches, uint64_t cap,
                                uint64_t *total, void *stream) {
    ApproxFlags f;
    TRY(approx_args(c, n, d_text, d_sa, d_q_off, nq, k, d_offsets, d_pos, cap, total, false, &f));
    TRY(enter(c, stream));
    *total = 0;
    if (nq == 0) return leave(c, empty_batch(c, d_offsets));
    return leave(c, approx_run(c, d_text, (uint32_t)n, d_sa, nullptr, 0, d_queries, d_q_off, nq, f, d_offsets, d_pos,
                               d_mismatches, cap, total, TextEnd{(uint32_t)n}));
}

int b200sa_docs_approx_positions_dev(b200sa_ctx *c, const uint8_t *d_text, uint64_t n, const uint32_t *d_gsa,
                                     const uint32_t *d_doc_starts, uint32_t ndocs, const uint8_t *d_queries,
                                     const uint64_t *d_q_off, uint32_t nq, uint32_t k, uint64_t *d_offsets,
                                     uint32_t *d_pos, uint32_t *d_mismatches, uint64_t cap, uint64_t *total,
                                     void *stream) {
    ApproxFlags f;
    TRY(approx_args(c, n, d_text, d_gsa, d_q_off, nq, k, d_offsets, d_pos, cap, total, true, &f));
    if (f.align && f.docs)
        return fail(c, B200SA_ERR_BAD_ARG,
                    "approx positions: B200SA_APPROX_ALIGN and B200SA_APPROX_DOCUMENTS do not combine");
    if (f.loci && f.docs)
        return fail(c, B200SA_ERR_BAD_ARG,
                    "approx positions: B200SA_APPROX_LOCI and B200SA_APPROX_DOCUMENTS do not combine (the document "
                    "listing already keeps one entry per document)");
    if (f.align && cap > 0 && !d_mismatches)
        return fail(c, B200SA_ERR_BAD_ARG,
                    "approx positions: with B200SA_APPROX_ALIGN, d_mismatches is required when cap > 0");
    if ((n > 0 || ndocs > 0) && !d_doc_starts) return null_ptr(c);
    if (ndocs == 0 && n > 0) return no_docs(c);
    TRY(enter(c, stream));
    *total = 0;
    if (nq == 0) return leave(c, empty_batch(c, d_offsets));
    return leave(c, approx_run(c, d_text, (uint32_t)n, d_gsa, d_doc_starts, ndocs, d_queries, d_q_off, nq, f,
                               d_offsets, d_pos, d_mismatches, cap, total, DocsEnd{d_doc_starts, ndocs, (uint32_t)n}));
}

// ------------------------------------------------------------ multi-GPU: communicator + sharded LMS sort
#define NCCL_TRY(ctx, expr)                                                                  \
    do {                                                                                     \
        ncclResult_t r__ = (expr);                                                           \
        if (r__ != ncclSuccess) {                                                            \
            char buf__[400];                                                                 \
            snprintf(buf__, sizeof buf__, "%s:%d: %s -> %s", __FILE__, __LINE__, #expr,      \
                     nccl_api().GetErrorString ? nccl_api().GetErrorString(r__) : "nccl error"); \
            (ctx)->last_error = buf__;                                                       \
            return B200SA_ERR_COMM;                                                          \
        }                                                                                    \
    } while (0)

int b200sa_comm_unique_id(uint8_t *id_out) {
    if (!id_out) return B200SA_ERR_BAD_ARG;
    NcclApi &N = nccl_api();
    if (!N.ok) return B200SA_ERR_COMM;
    ncclUniqueId id;
    if (N.GetUniqueId(&id) != ncclSuccess) return B200SA_ERR_COMM;
    memcpy(id_out, id.internal, NCCL_UNIQUE_ID_BYTES);
    return B200SA_OK;
}

int b200sa_comm_init(b200sa_ctx *c, int nranks, int rank, const uint8_t *id128) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!id128) return null_ptr(c);
    if (nranks < 1 || nranks > 16 || rank < 0 || rank >= nranks)
        return fail(c, B200SA_ERR_BAD_ARG, "comm init: nranks must be in [1, 16] and rank in [0, nranks)");
    NcclApi &N = nccl_api();
    if (!N.ok) return fail(c, B200SA_ERR_COMM, N.err);
    CU_TRY(c, cudaSetDevice(c->device));
    if (c->comm && c->comm_owned) N.CommDestroy(c->comm);
    c->comm = nullptr;
    ncclUniqueId id;
    memcpy(id.internal, id128, NCCL_UNIQUE_ID_BYTES);
    NCCL_TRY(c, N.CommInitRank(&c->comm, nranks, id, rank));
    c->comm_owned = true; c->nranks = nranks; c->comm_rank = rank;
    return B200SA_OK;
}

int b200sa_comm_attach(b200sa_ctx *c, void *nccl_comm) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!nccl_comm) return null_ptr(c);
    NcclApi &N = nccl_api();
    if (!N.ok) return fail(c, B200SA_ERR_COMM, N.err);
    if (c->comm && c->comm_owned) N.CommDestroy(c->comm);
    c->comm = (ncclComm_t)nccl_comm;
    c->comm_owned = false;
    NCCL_TRY(c, N.CommCount(c->comm, &c->nranks));
    NCCL_TRY(c, N.CommUserRank(c->comm, &c->comm_rank));
    if (c->nranks > 16) return fail(c, B200SA_ERR_BAD_ARG, "comm attach: more than 16 ranks");
    return B200SA_OK;
}

int b200sa_comm_destroy(b200sa_ctx *c) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (c->comm && c->comm_owned && nccl_api().ok) nccl_api().CommDestroy(c->comm);
    c->comm = nullptr; c->comm_owned = false; c->nranks = 1; c->comm_rank = 0;
    return B200SA_OK;
}

// Collective over the context's communicator (a context without one is a world of 1).
static int shard_lms_sort_core(b200sa_ctx *c, const uint8_t *d_shard, uint64_t len, unsigned long long *d_sorted_gpos,
                               uint32_t *d_names, uint64_t cap, b200sa_shard_stats *out) {
    NcclApi &N = nccl_api();
    const int W = c->comm ? c->nranks : 1, R = c->comm ? c->comm_rank : 0;
    memset(out, 0, sizeof *out);
    constexpr int HEAD = 64;                                   // bytes of every shard's head that travel (halo source)
    // ---- small exchange area: per rank {len, first byte, last byte, state, m, distinct} + head bytes
    const size_t REC = 8;                                      // u64 words per rank record
    TRY(ensure(c, c->sh_small, (size_t)W * (REC * 8 + HEAD) * 2 + (size_t)W * W * 8 + 8192));
    unsigned long long *rec_all = ptr<unsigned long long>(c->sh_small);            // [W][REC]
    unsigned long long *rec_mine = rec_all + (size_t)W * REC;                      // [REC]
    uint8_t *heads_all = reinterpret_cast<uint8_t *>(rec_mine + REC);              // [W][HEAD]
    unsigned long long *cntmat = reinterpret_cast<unsigned long long *>(heads_all + (((size_t)W * HEAD + 63) & ~(size_t)63));   // [W][W] send counts
    unsigned long long *cnt_mine = cntmat + (size_t)W * W;                         // [W]
    unsigned long long *h64 = cnt_mine + W;                                        // [768]
    TRY(mark(c, "shard_edges"));
    // record: len, first, last  (+ head bytes)
    {
        unsigned long long h_rec[REC] = {len, 0, 0, 0, 0, 0, 0, cap};        // [7]: output capacity, so that every rank can
                                                                            // see every rank's fit and all fail together
        CU_TRY(c, cudaMemcpyAsync(rec_mine, h_rec, sizeof h_rec, cudaMemcpyHostToDevice, c->stream));
        CU_TRY(c, cudaMemsetAsync(heads_all + (size_t)R * HEAD, 0, HEAD, c->stream));
        CU_TRY(c, cudaMemcpyAsync(heads_all + (size_t)R * HEAD, d_shard, len < HEAD ? len : HEAD, cudaMemcpyDeviceToDevice, c->stream));
        CU_TRY(c, cudaMemcpyAsync(reinterpret_cast<uint8_t *>(rec_mine + 1), d_shard, 1, cudaMemcpyDeviceToDevice, c->stream));
        CU_TRY(c, cudaMemcpyAsync(reinterpret_cast<uint8_t *>(rec_mine + 2), d_shard + len - 1, 1, cudaMemcpyDeviceToDevice, c->stream));
    }
    std::vector<unsigned long long> hrec((size_t)W * REC);
    std::vector<uint8_t> hheads((size_t)W * HEAD);
    auto gather_records = [&]() -> int {
        if (W > 1) {
            NCCL_TRY(c, N.AllGather(rec_mine, rec_all, REC, ncclUint64, c->comm, c->stream));
        } else {
            CU_TRY(c, cudaMemcpyAsync(rec_all, rec_mine, REC * 8, cudaMemcpyDeviceToDevice, c->stream));
        }
        CU_TRY(c, cudaMemcpyAsync(hrec.data(), rec_all, (size_t)W * REC * 8, cudaMemcpyDeviceToHost, c->stream));
        return B200SA_OK;
    };
    TRY(gather_records());
    if (W > 1) NCCL_TRY(c, N.AllGather(heads_all + (size_t)R * HEAD, heads_all, HEAD, ncclUint8, c->comm, c->stream));
    CU_TRY(c, cudaMemcpyAsync(hheads.data(), heads_all, (size_t)W * HEAD, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    uint64_t lo = 0, n_total = 0;
    for (int r = 0; r < W; r++) { if (r < R) lo += hrec[r * REC]; n_total += hrec[r * REC]; }
    int next_char = -1, prev_char = -1;
    if (R + 1 < W) next_char = (int)(hrec[(R + 1) * REC + 1] & 0xff);
    if (R > 0) prev_char = (int)(hrec[(R - 1) * REC + 2] & 0xff);
    // halo: the bytes that follow this shard, taken from the heads of the following shards
    std::vector<uint8_t> halo;                     // up to HEAD bytes (or everything up to the end of the text)
    for (int r = R + 1; r < W && halo.size() < (size_t)HEAD; r++) {
        uint64_t take = hrec[r * REC] < (uint64_t)HEAD ? hrec[r * REC] : (uint64_t)HEAD;
        halo.insert(halo.end(), hheads.begin() + (size_t)r * HEAD, hheads.begin() + (size_t)r * HEAD + take);
    }
    if (halo.size() > (size_t)HEAD) halo.resize(HEAD);
    // ---- shard state -> tail carries
    TRY(mark(c, "shard_classify"));
    int state = ST_L;
    if (next_char >= 0) {
        uint64_t nw = (len + 31) / 32;
        uint32_t nbc = cdiv(nw, CLS_WORDS);
        TRY(ensure(c, c->blkstate, nbc));
        TRY(ensure(c, c->carry, nbc));
        ShardEdge e0{next_char, -1, ST_P};
        LAUNCH(c, k_cls_block_state, nbc, d_shard, len, ptr<uint8_t>(c->blkstate), e0);
        LAUNCH(c, k_cls_carry, 1, ptr<uint8_t>(c->blkstate), nbc, ptr<uint8_t>(c->carry), (uint32_t)ST_P);
        uint8_t h2[2];
        CU_TRY(c, cudaMemcpyAsync(&h2[0], c->blkstate.p, 1, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaMemcpyAsync(&h2[1], c->carry.p, 1, cudaMemcpyDeviceToHost, c->stream));
        CU_TRY(c, cudaStreamSynchronize(c->stream));
        state = (h2[0] != ST_P) ? h2[0] : h2[1];
    }
    {
        unsigned long long st = (unsigned long long)state;
        CU_TRY(c, cudaMemcpyAsync(rec_mine + 3, &st, 8, cudaMemcpyHostToDevice, c->stream));
        TRY(gather_records());
        CU_TRY(c, cudaStreamSynchronize(c->stream));
    }
    uint32_t tail = ST_L;
    for (int r = R + 1; r < W; r++) if (hrec[r * REC + 3] != ST_P) { tail = (uint32_t)hrec[r * REC + 3]; break; }
    // ---- classification of the shard (fused kernel with halo chars), LMS positions descending
    uint32_t m = 0;
    TRY(classify_fused_dev(c, d_shard, len, &m, ShardEdge{next_char, prev_char, next_char >= 0 ? tail : ST_L}, false));
    // ---- global alphabet: all-reduce of the (byte, type) histogram
    TRY(mark(c, "shard_keys"));
    uint32_t *tab = ptr<uint32_t>(c->tables);
    LAUNCH(c, k_hist_to_u64, 3u, tab + T_HIST, h64, 768u);
    if (W > 1) NCCL_TRY(c, N.AllReduce(h64, h64, 768, ncclUint64, ncclSum, c->comm, c->stream));
    uint32_t *sm = ptr<uint32_t>(c->small);
    LAUNCH(c, k_alpha_from_hist64, 1u, h64, tab + T_CODE, sm + 3);
    TRY(read_words(c, sm + 3, 1));
    const uint32_t sigma = c->h_pin[0] < 2 ? 2u : c->h_pin[0];
    uint32_t kc = 0;
    {
        unsigned __int128 r = 1;
        while (kc < 32 && r * sigma <= ((unsigned __int128)1 << 64)) { r *= sigma; kc++; }
    }
    // ---- window keys of the local LMS suffixes (descending position order)
    TRY(ensure(c, c->sh_a, (size_t)(m + 1) * 8));                 // keys
    TRY(ensure(c, c->sh_b, (size_t)(m + 1) * 4));                 // local positions
    TRY(ensure(c, c->sh_c, (size_t)(m + 1) * 8));                 // keys partitioned by destination
    TRY(ensure(c, c->sh_d, (size_t)(m + 1) * 4));                 // positions partitioned
    TRY(ensure(c, c->flag, (size_t)m + 64 + HEAD));               // destinations (+ halo bytes at the end)
    uint8_t *d_halo = ptr<uint8_t>(c->flag) + (((size_t)m + 15) & ~(size_t)15);
    if (!halo.empty()) CU_TRY(c, cudaMemcpyAsync(d_halo, halo.data(), halo.size(), cudaMemcpyHostToDevice, c->stream));
    ShardWin SW{d_shard, d_halo, tab + T_CODE, len, (uint64_t)halo.size(), sigma, kc};
    uint64_t *K0 = ptr<uint64_t>(c->sh_a), *K1 = ptr<uint64_t>(c->sh_c);
    uint32_t *V0 = ptr<uint32_t>(c->sh_b), *V1 = ptr<uint32_t>(c->sh_d);
    if (m) LAUNCH(c, k_shard_keys, cdiv(m, BLK), SW, ptr<uint32_t>(c->lmsdesc), m, K0, V0);
    // ---- splitters from an all-gathered sample
    TRY(mark(c, "shard_partition"));
    const uint32_t PER = 1024;
    TRY(ensure(c, c->sh_e, (size_t)W * PER * 8 * 2 + (size_t)W * PER * 4 * 2 + 256));
    uint64_t *samp = ptr<uint64_t>(c->sh_e), *samp2 = samp + (size_t)W * PER;
    uint32_t *sv0 = reinterpret_cast<uint32_t *>(samp2 + (size_t)W * PER), *sv1 = sv0 + (size_t)W * PER;
    uint64_t *split = reinterpret_cast<uint64_t *>(sv1 + (size_t)W * PER);
    LAUNCH(c, k_shard_sample, cdiv(PER, BLK), K0, m, PER, samp + (size_t)R * PER);
    if (W > 1) NCCL_TRY(c, N.AllGather(samp + (size_t)R * PER, samp, PER, ncclUint64, c->comm, c->stream));
    {
        uint64_t *ks; uint32_t *vs;
        LAUNCH(c, k_iota, cdiv(W * PER, BLK), sv0, (uint32_t)(W * PER));
        TRY(sort_pairs<uint64_t>(c, samp, sv0, samp2, sv1, (uint64_t)W * PER, 64, &ks, &vs));
        LAUNCH(c, k_shard_splitters, 1u, ks, (uint32_t)(W * PER), (uint32_t)W, split);
    }
    CU_TRY(c, cudaMemsetAsync(cnt_mine, 0, (size_t)W * 8, c->stream));
    uint8_t *dest = ptr<uint8_t>(c->flag);
    if (m) {
        LAUNCH(c, k_shard_dest, cdiv(m, BLK), K0, m, split, (uint32_t)W, dest, cnt_mine);
        TRY(radix_pass(c, DigU8{dest}, MoveKV64{K0, V0, K1, V1}, m));        // stable: descending position inside a destination
    }
    if (W > 1) NCCL_TRY(c, N.AllGather(cnt_mine, cntmat, W, ncclUint64, c->comm, c->stream));
    else CU_TRY(c, cudaMemcpyAsync(cntmat, cnt_mine, 8, cudaMemcpyDeviceToDevice, c->stream));
    std::vector<unsigned long long> hcnt((size_t)W * W);
    CU_TRY(c, cudaMemcpyAsync(hcnt.data(), cntmat, (size_t)W * W * 8, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    // ---- all-to-all: chunks are received in DESCENDING source rank (larger text positions first)
    TRY(mark(c, "shard_exchange"));
    uint64_t recv_total = 0, m_total = 0;
    std::vector<uint64_t> roff(W + 1, 0), soff(W + 1, 0);
    for (int k = 0; k < W; k++) { int src = W - 1 - k; roff[k + 1] = roff[k] + hcnt[(size_t)src * W + R]; }
    for (int d = 0; d < W; d++) soff[d + 1] = soff[d] + hcnt[(size_t)R * W + d];
    recv_total = roff[W];
    for (int r = 0; r < W; r++) for (int d = 0; d < W; d++) m_total += hcnt[(size_t)r * W + d];
    for (int r = 0; r < W; r++) {                  // the same verdict on every rank: nobody enters the exchange alone
        uint64_t slice = 0;
        for (int q = 0; q < W; q++) slice += hcnt[(size_t)q * W + r];
        if (slice > 0xfffffff0ull) return fail(c, B200SA_ERR_TOO_LARGE, "more than 2^32 LMS suffixes on one rank");
        if (slice > hrec[r * REC + 7]) {
            char b[160]; snprintf(b, sizeof b, "output capacity of rank %d too small for its slice (%llu entries)", r, (unsigned long long)slice);
            c->last_error = b; return B200SA_ERR_BAD_ARG;
        }
    }
    TRY(ensure(c, c->sh_a, (size_t)(recv_total + 1) * 8));         // received keys (K0 is free after the partition)
    TRY(ensure(c, c->sh_b, (size_t)(recv_total + 1) * 4));         // received local positions
    K0 = ptr<uint64_t>(c->sh_a); V0 = ptr<uint32_t>(c->sh_b);
    if (W > 1) {
        NCCL_TRY(c, N.GroupStart());
        for (int k = 0; k < W; k++) {
            int src = W - 1 - k;
            uint64_t cnt = roff[k + 1] - roff[k];
            if (cnt) {
                NCCL_TRY(c, N.Recv(K0 + roff[k], cnt, ncclUint64, src, c->comm, c->stream));
                NCCL_TRY(c, N.Recv(V0 + roff[k], cnt, ncclUint32, src, c->comm, c->stream));
            }
        }
        for (int d = 0; d < W; d++) {
            uint64_t cnt = soff[d + 1] - soff[d];
            if (cnt) {
                NCCL_TRY(c, N.Send(K1 + soff[d], cnt, ncclUint64, d, c->comm, c->stream));
                NCCL_TRY(c, N.Send(V1 + soff[d], cnt, ncclUint32, d, c->comm, c->stream));
                if (d != R) { out->bytes_sent += (double)cnt * 12.0; }
            }
        }
        NCCL_TRY(c, N.GroupEnd());
    } else if (recv_total) {
        CU_TRY(c, cudaMemcpyAsync(K0, K1, recv_total * 8, cudaMemcpyDeviceToDevice, c->stream));
        CU_TRY(c, cudaMemcpyAsync(V0, V1, recv_total * 4, cudaMemcpyDeviceToDevice, c->stream));
    }
    // ---- local sort of the received slice, global positions, groups, names
    TRY(mark(c, "shard_sort"));
    uint32_t cnt32 = (uint32_t)recv_total;
    TRY(ensure(c, c->sh_c, (size_t)(recv_total + 1) * 8));
    TRY(ensure(c, c->sh_d, (size_t)(recv_total + 1) * 4));
    TRY(ensure(c, c->sh_f, (size_t)(recv_total + 1) * 4));
    uint32_t *I0 = ptr<uint32_t>(c->sh_d), *I1 = ptr<uint32_t>(c->sh_f);
    uint64_t *Ks = K0; uint32_t *Is = I0;
    unsigned long long *chunk_off = cnt_mine;                      // reuse: [W+1] offsets, then [W] lo
    std::vector<unsigned long long> hco((size_t)2 * W + 1);
    for (int k = 0; k <= W; k++) hco[k] = roff[k];
    for (int k = 0; k < W; k++) { int src = W - 1 - k; uint64_t l2 = 0; for (int r = 0; r < src; r++) l2 += hrec[r * REC]; hco[W + 1 + k] = l2; }
    TRY(ensure(c, c->sh_e, (size_t)(2 * W + 1) * 8 + 64));
    chunk_off = ptr<unsigned long long>(c->sh_e);
    CU_TRY(c, cudaMemcpyAsync(chunk_off, hco.data(), hco.size() * 8, cudaMemcpyHostToDevice, c->stream));
    unsigned long long *d_ties = h64;                              // reuse (the histogram is consumed)
    CU_TRY(c, cudaMemsetAsync(d_ties, 0, 16, c->stream));
    if (cnt32) {
        LAUNCH(c, k_iota, cdiv(cnt32, BLK), I0, cnt32);
        int kbits = 64;
        TRY(sort_pairs<uint64_t>(c, K0, I0, ptr<uint64_t>(c->sh_c), I1, cnt32, kbits, &Ks, &Is));
        LAUNCH(c, k_shard_gpos, cdiv(cnt32, BLK), Is, V0, cnt32, chunk_off, chunk_off + W + 1, (uint32_t)W, d_sorted_gpos);
        InShardHead in{Ks, d_sorted_gpos, cnt32, n_total, kc};
        TRY((dev_scan<OpSum>(c, in, OutShardName{in, 0u, d_names, d_ties}, cnt32, sm + 16)));
    } else {
        CU_TRY(c, cudaMemsetAsync(sm + 16, 0, 4, c->stream));
    }
    // ---- name offsets: exclusive prefix of the distinct counts over ranks; ties summed
    TRY(mark(c, "shard_names"));
    CU_TRY(c, cudaMemcpyAsync(reinterpret_cast<uint32_t *>(rec_mine + 5), sm + 16, 4, cudaMemcpyDeviceToDevice, c->stream));
    CU_TRY(c, cudaMemcpyAsync(rec_mine + 6, d_ties, 8, cudaMemcpyDeviceToDevice, c->stream));
    {
        unsigned long long mm = m;
        CU_TRY(c, cudaMemcpyAsync(rec_mine + 4, &mm, 8, cudaMemcpyHostToDevice, c->stream));
    }
    TRY(gather_records());
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    uint64_t name_off = 0, ties = 0;
    for (int r = 0; r < W; r++) { if (r < R) name_off += (uint32_t)hrec[r * REC + 5]; ties += hrec[r * REC + 6]; }
    if (cnt32 && name_off) LAUNCH(c, k_add_u32, cdiv(cnt32, BLK), d_names, cnt32, (uint32_t)name_off);
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    out->n_total = n_total; out->m_total = m_total; out->m_local = m; out->recv_count = recv_total;
    out->distinct_local = (uint32_t)hrec[R * REC + 5]; out->name_offset = name_off; out->ties_total = ties;
    out->kc = kc; out->lo = lo; out->nranks = (uint32_t)W; out->rank = (uint32_t)R;
    out->bytes_recv = 0;
    for (int k = 0; k < W; k++) { int src = W - 1 - k; if (src != R) out->bytes_recv += (double)(roff[k + 1] - roff[k]) * 12.0; }
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

// A collective call needs NCCL when the context's communicator has more than one rank.
static int comm_ready(b200sa_ctx *c) {
    if (c->comm && c->nranks > 1 && !nccl_api().ok) return fail(c, B200SA_ERR_COMM, nccl_api().err);
    return B200SA_OK;
}

int b200sa_shard_lms_sort(b200sa_ctx *c, const uint8_t *d_shard, uint64_t len, unsigned long long *d_sorted_gpos,
                          uint32_t *d_names, uint64_t cap, b200sa_shard_stats *out, void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!out) return null_ptr(c);
    TRY(shard_args(c, d_shard, len, -1));
    TRY(comm_ready(c));
    TRY(enter(c, stream));
    return leave(c, shard_lms_sort_core(c, d_shard, len, d_sorted_gpos, d_names, cap, out));
}

// Sharded LCP (SURVEY 8e row 5): text and SA are replicated (broadcast from rank 0 unless the caller
// says they already are), every rank computes Phi and PLCP for ITS text range only, the PLCP ranges
// are all-gathered, every rank turns its rank range into LCP values and the slices are all-gathered.
// Same values as lcp_lens_quadratic (src/table.rs:348-361).
static int lcp_sharded_core(b200sa_ctx *c, uint8_t *d_text, uint64_t n, uint32_t *d_sa, uint32_t *d_lcp,
                            int replicated) {
    NcclApi &N = nccl_api();
    const int W = c->comm ? c->nranks : 1, R = c->comm ? c->comm_rank : 0;
    if (n == 0) return B200SA_OK;
    if (((uintptr_t)d_text & 15) != 0) return fail(c, B200SA_ERR_BAD_ARG, "text pointer must be 16-byte aligned");
    const uint32_t n32 = (uint32_t)n;
    TRY(mark(c, "lcps_bcast"));
    if (W > 1 && !replicated) {
        NCCL_TRY(c, N.Broadcast(d_text, d_text, n, ncclUint8, 0, c->comm, c->stream));
        NCCL_TRY(c, N.Broadcast(d_sa, d_sa, n, ncclUint32, 0, c->comm, c->stream));
    }
    // ---- every rank: validate the table, pack the text (same steps as the stand-alone b200sa_lcp_dev)
    TRY(mark(c, "lcps_pack"));
    const uint64_t per = ((n + W - 1) / W + 1023) / 1024 * 1024;       // positions (and ranks) per GPU
    TRY(ensure(c, c->isa, (size_t)W * per * 4));
    TRY(ensure(c, c->small, 4096));
    TRY(ensure(c, c->tables, T_END * 4));
    uint32_t *tab = ptr<uint32_t>(c->tables), *sm = ptr<uint32_t>(c->small);
    {
        uint64_t nwv = (n + 31) / 32;
        uint32_t *seen = ptr<uint32_t>(c->isa), *bad = sm + 12;
        CU_TRY(c, cudaMemsetAsync(seen, 0, nwv * 4, c->stream));
        CU_TRY(c, cudaMemsetAsync(bad, 0, 4, c->stream));
        CU_TRY(c, cudaMemsetAsync(bad + 1, 0, 4, c->stream));
        LAUNCH(c, k_sa_validate, cdiv(cdiv(n, 4), BLK), d_sa, n32, seen, bad);
        LAUNCH(c, k_sa_validate_count, (uint32_t)c->sm_count * 4u, seen, n32, bad + 1);
        LAUNCH(c, k_sa_validate_verdict, 1u, bad + 1, n32, bad);
        CU_TRY(c, cudaMemsetAsync(tab + T_HIST, 0, 256 * 4, c->stream));
        uint32_t hb = cdiv(n, BLK * 64);
        if (hb > grid_cap(c)) hb = grid_cap(c);
        LAUNCH(c, k_byte_hist, hb, d_text, n, tab + T_HIST, (const uint32_t *)nullptr);
        LAUNCH(c, k_alpha_from_hist, 1, tab + T_HIST, tab + T_CODE, tab + T_ALPHA, sm + 3, (const uint32_t *)nullptr);
        TRY(read_words(c, sm, 16));
        if (c->h_pin[12] != 0)        // identical on every rank: all fail together
            return fail(c, B200SA_ERR_BAD_ARG, "table is not a permutation of 0..n-1 (index out of range or repeated)");
        TRY(pack_text(c, d_text, n, c->h_pin[3]));
    }
    // ---- Phi and PLCP of this rank's text range
    TRY(mark(c, "lcps_plcp"));
    const uint64_t lo = (uint64_t)R * per, hi = (lo + per < n) ? lo + per : (lo < n ? n : lo);
    uint32_t *phi = ptr<uint32_t>(c->isa);
    uint32_t nchunk = cdiv(n, LCP_CHUNK);
    TRY(ensure(c, c->plcp_samp, (size_t)nchunk * 4));
    uint32_t *samp = ptr<uint32_t>(c->plcp_samp);
    if (hi > lo) {
        LAUNCH(c, k_phi_range, cdiv(n, BLK), d_sa, n32, (uint32_t)lo, (uint32_t)hi, phi);
        uint64_t len = hi - lo;
        uint32_t chunks = cdiv(len, LCP_CHUNK);
        uint32_t pg = cdiv(chunks, BLK), sg = cdiv(cdiv(chunks, 32), BLK);
        uint64_t toff_s = lo / (32ull * LCP_CHUNK), toff_p = lo / LCP_CHUNK;
        if (c->bits == 2) LAUNCH(c, (k_plcp_samples<2>), sg, c->ptext, n32, phi, samp, toff_s, hi);
        else if (c->bits == 4) LAUNCH(c, (k_plcp_samples<4>), sg, c->ptext, n32, phi, samp, toff_s, hi);
        else LAUNCH(c, (k_plcp_samples<8>), sg, c->ptext, n32, phi, samp, toff_s, hi);
        if (c->bits == 2) LAUNCH(c, (k_plcp<2>), pg, c->ptext, n32, phi, samp, toff_p, hi);
        else if (c->bits == 4) LAUNCH(c, (k_plcp<4>), pg, c->ptext, n32, phi, samp, toff_p, hi);
        else LAUNCH(c, (k_plcp<8>), pg, c->ptext, n32, phi, samp, toff_p, hi);
    }
    TRY(mark(c, "lcps_allgather_plcp"));
    if (W > 1) NCCL_TRY(c, N.AllGather(phi + lo, phi, per, ncclUint32, c->comm, c->stream));
    // ---- LCP of this rank's RANK range, then the slices to everybody
    TRY(mark(c, "lcps_gather"));
    TRY(ensure(c, c->phik, (size_t)W * per * 4));
    uint32_t *slices = ptr<uint32_t>(c->phik);
    if (hi > lo) LAUNCH(c, k_lcp_gather_range, cdiv(hi - lo, BLK), d_sa, phi, (uint32_t)lo, (uint32_t)hi, slices + lo);
    TRY(mark(c, "lcps_allgather_lcp"));
    if (W > 1) NCCL_TRY(c, N.AllGather(slices + lo, slices, per, ncclUint32, c->comm, c->stream));
    CU_TRY(c, cudaMemcpyAsync(d_lcp, slices, n * 4, cudaMemcpyDeviceToDevice, c->stream));
    TRY(mark(c, "end"));
    CU_TRY(c, cudaGetLastError());
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    return B200SA_OK;
}

int b200sa_lcp_sharded(b200sa_ctx *c, uint8_t *d_text, uint64_t n, uint32_t *d_sa, uint32_t *d_lcp, int replicated,
                       void *stream) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!d_text || !d_sa || !d_lcp)) return null_ptr(c);
    if (n > B200SA_MAX_N) return too_long(c);
    TRY(comm_ready(c));
    TRY(enter(c, stream));
    return leave(c, lcp_sharded_core(c, d_text, n, d_sa, d_lcp, replicated));
}

// ------------------------------------------------------------ test hooks
// The classification of a host text by the fused byte classifier, copied back (LMS positions descending).
static int test_classify_core(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t *stype_words,
                              uint32_t *lms_words, uint32_t *hist768, uint32_t *lmspos_desc, uint64_t cap_lms,
                              uint64_t *m_out) {
    TRY(ensure(c, c->text, n));
    CU_TRY(c, cudaMemcpyAsync(c->text.p, text, n, cudaMemcpyHostToDevice, c->stream));
    uint32_t m = 0;
    TRY(classify_fused_dev(c, ptr<uint8_t>(c->text), n, &m));
    uint64_t nw = (n + 31) / 32;
    if (stype_words) CU_TRY(c, cudaMemcpyAsync(stype_words, c->stype.p, nw * 4, cudaMemcpyDeviceToHost, c->stream));
    if (lms_words) CU_TRY(c, cudaMemcpyAsync(lms_words, c->lmsb.p, nw * 4, cudaMemcpyDeviceToHost, c->stream));
    if (hist768) CU_TRY(c, cudaMemcpyAsync(hist768, ptr<uint32_t>(c->tables) + T_HIST, 768 * 4, cudaMemcpyDeviceToHost, c->stream));
    if (lmspos_desc && m > 0) {
        uint64_t k = m < cap_lms ? m : cap_lms;
        CU_TRY(c, cudaMemcpyAsync(lmspos_desc, c->lmsdesc.p, k * 4, cudaMemcpyDeviceToHost, c->stream));
    }
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    if (m_out) *m_out = m;
    return B200SA_OK;
}

int b200sa_test_classify_fused(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t *stype_words, uint32_t *lms_words,
                               uint32_t *hist768, uint32_t *lmspos_desc, uint64_t cap_lms, uint64_t *m_out) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!text) return null_ptr(c);
    if (n < 1 || n > B200SA_MAX_N) return fail(c, B200SA_ERR_BAD_ARG, "test classify: n must be in [1, 2^32-4096]");
    TRY(enter(c, nullptr));
    return leave(c, test_classify_core(c, text, n, stype_words, lms_words, hist768, lmspos_desc, cap_lms, m_out));
}

// The classification of a host text of at most 4 distinct bytes from its 2-bit packed words
// (k_classify_packed), copied back: the bitmaps, hist768, the LMS positions in descending order, their
// window keys and the digit counts of key bits 16-23 / 24-31 (dig512).  A text with a larger alphabet is an
// argument error.  Only the tests call it, through ctypes; it is not part of the C headers.
static int test_classify_packed_core(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t *stype_words,
                                     uint32_t *lms_words, uint32_t *hist768, uint32_t *lmsdesc, uint32_t *keys,
                                     uint32_t *dig512, uint64_t cap_lms, uint64_t *m_out) {
    TRY(ensure(c, c->text, n));
    CU_TRY(c, cudaMemcpyAsync(c->text.p, text, n, cudaMemcpyHostToDevice, c->stream));
    uint32_t m = 0;
    TRY(classify_fused_dev(c, ptr<uint8_t>(c->text), n, &m, ShardEdge{-1, -1, ST_L}, true, true));
    if (!c->lms_keys_ready)
        return fail(c, B200SA_ERR_BAD_ARG, "test classify packed: the text needs at most 4 distinct bytes");
    uint64_t nw = (n + 31) / 32, k = m < cap_lms ? m : cap_lms;
    if (stype_words) CU_TRY(c, cudaMemcpyAsync(stype_words, c->stype.p, nw * 4, cudaMemcpyDeviceToHost, c->stream));
    if (lms_words) CU_TRY(c, cudaMemcpyAsync(lms_words, c->lmsb.p, nw * 4, cudaMemcpyDeviceToHost, c->stream));
    if (hist768) CU_TRY(c, cudaMemcpyAsync(hist768, ptr<uint32_t>(c->tables) + T_HIST, 768 * 4, cudaMemcpyDeviceToHost, c->stream));
    if (lmsdesc && k) CU_TRY(c, cudaMemcpyAsync(lmsdesc, c->lmsdesc.p, k * 4, cudaMemcpyDeviceToHost, c->stream));
    if (keys && k) CU_TRY(c, cudaMemcpyAsync(keys, c->reduced.p, k * 4, cudaMemcpyDeviceToHost, c->stream));
    if (dig512) CU_TRY(c, cudaMemcpyAsync(dig512, c->os_hist.p, 512 * 4, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    if (m_out) *m_out = m;
    return B200SA_OK;
}

extern "C" int b200sa_test_classify_packed(b200sa_ctx *c, const uint8_t *text, uint64_t n, uint32_t *stype_words,
                                           uint32_t *lms_words, uint32_t *hist768, uint32_t *lmsdesc, uint32_t *keys,
                                           uint32_t *dig512, uint64_t cap_lms, uint64_t *m_out) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!text) return null_ptr(c);
    if (n < 2 || n > B200SA_MAX_N) return fail(c, B200SA_ERR_BAD_ARG, "test classify packed: n must be in [2, 2^32-4096]");
    TRY(enter(c, nullptr));
    return leave(c, test_classify_packed_core(c, text, n, stype_words, lms_words, hist768, lmsdesc, keys, dig512,
                                              cap_lms, m_out));
}

static int test_scan_core(b200sa_ctx *c, const uint32_t *in, uint64_t n, int op, uint32_t *out_excl, uint32_t *total) {
    TRY(ensure(c, c->v0, n * 4));
    TRY(ensure(c, c->v1, n * 4));
    TRY(ensure(c, c->small, 4096));
    CU_TRY(c, cudaMemcpyAsync(c->v0.p, in, n * 4, cudaMemcpyHostToDevice, c->stream));
    uint32_t *d_tot = ptr<uint32_t>(c->small);
    if (op == 0) TRY((dev_scan<OpSum>(c, InArray{ptr<uint32_t>(c->v0)}, OutStoreExcl{ptr<uint32_t>(c->v1)}, n, d_tot)));
    else TRY((dev_scan<OpMax>(c, InArray{ptr<uint32_t>(c->v0)}, OutStoreExcl{ptr<uint32_t>(c->v1)}, n, d_tot)));
    if (n) CU_TRY(c, cudaMemcpyAsync(out_excl, c->v1.p, n * 4, cudaMemcpyDeviceToHost, c->stream));
    TRY(read_words(c, d_tot, 1));
    if (total) *total = c->h_pin[0];
    return B200SA_OK;
}

int b200sa_test_scan(b200sa_ctx *c, const uint32_t *in, uint64_t n, int op, uint32_t *out_excl, uint32_t *total) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (n > 0 && (!in || !out_excl)) return null_ptr(c);
    TRY(enter(c, nullptr));
    return leave(c, test_scan_core(c, in, n, op, out_excl, total));
}

int b200sa_test_sort_pairs32(b200sa_ctx *c, uint32_t *keys, uint32_t *vals, uint64_t n, int bits) {
    return test_sort<uint32_t>(c, keys, vals, n, bits);
}
int b200sa_test_sort_pairs64(b200sa_ctx *c, uint64_t *keys, uint32_t *vals, uint64_t n, int bits) {
    return test_sort<uint64_t>(c, keys, vals, n, bits);
}

static int test_reduced_sa_core(b200sa_ctx *c, const uint32_t *R, uint64_t m, uint32_t names, uint32_t *sa_out,
                                uint32_t *rounds_out) {
    TRY(ensure(c, c->reduced, m * 4));
    CU_TRY(c, cudaMemcpyAsync(c->reduced.p, R, m * 4, cudaMemcpyHostToDevice, c->stream));
    uint32_t rounds = 0;
    TRY(reduced_sa(c, ptr<uint32_t>(c->reduced), (uint32_t)m, names, &rounds));
    CU_TRY(c, cudaMemcpyAsync(sa_out, c->sa_r.p, m * 4, cudaMemcpyDeviceToHost, c->stream));
    CU_TRY(c, cudaStreamSynchronize(c->stream));
    if (rounds_out) *rounds_out = rounds;
    return B200SA_OK;
}

int b200sa_test_reduced_sa(b200sa_ctx *c, const uint32_t *R, uint64_t m, uint32_t names, uint32_t *sa_out,
                           uint32_t *rounds_out) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!R || !sa_out) return null_ptr(c);
    if (m < 1 || m > 0x7FFFFFFFull) return fail(c, B200SA_ERR_BAD_ARG, "test reduced sa: m must be in [1, 2^31)");
    TRY(enter(c, nullptr));
    return leave(c, test_reduced_sa_core(c, R, m, names, sa_out, rounds_out));
}

int64_t b200sa_debug_fetch(b200sa_ctx *c, int which, void *out, uint64_t cap) {
    if (!c) return B200SA_ERR_BAD_ARG;
    if (!out) return null_ptr(c);
    if (cudaSetDevice(c->device) != cudaSuccess) return B200SA_ERR_CUDA;
    const void *src = nullptr;
    uint64_t count = 0;
    switch (which) {
        case 0: src = c->lmspos.p; count = c->last_m; break;
        case 1: src = c->sorted.p; count = c->last_m; break;
        case 2: src = c->reduced.p; count = c->last_m; break;
        case 3: src = c->sa_r.p; count = c->last_m; break;
        case 4: src = c->lmslist.p; count = c->last_m; break;
        case 5: src = c->small.p ? (const void *)(ptr<uint32_t>(c->small) + 32) : nullptr; count = 10; break;
        case 6: src = c->tables.p; count = T_HIST; break;
        case 7: src = c->steplog.p; count = c->steplog.p ? 16384 : 0; break;     // u64 records viewed as u32 pairs
        default: return fail(c, B200SA_ERR_BAD_ARG, "debug fetch: unknown buffer");
    }
    if (!src) return 0;
    uint64_t k = count < cap ? count : cap;
    if (k && cudaMemcpy(out, src, k * 4, cudaMemcpyDeviceToHost) != cudaSuccess) return B200SA_ERR_CUDA;
    return (int64_t)count;
}
