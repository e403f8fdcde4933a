/* xgm_host.cu — host side of libxgm.so: index builder (HBM block format), term dictionary, query
 * planner (the host half of the reference's LocalSubMatch/Weight::init_ work) and the C-ABI of
 * include/xgm.h.  There is no CPU matching path in this file: every search goes through the kernels
 * in xgm_kernels.cu, and the library refuses to create an index without a CUDA device. */
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cfloat>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <chrono>
#include <cstring>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/xgm.h"
#include "xgm_corpus.h"
#include "xgm_device.h"

/* ------------------------------------------------------------------ errors */

static thread_local char g_err[512] = "";
static const bool g_trace = getenv("XGM_TRACE") != nullptr && atoi(getenv("XGM_TRACE")) != 0;
static cudaEvent_t g_tr_base = nullptr; /* XGM_TRACE: common origin of every searcher's timeline */
static std::chrono::steady_clock::time_point g_tr_t0;

static xgm_status fail(xgm_status st, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return st;
}

#define CUDA_TRY(expr)                                                                         \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess)                                                                \
            return fail(XGM_E_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

/* for the other translation units of the library (xgm_glass.cu) */
xgm_status xgm_fail(xgm_status st, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return st;
}

extern "C" const char* xgm_last_error(void) { return g_err; }
extern "C" uint32_t xgm_abi_version(void) { return XGM_ABI_VERSION; }

/* ------------------------------------------------------------------ small helpers */

template <class F>
static void parallel_for(size_t n, int threads, F f) {
    if (threads <= 1 || n < 2) {
        for (size_t i = 0; i < n; ++i) f(i, 0);
        return;
    }
    if ((size_t)threads > n) threads = (int)n;
    std::atomic<size_t> next{0};
    std::vector<std::thread> th;
    for (int t = 0; t < threads; ++t)
        th.emplace_back([&, t]() {
            for (;;) {
                size_t i = next.fetch_add(1);
                if (i >= n) break;
                f(i, t);
            }
        });
    for (auto& x : th) x.join();
}

static int default_threads() {
    unsigned hc = std::thread::hardware_concurrency();
    if (hc == 0) hc = 4;
    if (hc > 64) hc = 64;
    return (int)hc;
}

static inline uint32_t bits_for(uint32_t v) { return v ? 32u - (uint32_t)__builtin_clz(v) : 0u; }

/* ------------------------------------------------------------------ owned CUDA resources */

/* A device (cudaMalloc) or pinned host (cudaMallocHost) array of T that frees itself.  The destructor and every
 * reallocation free on the current device: whoever frees one sets it first. */
template <class T, bool Pinned> class Buf {
  public:
    Buf() = default;
    Buf(const Buf&) = delete;
    Buf& operator=(const Buf&) = delete;
    ~Buf() { release(); }
    /* n elements; what was held before is freed first */
    cudaError_t alloc(size_t n) {
        release();
        void* p = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&p, n * sizeof(T)) : cudaMalloc(&p, n * sizeof(T));
        if (e == cudaSuccess) { p_ = static_cast<T*>(p); cap_ = n; }
        return e;
    }
    /* room for `need` elements, grown to max(2 need, floor); the stream's copies and kernels may still read the
     * old array, so it is waited for before the array is freed */
    cudaError_t grow(size_t need, size_t floor, cudaStream_t st) {
        if (need <= cap_) return cudaSuccess;
        const cudaError_t e = cudaStreamSynchronize(st);
        return e != cudaSuccess ? e : alloc(std::max(need * 2, floor));
    }
    T* get() const { return p_; }

  private:
    void release() {
        if (p_) { if (Pinned) cudaFreeHost(p_); else cudaFree(p_); }
        p_ = nullptr; cap_ = 0;
    }
    T* p_ = nullptr;
    size_t cap_ = 0;
};
template <class T> using DevBuf = Buf<T, false>;
template <class T> using HostBuf = Buf<T, true>;

/* A CUDA event or stream that is destroyed with its owner */
template <class H, cudaError_t (*Create)(H*, unsigned int), cudaError_t (*Destroy)(H)> class Handle {
  public:
    Handle() = default;
    Handle(const Handle&) = delete;
    Handle& operator=(const Handle&) = delete;
    ~Handle() { if (h_) Destroy(h_); }
    cudaError_t create(unsigned int flags) { return Create(&h_, flags); }
    H get() const { return h_; }

  private:
    H h_ = nullptr;
};
using Event = Handle<cudaEvent_t, cudaEventCreateWithFlags, cudaEventDestroy>;
using Stream = Handle<cudaStream_t, cudaStreamCreateWithFlags, cudaStreamDestroy>;

/* ------------------------------------------------------------------ index */

struct TermInfo {
    uint32_t blk_begin = 0;
    uint32_t nblocks = 0;
    uint32_t termfreq = 0;
    uint32_t wdf_ub = 0;
    uint64_t collfreq = 0;
    uint64_t bytes = 0; /* docs + tfs + headers */
    uint64_t bm_off = XGM_NO_BITMAP, rk_off = 0; /* membership bitmap + rank directory (u32 units) */
};

struct HostSlot {
    bool present = false;
    bool exact = true; /* every value is represented one-to-one by its 8-byte key */
    std::vector<uint32_t> voff;
    std::vector<uint64_t> vals;
};

struct xgm_index {
    int device = 0;
    uint32_t doccount = 0, lastdocid = 0;
    uint64_t total_length = 0;
    uint32_t doclen_lb = 0, doclen_ub = 0;
    uint64_t npostings = 0, nblocks = 0;
    uint64_t bytes_docs = 0, bytes_tfs = 0, bytes_hdr = 0, bytes_doclen = 0, bytes_bitmaps = 0;
    uint32_t nbitmaps = 0;
    uint64_t revision = 0;
    std::vector<TermInfo> terms;
    std::unordered_map<std::string, uint32_t> dict;
    bool synthetic_names = false; /* "T%06u" names resolved arithmetically, no dictionary */
    /* Large batches fill the GPU on their own: the kernels of all searchers of this index go through one
     * FIFO compute stream (copies stay on the searchers' streams), so that batch k's results are not
     * delayed by batch k+1's kernels sharing the SMs with them.  Declared before the arrays: destroyed after them. */
    mutable Stream compute_stream;
    mutable std::mutex launch_mu;
    /* device */
    DevBuf<XgmBlockHdr> d_hdr;
    DevBuf<uint32_t> d_docs; /* the kernels read it as uint4 */
    DevBuf<uint32_t> d_tfs;
    DevBuf<uint32_t> d_doclen;
    DevBuf<uint32_t> d_bitmaps;
    DevBuf<uint32_t> d_coarse; /* a bit per 8 docids of d_bitmaps (xgm_format.h) */
    DevBuf<uint32_t> d_ranks;
    DevBuf<uint32_t> d_voff[XGM_MAX_SLOTS];
    DevBuf<uint64_t> d_vals[XGM_MAX_SLOTS];
    uint64_t slot_max[XGM_MAX_SLOTS] = {};
    uint64_t slot_min[XGM_MAX_SLOTS] = {};
    uint32_t slot_freq[XGM_MAX_SLOTS] = {}; /* documents with a value in the slot (Database::get_value_freq) */
    /* least and greatest first value of a document: the slot's value bounds as a stock value range, which reads
     * the first value, sees them (Database::get_value_lower_bound / get_value_upper_bound) */
    uint64_t slot_first_min[XGM_MAX_SLOTS] = {};
    uint64_t slot_first_max[XGM_MAX_SLOTS] = {};
    bool slot_exact[XGM_MAX_SLOTS] = {};
    int sm_count = 132; /* H100 SXM; replaced by the device's count at upload */
    /* the members free their arrays and stream on the index's device, also when a build failed half-way */
    ~xgm_index() { cudaSetDevice(device); }
};

/* Compressed form of a contiguous range of terms, produced by one builder thread. */
struct Chunk {
    std::vector<XgmBlockHdr> hdr;
    std::vector<uint32_t> docs; /* packed words, 4*bits words per block */
    std::vector<uint32_t> tfs;
    std::vector<uint32_t> bitmaps; /* membership bitmaps of the frequent terms of this chunk */
    std::vector<uint32_t> ranks;
};

/* Terms with termfreq >= lastdocid / K get a membership bitmap (K bits per posting at most).
 * XGM_BITMAP_K=0 disables the bitmaps (everything goes through the block-decoding intersection). */
static uint32_t bitmap_k() {
    const char* e = getenv("XGM_BITMAP_K");
    return e ? (uint32_t)strtoul(e, nullptr, 10) : 256u;
}
static uint32_t bitmap_min_df(uint32_t lastdocid) {
    uint32_t k = bitmap_k();
    if (k == 0) return 0xffffffffu;
    return std::max<uint32_t>(64u, lastdocid / k);
}

static inline void pack_bits(std::vector<uint32_t>& out, const uint32_t* v, uint32_t n, uint32_t bits) {
    /* 128 slots x bits, little-endian bit order; slots >= n are zero */
    if (bits == 0) return;
    size_t base = out.size();
    out.resize(base + 4 * (size_t)bits, 0u);
    uint32_t* w = out.data() + base;
    for (uint32_t i = 0; i < n; ++i) {
        uint64_t o = (uint64_t)i * bits;
        uint32_t wi = (uint32_t)(o >> 5), sh = (uint32_t)(o & 31);
        uint64_t val = (uint64_t)v[i] << sh;
        w[wi] |= (uint32_t)val;
        if (sh + bits > 32) w[wi + 1] |= (uint32_t)(val >> 32);
    }
}

/* Append one term's postings to a chunk in the block format of xgm_format.h. */
static void compress_term(Chunk& c, const uint32_t* docids, const uint32_t* wdfs, uint32_t n, TermInfo& ti,
                          uint32_t lastdocid = 0, uint32_t min_bitmap_df = 0xffffffffu) {
    if (n >= min_bitmap_df && n > 0 && lastdocid >= docids[n - 1]) {
        const size_t ngroups = (size_t)lastdocid / 256 + 1;
        ti.bm_off = c.bitmaps.size(); /* chunk-relative, fixed up later */
        ti.rk_off = c.ranks.size();
        c.bitmaps.resize(c.bitmaps.size() + ngroups * 8, 0u);
        c.ranks.resize(c.ranks.size() + ngroups + 1, 0u);
        uint32_t* bm = c.bitmaps.data() + ti.bm_off;
        uint32_t* rk = c.ranks.data() + ti.rk_off;
        for (uint32_t i = 0; i < n; ++i) bm[docids[i] >> 5] |= 1u << (docids[i] & 31);
        uint32_t acc = 0;
        for (size_t g = 0; g < ngroups; ++g) {
            rk[g] = acc;
            for (int w = 0; w < 8; ++w) acc += (uint32_t)__builtin_popcount(bm[g * 8 + w]);
        }
        rk[ngroups] = acc;
    }
    ti.blk_begin = (uint32_t)c.hdr.size(); /* chunk-relative, fixed up later */
    ti.nblocks = (n + XGM_BLOCK - 1) / XGM_BLOCK;
    ti.termfreq = n;
    uint32_t delta[XGM_BLOCK];
    size_t d0 = c.docs.size(), t0 = c.tfs.size();
    for (uint32_t b = 0; b < ti.nblocks; ++b) {
        uint32_t off = b * XGM_BLOCK;
        uint32_t cnt = std::min<uint32_t>(XGM_BLOCK, n - off);
        uint32_t maxd = 0, maxw = 0;
        delta[0] = 0;
        for (uint32_t i = 1; i < cnt; ++i) {
            delta[i] = docids[off + i] - docids[off + i - 1] - 1;
            maxd = std::max(maxd, delta[i]);
        }
        for (uint32_t i = 0; i < cnt; ++i) maxw = std::max(maxw, wdfs[off + i]);
        uint32_t db = bits_for(maxd), tb = bits_for(maxw);
        XgmBlockHdr h;
        h.first = docids[off];
        h.doc_off = (uint32_t)(c.docs.size() / 4);
        h.tf_off = (uint32_t)(c.tfs.size() / 4);
        h.meta = db | (tb << 8) | ((cnt - 1) << 16) | (std::min<uint32_t>(maxw, 255u) << 24);
        c.hdr.push_back(h);
        pack_bits(c.docs, delta, cnt, db);
        pack_bits(c.tfs, wdfs + off, cnt, tb);
    }
    XgmBlockHdr s;
    s.first = XGM_SENTINEL;
    s.doc_off = (uint32_t)(c.docs.size() / 4);
    s.tf_off = (uint32_t)(c.tfs.size() / 4);
    s.meta = 0;
    c.hdr.push_back(s);
    ti.bytes = (c.docs.size() - d0) * 4 + (c.tfs.size() - t0) * 4 + (uint64_t)ti.nblocks * sizeof(XgmBlockHdr);
}

/* reference wdf upper bound: glass_postlist.cc:175-190 + glass_database.cc:822-829 */
static uint32_t derive_wdf_ub(uint32_t tf, uint64_t cf, uint32_t first_wdf, uint32_t db_wdf_ub) {
    uint64_t ub;
    if (cf == 0 || tf == 1) ub = cf;
    else ub = (cf - first_wdf > first_wdf) ? cf - first_wdf : first_wdf;
    if (ub > db_wdf_ub) ub = db_wdf_ub;
    return (uint32_t)ub;
}

struct xgm_builder {
    uint32_t doccount = 0, lastdocid = 0;
    uint64_t total_length = 0;
    uint32_t doclen_lb = 0, doclen_ub = 0;
    std::vector<uint32_t> doclen;
    std::vector<std::string> names;
    std::vector<TermInfo> terms;
    std::vector<uint32_t> first_wdf;
    std::vector<bool> ub_given;
    uint32_t db_wdf_ub = 0;
    Chunk chunk; /* sequential builder: one chunk */
    HostSlot slots[XGM_MAX_SLOTS];
    bool have_docs = false;
    uint64_t revision = 0;
};

static xgm_status upload_index(xgm_index* ix, std::vector<Chunk>& chunks, const std::vector<size_t>& chunk_first_term,
                               const std::vector<uint32_t>& doclen, HostSlot* slots, int device) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
        return fail(XGM_E_NODEVICE, "no CUDA device visible: libxgm has no CPU path");
    if (device < 0 || device >= ndev) return fail(XGM_E_INVALID, "device %d out of range (%d visible)", device, ndev);
    CUDA_TRY(cudaSetDevice(device));
    ix->device = device;
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    ix->sm_count = prop.multiProcessorCount;
    /* global bases per chunk */
    size_t nh = 0, nd = 0, nt = 0, nbm = 0, nrk = 0;
    std::vector<size_t> hb(chunks.size()), dbase(chunks.size()), tb(chunks.size()), bmb(chunks.size()), rkb(chunks.size());
    for (size_t i = 0; i < chunks.size(); ++i) {
        hb[i] = nh; dbase[i] = nd; tb[i] = nt; bmb[i] = nbm; rkb[i] = nrk;
        nh += chunks[i].hdr.size(); nd += chunks[i].docs.size(); nt += chunks[i].tfs.size();
        nbm += chunks[i].bitmaps.size(); nrk += chunks[i].ranks.size();
    }
    if (nh >= 0xffffffffull || nd / 4 >= 0xffffffffull || nt / 4 >= 0xffffffffull)
        return fail(XGM_E_INVALID, "index too large for 32-bit block offsets");
    /* fix up offsets */
    parallel_for(chunks.size(), default_threads(), [&](size_t i, int) {
        uint32_t dadd = (uint32_t)(dbase[i] / 4), tadd = (uint32_t)(tb[i] / 4);
        for (auto& h : chunks[i].hdr) { h.doc_off += dadd; h.tf_off += tadd; }
        size_t t_begin = chunk_first_term[i], t_end = chunk_first_term[i + 1];
        for (size_t t = t_begin; t < t_end; ++t) {
            ix->terms[t].blk_begin += (uint32_t)hb[i];
            if (ix->terms[t].bm_off != XGM_NO_BITMAP) { ix->terms[t].bm_off += bmb[i]; ix->terms[t].rk_off += rkb[i]; }
        }
    });
    CUDA_TRY(ix->d_bitmaps.alloc(std::max<size_t>(nbm, 8)));
    CUDA_TRY(ix->d_ranks.alloc(std::max<size_t>(nrk, 8)));
    for (size_t i = 0; i < chunks.size(); ++i) {
        if (!chunks[i].bitmaps.empty())
            CUDA_TRY(cudaMemcpy(ix->d_bitmaps.get() + bmb[i], chunks[i].bitmaps.data(), chunks[i].bitmaps.size() * 4, cudaMemcpyHostToDevice));
        if (!chunks[i].ranks.empty())
            CUDA_TRY(cudaMemcpy(ix->d_ranks.get() + rkb[i], chunks[i].ranks.data(), chunks[i].ranks.size() * 4, cudaMemcpyHostToDevice));
        std::vector<uint32_t>().swap(chunks[i].bitmaps);
        std::vector<uint32_t>().swap(chunks[i].ranks);
    }
    /* the coarse bitmaps: one word per 8 fine words, so a term's coarse word of docid d is coarse[bm_off / 8 + (d >> 8)] */
    for (const auto& t : ix->terms)
        if (t.bm_off != XGM_NO_BITMAP && (t.bm_off & 7u) != 0)
            return fail(XGM_E_INVALID, "membership bitmap offset %llu is not a multiple of 8 words", (unsigned long long)t.bm_off);
    const size_t ncoarse = nbm / 8;
    CUDA_TRY(ix->d_coarse.alloc(std::max<size_t>(ncoarse, 8)));
    CUDA_TRY(xgm_launch_coarse(ix->d_bitmaps.get(), ncoarse, ix->d_coarse.get(), 0));
    CUDA_TRY(cudaDeviceSynchronize());
    ix->bytes_bitmaps = (nbm + ncoarse + nrk) * 4;
    /* +16 bytes slack at the end of each column: the unpackers may read one word past a block */
    CUDA_TRY(ix->d_hdr.alloc(nh + 1));
    CUDA_TRY(ix->d_docs.alloc(nd + 16));
    CUDA_TRY(ix->d_tfs.alloc(nt + 16));
    CUDA_TRY(cudaMemset(ix->d_docs.get() + nd, 0, 64));
    CUDA_TRY(cudaMemset(ix->d_tfs.get() + nt, 0, 64));
    for (size_t i = 0; i < chunks.size(); ++i) {
        if (!chunks[i].hdr.empty())
            CUDA_TRY(cudaMemcpy(ix->d_hdr.get() + hb[i], chunks[i].hdr.data(), chunks[i].hdr.size() * sizeof(XgmBlockHdr), cudaMemcpyHostToDevice));
        if (!chunks[i].docs.empty())
            CUDA_TRY(cudaMemcpy(ix->d_docs.get() + dbase[i], chunks[i].docs.data(), chunks[i].docs.size() * 4, cudaMemcpyHostToDevice));
        if (!chunks[i].tfs.empty())
            CUDA_TRY(cudaMemcpy(ix->d_tfs.get() + tb[i], chunks[i].tfs.data(), chunks[i].tfs.size() * 4, cudaMemcpyHostToDevice));
        std::vector<XgmBlockHdr>().swap(chunks[i].hdr);
        std::vector<uint32_t>().swap(chunks[i].docs);
        std::vector<uint32_t>().swap(chunks[i].tfs);
    }
    XgmBlockHdr tail;
    tail.first = XGM_SENTINEL; tail.doc_off = 0; tail.tf_off = 0; tail.meta = 0;
    CUDA_TRY(cudaMemcpy(ix->d_hdr.get() + nh, &tail, sizeof(tail), cudaMemcpyHostToDevice));
    CUDA_TRY(ix->d_doclen.alloc(doclen.size()));
    CUDA_TRY(cudaMemcpy(ix->d_doclen.get(), doclen.data(), doclen.size() * 4, cudaMemcpyHostToDevice));
    for (int s = 0; s < XGM_MAX_SLOTS; ++s) {
        if (!slots || !slots[s].present) continue;
        CUDA_TRY(ix->d_voff[s].alloc(slots[s].voff.size()));
        CUDA_TRY(cudaMemcpy(ix->d_voff[s].get(), slots[s].voff.data(), slots[s].voff.size() * 4, cudaMemcpyHostToDevice));
        CUDA_TRY(ix->d_vals[s].alloc(std::max<size_t>(1, slots[s].vals.size())));
        if (!slots[s].vals.empty())
            CUDA_TRY(cudaMemcpy(ix->d_vals[s].get(), slots[s].vals.data(), slots[s].vals.size() * 8, cudaMemcpyHostToDevice));
        ix->slot_min[s] = slots[s].vals.empty() ? 0 : ~0ull;
        for (uint64_t v : slots[s].vals) { ix->slot_max[s] = std::max(ix->slot_max[s], v); ix->slot_min[s] = std::min(ix->slot_min[s], v); }
        ix->slot_first_min[s] = slots[s].vals.empty() ? 0 : ~0ull;
        for (size_t d = 0; d + 1 < slots[s].voff.size(); ++d) {
            if (slots[s].voff[d + 1] == slots[s].voff[d]) continue;
            const uint64_t v = slots[s].vals[slots[s].voff[d]];
            ++ix->slot_freq[s];
            ix->slot_first_min[s] = std::min(ix->slot_first_min[s], v);
            ix->slot_first_max[s] = std::max(ix->slot_first_max[s], v);
        }
        ix->slot_exact[s] = slots[s].exact;
    }
    ix->nblocks = 0;
    ix->npostings = 0;
    ix->nbitmaps = 0;
    for (auto& t : ix->terms) { ix->nblocks += t.nblocks; ix->npostings += t.termfreq; ix->nbitmaps += t.bm_off != XGM_NO_BITMAP; }
    ix->bytes_docs = nd * 4;
    ix->bytes_tfs = nt * 4;
    ix->bytes_hdr = nh * sizeof(XgmBlockHdr);
    ix->bytes_doclen = doclen.size() * 4;
    return XGM_OK;
}

extern "C" xgm_status xgm_builder_new(xgm_builder** out) {
    if (!out) return fail(XGM_E_INVALID, "null out");
    *out = new (std::nothrow) xgm_builder();
    return *out ? XGM_OK : fail(XGM_E_NOMEM, "out of memory");
}

extern "C" void xgm_builder_free(xgm_builder* b) { delete b; }

extern "C" xgm_status xgm_builder_set_docs(xgm_builder* b, uint32_t doccount, uint32_t lastdocid, uint64_t total_length,
                                           uint32_t doclen_lb, uint32_t doclen_ub, const uint32_t* doclen) {
    if (!b || !doclen) return fail(XGM_E_INVALID, "null argument");
    b->doccount = doccount; b->lastdocid = lastdocid; b->total_length = total_length;
    b->doclen_lb = doclen_lb; b->doclen_ub = doclen_ub;
    b->doclen.assign(doclen, doclen + (size_t)lastdocid + 1);
    b->doclen.push_back(0);
    b->have_docs = true;
    return XGM_OK;
}

extern "C" xgm_status xgm_builder_add_term(xgm_builder* b, const char* term, uint32_t term_len, const uint32_t* docids,
                                           const uint32_t* wdfs, uint32_t n, uint64_t collfreq, uint32_t wdf_ub,
                                           uint32_t* term_id) {
    if (!b || !term || (n && (!docids || !wdfs))) return fail(XGM_E_INVALID, "null argument");
    if (!b->have_docs) return fail(XGM_E_INVALID, "call xgm_builder_set_docs before xgm_builder_add_term");
    if (n && docids[n - 1] > b->lastdocid) return fail(XGM_E_INVALID, "docid %u of term beyond lastdocid %u", docids[n - 1], b->lastdocid);
    for (uint32_t i = 0; i < n; ++i) {
        if (docids[i] == 0 || docids[i] == XGM_SENTINEL || (i && docids[i] <= docids[i - 1]))
            return fail(XGM_E_INVALID, "docids of term must be strictly ascending and in [1, 2^32-2]");
        b->db_wdf_ub = std::max(b->db_wdf_ub, wdfs[i]);
    }
    TermInfo ti;
    compress_term(b->chunk, docids, wdfs, n, ti, b->have_docs ? b->lastdocid : 0,
                  b->have_docs ? bitmap_min_df(b->lastdocid) : 0xffffffffu);
    ti.collfreq = collfreq;
    ti.wdf_ub = wdf_ub;
    if (term_id) *term_id = (uint32_t)b->terms.size();
    b->terms.push_back(ti);
    b->names.emplace_back(term, term_len);
    b->first_wdf.push_back(n ? wdfs[0] : 0);
    b->ub_given.push_back(wdf_ub != 0);
    return XGM_OK;
}

/* internal: a reference-provided wdf bound of 0 is authoritative (0 otherwise means "derive it") */
xgm_status xgm_builder_force_wdf_ub(xgm_builder* b, uint32_t term_id, uint32_t wdf_ub) {
    if (!b || term_id >= b->terms.size()) return fail(XGM_E_INVALID, "bad term id");
    b->terms[term_id].wdf_ub = wdf_ub;
    b->ub_given[term_id] = true;
    return XGM_OK;
}

extern "C" xgm_status xgm_builder_add_value_slot(xgm_builder* b, uint32_t slot, const uint64_t* voff, const uint64_t* vals) {
    if (!b || !voff || slot >= XGM_MAX_SLOTS) return fail(XGM_E_INVALID, "bad slot");
    if (!b->have_docs) return fail(XGM_E_INVALID, "call xgm_builder_set_docs first");
    HostSlot& s = b->slots[slot];
    size_t n = (size_t)b->lastdocid + 2;
    if (voff[n - 1] >= 0xffffffffull) return fail(XGM_E_INVALID, "too many values");
    s.voff.resize(n);
    for (size_t i = 0; i < n; ++i) {
        if (i && voff[i] < voff[i - 1]) return fail(XGM_E_INVALID, "value offsets must not decrease");
        s.voff[i] = (uint32_t)voff[i];
    }
    s.vals.assign(vals, vals + voff[n - 1]);
    s.present = true;
    return XGM_OK;
}

extern "C" xgm_status xgm_builder_set_revision(xgm_builder* b, uint64_t revision) {
    if (!b) return fail(XGM_E_INVALID, "null argument");
    b->revision = revision;
    return XGM_OK;
}

/* ---- value keys: a slot value is its first 8 bytes, big-endian, zero padded (xgm.h) ---- */
extern "C" int xgm_value_key(const void* bytes, size_t len, uint64_t* key) {
    const unsigned char* p = static_cast<const unsigned char*>(bytes);
    uint64_t k = 0;
    for (size_t i = 0; i < 8; ++i) k = (k << 8) | (i < len ? p[i] : 0u);
    if (key) *key = k;
    return len <= 8 && (len == 0 || p[len - 1] != 0) ? 1 : 0;
}

extern "C" size_t xgm_value_key_bytes(uint64_t key, unsigned char out[8]) {
    size_t n = 8;
    while (n > 0 && ((key >> (8 * (8 - n))) & 0xffu) == 0) --n;
    for (size_t i = 0; i < n; ++i) out[i] = (unsigned char)(key >> (8 * (7 - i)));
    return n;
}

/* Multi_MultiValueKeyMaker::operator() (src/multivalue/keymaker.cc:704-757) for one SerialiseKey slot: the
 * slot is the last one, so a forward value is appended as it is (:727-731); a reverse one is subtracted
 * bytewise from 0xff, '\0' becoming "\xff\0", and followed by "\xff\xff" (:733-743). */
extern "C" size_t xgm_sort_key_bytes(uint64_t key, int reverse, unsigned char out[20]) {
    unsigned char v[8];
    size_t n = xgm_value_key_bytes(key, v);
    size_t o = 0;
    if (!reverse) {
        for (size_t i = 0; i < n; ++i) out[o++] = v[i];
        return o;
    }
    for (size_t i = 0; i < n; ++i) {
        out[o++] = (unsigned char)(255 - v[i]);
        if (v[i] == 0) out[o++] = 0;
    }
    out[o++] = 0xff; out[o++] = 0xff;
    return o;
}

/* unserialise_length, src/length.cc:62-85 (the StringList element length prefix) */
static bool read_length(const unsigned char*& p, const unsigned char* end, uint64_t& len) {
    if (p == end) return false;
    len = *p++;
    if (len == 0xff) {
        len = 0;
        unsigned shift = 0;
        unsigned char ch;
        do {
            if (p == end || shift > 63) return false;
            ch = *p++;
            len |= (uint64_t)(ch & 0x7f) << shift;
            shift += 7;
        } while ((ch & 0x80) == 0);
        len += 255;
    }
    return true;
}

extern "C" xgm_status xgm_builder_add_value_slot_serialised(xgm_builder* b, uint32_t slot, const uint64_t* off,
                                                            const unsigned char* bytes) {
    if (!b || !off || slot >= XGM_MAX_SLOTS) return fail(XGM_E_INVALID, "bad slot");
    if (!b->have_docs) return fail(XGM_E_INVALID, "call xgm_builder_set_docs first");
    HostSlot& s = b->slots[slot];
    const size_t n = (size_t)b->lastdocid + 2;
    s.voff.assign(n, 0);
    s.vals.clear();
    s.exact = true;
    for (size_t d = 0; d + 1 < n; ++d) {
        s.voff[d] = (uint32_t)s.vals.size();
        if (off[d + 1] < off[d]) return fail(XGM_E_INVALID, "value offsets must not decrease");
        const unsigned char* p = bytes + off[d];
        const unsigned char* end = bytes + off[d + 1];
        if (p == end) continue;
        uint64_t key;
        if (*p != 0) { /* a single value is stored as it is (StringList::serialise, serialise_list.h:318-322) */
            if (!xgm_value_key(p, (size_t)(end - p), &key)) s.exact = false;
            s.vals.push_back(key);
            continue;
        }
        ++p; /* SERIALISED_LIST_MAGIC */
        while (p != end) {
            uint64_t len;
            if (!read_length(p, end, len) || len > (uint64_t)(end - p))
                return fail(XGM_E_INVALID, "slot %u, docid %zu: bad StringList encoding", slot, d);
            if (!xgm_value_key(p, (size_t)len, &key)) s.exact = false;
            s.vals.push_back(key);
            p += len;
        }
        if (s.vals.size() >= 0xffffffffull) return fail(XGM_E_INVALID, "too many values");
    }
    s.voff[n - 1] = (uint32_t)s.vals.size();
    s.present = true;
    return XGM_OK;
}

extern "C" xgm_status xgm_builder_finish(xgm_builder* b, int device, xgm_index** out) {
    if (!b || !out) return fail(XGM_E_INVALID, "null argument");
    if (!b->have_docs) { delete b; return fail(XGM_E_INVALID, "xgm_builder_set_docs was not called"); }
    std::unique_ptr<xgm_index> ix(new xgm_index());
    ix->doccount = b->doccount; ix->lastdocid = b->lastdocid; ix->total_length = b->total_length;
    ix->doclen_lb = b->doclen_lb; ix->doclen_ub = b->doclen_ub;
    ix->revision = b->revision;
    ix->terms = b->terms;
    for (size_t t = 0; t < ix->terms.size(); ++t) {
        if (!b->ub_given[t])
            ix->terms[t].wdf_ub = derive_wdf_ub(ix->terms[t].termfreq, ix->terms[t].collfreq, b->first_wdf[t], b->db_wdf_ub);
        ix->dict.emplace(b->names[t], (uint32_t)t);
    }
    std::vector<Chunk> chunks;
    chunks.emplace_back(std::move(b->chunk));
    std::vector<size_t> first = {0, ix->terms.size()};
    xgm_status st = upload_index(ix.get(), chunks, first, b->doclen, b->slots, device);
    delete b;
    if (st != XGM_OK) return st;
    *out = ix.release();
    return XGM_OK;
}

extern "C" void xgm_index_close(xgm_index* ix) { delete ix; }

/* ---- synthetic corpus straight into the block format (bench / tests) ---------------------- */

extern "C" xgm_status xgm_index_build_synthetic(uint32_t ndocs, uint32_t vocab, uint64_t seed, uint32_t nshards,
                                                uint32_t shard, int with_values, int device, int host_threads,
                                                xgm_index** out) {
    if (!out || nshards == 0 || shard >= nshards || vocab == 0) return fail(XGM_E_INVALID, "bad arguments");
    int T = host_threads > 0 ? host_threads : default_threads();
    xgm_zipf z;
    if (xgm_zipf_init(&z, vocab)) return fail(XGM_E_NOMEM, "zipf table");
    uint32_t nlocal = shard < ndocs ? (ndocs - shard - 1) / nshards + 1 : 0;
    std::unique_ptr<xgm_index> ix(new xgm_index());
    ix->doccount = ix->lastdocid = nlocal;
    ix->synthetic_names = true;
    std::vector<uint32_t> doclen((size_t)nlocal + 2, 0);
    /* pass 1: per-thread, per-term posting counts over contiguous local-docid ranges */
    size_t per = ((size_t)nlocal + T - 1) / T;
    if (per == 0) per = 1;
    int nparts = (int)(((size_t)nlocal + per - 1) / per);
    if (nparts < 1) nparts = 1;
    std::vector<std::vector<uint32_t>> cnt(nparts);
    std::vector<uint64_t> part_len(nparts, 0);
    std::vector<uint32_t> part_lb(nparts, 0xffffffffu), part_ub(nparts, 0), part_wub(nparts, 0);
    parallel_for((size_t)nparts, T, [&](size_t pi, int) {
        cnt[pi].assign(vocab, 0);
        uint32_t ranks[XGM_CORPUS_MAX_LEN], wdf[XGM_CORPUS_MAX_LEN];
        size_t a = pi * per + 1, b = std::min<size_t>((size_t)nlocal, (pi + 1) * per);
        for (size_t l = a; l <= b; ++l) {
            uint32_t gd = (uint32_t)((l - 1) * nshards + shard + 1);
            uint32_t len = xgm_corpus_doc(&z, seed, gd, ranks);
            uint32_t n = xgm_corpus_collapse(ranks, len, wdf);
            for (uint32_t i = 0; i < n; ++i) { cnt[pi][ranks[i]]++; part_wub[pi] = std::max(part_wub[pi], wdf[i]); }
            doclen[l] = len;
            part_len[pi] += len;
            part_lb[pi] = std::min(part_lb[pi], len);
            part_ub[pi] = std::max(part_ub[pi], len);
        }
    });
    uint32_t db_wdf_ub = 0;
    ix->doclen_lb = nlocal ? 0xffffffffu : 0;
    for (int pi = 0; pi < nparts; ++pi) {
        ix->total_length += part_len[pi];
        ix->doclen_lb = std::min(ix->doclen_lb, part_lb[pi]);
        ix->doclen_ub = std::max(ix->doclen_ub, part_ub[pi]);
        db_wdf_ub = std::max(db_wdf_ub, part_wub[pi]);
    }
    /* term offsets, then per-part write cursors */
    std::vector<uint64_t> off((size_t)vocab + 1, 0);
    for (uint32_t t = 0; t < vocab; ++t) {
        uint64_t s = 0;
        for (int pi = 0; pi < nparts; ++pi) s += cnt[pi][t];
        off[t + 1] = off[t] + s;
    }
    uint64_t total = off[vocab];
    std::vector<uint32_t> docids(total), wdfs(total);
    /* convert counts into start cursors (part-major within a term keeps docids ascending) */
    parallel_for((size_t)T, T, [&](size_t ti, int) {
        size_t a = (size_t)vocab * ti / T, b = (size_t)vocab * (ti + 1) / T;
        for (size_t t = a; t < b; ++t) {
            uint64_t cur = off[t];
            for (int pi = 0; pi < nparts; ++pi) { uint32_t c = cnt[pi][t]; cnt[pi][t] = (uint32_t)(cur - off[t]); cur += c; }
        }
    });
    parallel_for((size_t)nparts, T, [&](size_t pi, int) {
        uint32_t ranks[XGM_CORPUS_MAX_LEN], wdf[XGM_CORPUS_MAX_LEN];
        size_t a = pi * per + 1, b = std::min<size_t>((size_t)nlocal, (pi + 1) * per);
        std::vector<uint32_t>& cur = cnt[pi];
        for (size_t l = a; l <= b; ++l) {
            uint32_t gd = (uint32_t)((l - 1) * nshards + shard + 1);
            uint32_t len = xgm_corpus_doc(&z, seed, gd, ranks);
            uint32_t n = xgm_corpus_collapse(ranks, len, wdf);
            for (uint32_t i = 0; i < n; ++i) {
                uint64_t p = off[ranks[i]] + cur[ranks[i]]++;
                docids[p] = (uint32_t)l;
                wdfs[p] = wdf[i];
            }
        }
    });
    cnt.clear();
    cnt.shrink_to_fit();
    /* compress: contiguous term ranges balanced by posting count */
    int nchunks = std::max(1, T * 4);
    std::vector<size_t> first(nchunks + 1, 0);
    {
        size_t t = 0;
        for (int c = 1; c < nchunks; ++c) {
            uint64_t target = total / nchunks * c;
            while (t < vocab && off[t] < target) ++t;
            first[c] = t;
        }
        first[nchunks] = vocab;
        for (int c = 1; c <= nchunks; ++c) first[c] = std::max(first[c], first[c - 1]);
    }
    ix->terms.resize(vocab);
    std::vector<Chunk> chunks(nchunks);
    parallel_for((size_t)nchunks, T, [&](size_t c, int) {
        for (size_t t = first[c]; t < first[c + 1]; ++t) {
            uint32_t n = (uint32_t)(off[t + 1] - off[t]);
            TermInfo& ti = ix->terms[t];
            compress_term(chunks[c], docids.data() + off[t], wdfs.data() + off[t], n, ti, nlocal, bitmap_min_df(nlocal));
            uint64_t cf = 0;
            for (uint64_t p = off[t]; p < off[t + 1]; ++p) cf += wdfs[p];
            ti.collfreq = cf;
            ti.wdf_ub = n ? derive_wdf_ub(n, cf, wdfs[off[t]], db_wdf_ub) : 0;
        }
    });
    std::vector<uint32_t>().swap(docids);
    std::vector<uint32_t>().swap(wdfs);
    HostSlot slots[XGM_MAX_SLOTS];
    if (with_values) {
        slots[0].present = slots[1].present = true;
        slots[0].voff.assign((size_t)nlocal + 2, 0);
        slots[1].voff.assign((size_t)nlocal + 2, 0);
        slots[1].vals.assign((size_t)nlocal, 0);
        std::vector<uint8_t> n0((size_t)nlocal + 1, 0);
        std::vector<uint64_t> v0(3 * ((size_t)nlocal + 1), 0);
        parallel_for((size_t)nparts, T, [&](size_t pi, int) {
            size_t a = pi * per + 1, b = std::min<size_t>((size_t)nlocal, (pi + 1) * per);
            for (size_t l = a; l <= b; ++l) {
                uint32_t gd = (uint32_t)((l - 1) * nshards + shard + 1);
                uint64_t v[3], v1;
                uint32_t k = xgm_corpus_values(seed, gd, v, &v1);
                n0[l] = (uint8_t)k;
                for (uint32_t i = 0; i < k; ++i) v0[3 * l + i] = v[i];
                slots[1].vals[l - 1] = v1;
            }
        });
        uint32_t acc = 0;
        slots[0].voff[0] = slots[0].voff[1] = 0;
        for (size_t l = 1; l <= nlocal; ++l) {
            slots[0].voff[l] = acc;
            acc += n0[l];
            slots[1].voff[l] = (uint32_t)(l - 1);
        }
        slots[0].voff[(size_t)nlocal + 1] = acc;
        slots[1].voff[(size_t)nlocal + 1] = nlocal;
        slots[0].vals.resize(acc);
        for (size_t l = 1; l <= nlocal; ++l)
            for (uint32_t i = 0; i < n0[l]; ++i) slots[0].vals[slots[0].voff[l] + i] = v0[3 * l + i];
    }
    xgm_zipf_free(&z);
    xgm_status st = upload_index(ix.get(), chunks, first, doclen, slots, device);
    if (st != XGM_OK) return st;
    *out = ix.release();
    return XGM_OK;
}

/* ---- XGMFLAT1 loader -------------------------------------------------------------------- */

static bool rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }

extern "C" xgm_status xgm_index_load_flat(const char* path, int device, xgm_index** out) {
    if (!path || !out) return fail(XGM_E_INVALID, "null argument");
    FILE* f = fopen(path, "rb");
    if (!f) return fail(XGM_E_IO, "cannot open %s", path);
    char magic[8];
    uint32_t doccount, lastdocid, nterms, nslots, lb, ub;
    uint64_t total_length;
    if (!rd(f, magic, 8) || memcmp(magic, "XGMFLAT1", 8) || !rd(f, &doccount, 4) || !rd(f, &lastdocid, 4) ||
        !rd(f, &total_length, 8) || !rd(f, &nterms, 4) || !rd(f, &nslots, 4) || !rd(f, &lb, 4) || !rd(f, &ub, 4)) {
        fclose(f);
        return fail(XGM_E_IO, "%s: bad XGMFLAT1 header", path);
    }
    xgm_builder* b = nullptr;
    xgm_status st = xgm_builder_new(&b);
    if (st != XGM_OK) { fclose(f); return st; }
    std::vector<uint32_t> dl((size_t)lastdocid + 1);
    if (!rd(f, dl.data(), dl.size() * 4)) { fclose(f); delete b; return fail(XGM_E_IO, "%s: truncated", path); }
    xgm_builder_set_docs(b, doccount, lastdocid, total_length, lb, ub, dl.data());
    std::vector<uint32_t> dids, wdfs;
    std::string name;
    for (uint32_t t = 0; t < nterms; ++t) {
        uint32_t nl, tf, wub, n;
        uint64_t cf;
        if (!rd(f, &nl, 4)) goto trunc;
        name.resize(nl);
        if (!rd(f, &name[0], nl) || !rd(f, &tf, 4) || !rd(f, &cf, 8) || !rd(f, &wub, 4) || !rd(f, &n, 4)) goto trunc;
        dids.resize(n); wdfs.resize(n);
        if (!rd(f, dids.data(), (size_t)n * 4) || !rd(f, wdfs.data(), (size_t)n * 4)) goto trunc;
        st = xgm_builder_add_term(b, name.data(), nl, dids.data(), wdfs.data(), n, cf, wub, nullptr);
        if (st != XGM_OK) { fclose(f); delete b; return st; }
        /* the reference's own bound is authoritative even when it is 0 */
        b->terms.back().wdf_ub = wub;
        b->ub_given.back() = true;
    }
    /* value slots: numeric slots hold sortable_serialise()d doubles; decoding them is the shim's job
     * (INTEGRATION.md); the flat file keeps raw bytes, so slots are added through
     * xgm_builder_add_value_slot by the caller when needed. */
    fclose(f);
    return xgm_builder_finish(b, device, out);
trunc:
    fclose(f);
    delete b;
    return fail(XGM_E_IO, "%s: truncated", path);
}

extern "C" xgm_status xgm_index_value_freq(const xgm_index* ix, uint32_t slot, uint32_t* out) {
    if (!ix || !out || slot >= XGM_MAX_SLOTS) return fail(XGM_E_INVALID, "bad arguments");
    *out = ix->slot_freq[slot];
    return XGM_OK;
}

extern "C" xgm_status xgm_index_info_get(const xgm_index* ix, xgm_index_info* o) {
    if (!ix || !o) return fail(XGM_E_INVALID, "null argument");
    memset(o, 0, sizeof(*o));
    o->doccount = ix->doccount; o->lastdocid = ix->lastdocid; o->total_length = ix->total_length;
    o->doclen_lower_bound = ix->doclen_lb; o->doclen_upper_bound = ix->doclen_ub;
    o->nterms = (uint32_t)ix->terms.size(); o->npostings = ix->npostings; o->nblocks = ix->nblocks;
    o->bytes_docids = ix->bytes_docs; o->bytes_wdfs = ix->bytes_tfs; o->bytes_headers = ix->bytes_hdr;
    o->bytes_doclen = ix->bytes_doclen; o->device = ix->device; o->revision = ix->revision;
    o->bytes_bitmaps = ix->bytes_bitmaps; o->nbitmaps = ix->nbitmaps;
    return XGM_OK;
}

static bool lookup_term(const xgm_index* ix, const char* term, uint32_t len, uint32_t* id) {
    if (ix->synthetic_names) {
        if (len < 2 || term[0] != 'T') return false;
        uint64_t r = 0;
        for (uint32_t i = 1; i < len; ++i) {
            if (term[i] < '0' || term[i] > '9') return false;
            r = r * 10 + (uint64_t)(term[i] - '0');
            if (r > 0xffffffffull) return false;
        }
        if (r >= ix->terms.size()) return false;
        char b[16];
        int k = xgm_corpus_term((uint32_t)r, b);
        if ((uint32_t)k != len || memcmp(b, term, len) != 0) return false;
        *id = (uint32_t)r;
        return true;
    }
    auto it = ix->dict.find(std::string(term, len));
    if (it == ix->dict.end()) return false;
    *id = it->second;
    return true;
}

extern "C" xgm_status xgm_term_stats_get(const xgm_index* ix, const char* term, uint32_t len, xgm_term_stats* o) {
    if (!ix || !term || !o) return fail(XGM_E_INVALID, "null argument");
    memset(o, 0, sizeof(*o));
    o->term_id = 0xffffffffu;
    uint32_t id;
    if (!lookup_term(ix, term, len, &id)) return XGM_OK;
    const TermInfo& t = ix->terms[id];
    o->term_id = id; o->termfreq = t.termfreq; o->collfreq = t.collfreq; o->wdf_upper_bound = t.wdf_ub; o->bytes = t.bytes;
    return XGM_OK;
}

extern "C" xgm_status xgm_term_stats_many(const xgm_index* ix, uint32_t n, const char* const* terms, const uint32_t* lens,
                                          uint32_t* termfreq) {
    if (!ix || (n && (!terms || !termfreq))) return fail(XGM_E_INVALID, "null argument");
    for (uint32_t i = 0; i < n; ++i) {
        uint32_t id;
        const uint32_t len = lens ? lens[i] : (uint32_t)strlen(terms[i]);
        termfreq[i] = lookup_term(ix, terms[i], len, &id) ? ix->terms[id].termfreq : 0u;
    }
    return XGM_OK;
}

static void fill_index_params(const xgm_index* ix, XgmKernelParams& p) {
    memset(&p, 0, sizeof(p));
    p.hdr = ix->d_hdr.get(); p.docs = reinterpret_cast<const uint4*>(ix->d_docs.get());
    p.tfs = reinterpret_cast<const uint4*>(ix->d_tfs.get()); p.doclen = ix->d_doclen.get(); p.lastdocid = ix->lastdocid;
    p.bitmaps = ix->d_bitmaps.get(); p.coarse = ix->d_coarse.get(); p.ranks = ix->d_ranks.get(); p.doclen_lb = ix->doclen_lb;
    for (int s = 0; s < XGM_MAX_SLOTS; ++s) { p.slots[s].voff = ix->d_voff[s].get(); p.slots[s].vals = ix->d_vals[s].get(); }
}

extern "C" xgm_status xgm_index_decode_term(const xgm_index* ix, uint32_t term_id, uint32_t* docids, uint32_t* wdfs,
                                            uint32_t capacity, uint32_t* n) {
    if (!ix || !n) return fail(XGM_E_INVALID, "null argument");
    if (term_id >= ix->terms.size()) return fail(XGM_E_INVALID, "term id out of range");
    const TermInfo& t = ix->terms[term_id];
    *n = t.termfreq;
    if (t.termfreq == 0 || (!docids && !wdfs && capacity == 0)) return XGM_OK;
    if (capacity < t.termfreq || !docids || !wdfs) return fail(XGM_E_INVALID, "capacity %u < termfreq %u", capacity, t.termfreq);
    CUDA_TRY(cudaSetDevice(ix->device));
    DevBuf<uint32_t> dd, dw;
    size_t cap = (size_t)t.nblocks * XGM_BLOCK;
    CUDA_TRY(dd.alloc(cap));
    CUDA_TRY(dw.alloc(cap));
    XgmKernelParams p;
    fill_index_params(ix, p);
    CUDA_TRY(xgm_launch_decode(p, t.blk_begin, t.nblocks, ix->sm_count, dd.get(), dw.get(), 0));
    CUDA_TRY(cudaMemcpy(docids, dd.get(), (size_t)t.termfreq * 4, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(wdfs, dw.get(), (size_t)t.termfreq * 4, cudaMemcpyDeviceToHost));
    return XGM_OK;
}

/* ------------------------------------------------------------------ planner pool */

/* Query planning is independent per query; large batches are split over a few helper threads.  The helpers
 * live as long as the process (one pool, shared by all searchers): spawning threads per batch cost more than
 * the planning itself once several searchers and several ranks per box were submitting at the same time. */
class PlannerPool {
  public:
    /* never destroyed: its helper threads are detached and wait on the condition variable for the life of the
     * process (destroying a condition variable that has waiters blocks in glibc — at exit() of the host program) */
    static PlannerPool& get() { static PlannerPool* p = new PlannerPool(); return *p; }
    /* run fn(part) for part in [0, nparts) on the pool (the caller takes parts too); returns when all are done */
    void run(int nparts, const std::function<void(int)>& fn) {
        if (nparts <= 1 || nthreads_ == 0) { for (int i = 0; i < nparts; ++i) fn(i); return; }
        std::unique_lock<std::mutex> lk(mu_);
        run_cv_.wait(lk, [&] { return !busy_; }); /* one batch at a time */
        busy_ = true; fn_ = &fn; nparts_ = nparts; next_ = 0; done_ = 0; ++gen_;
        lk.unlock();
        cv_.notify_all();
        work();
        lk.lock();
        done_cv_.wait(lk, [&] { return done_ == nparts_; });
        busy_ = false; fn_ = nullptr;
        lk.unlock();
        run_cv_.notify_one();
    }
    int threads() const { return nthreads_ + 1; }

  private:
    PlannerPool() {
        int t = std::min(default_threads(), 8);
        if (const char* e = getenv("XGM_HOST_THREADS")) t = std::max(1, atoi(e));
        nthreads_ = t - 1;
        for (int i = 0; i < nthreads_; ++i) std::thread([this] { loop(); }).detach();
    }
    void work() {
        for (;;) {
            int i;
            {
                std::lock_guard<std::mutex> lk(mu_);
                if (!fn_ || next_ >= nparts_) return;
                i = next_++;
            }
            (*fn_)(i);
            bool last;
            {
                std::lock_guard<std::mutex> lk(mu_);
                last = ++done_ == nparts_;
            }
            if (last) done_cv_.notify_all();
        }
    }
    void loop() {
        uint64_t seen = 0;
        for (;;) {
            {
                std::unique_lock<std::mutex> lk(mu_);
                cv_.wait(lk, [&] { return gen_ != seen; });
                seen = gen_;
            }
            work();
        }
    }
    std::mutex mu_;
    std::condition_variable cv_, done_cv_, run_cv_;
    const std::function<void(int)>* fn_ = nullptr;
    int nthreads_ = 0, nparts_ = 0, next_ = 0, done_ = 0;
    uint64_t gen_ = 0;
    bool busy_ = false;
};

/* ------------------------------------------------------------------ searcher */

struct PlannedQuery {
    uint32_t status = XGM_OK;
    bool on_device = false;   /* false: answered on the host (empty / bounds-only) */
    uint32_t first = 0, maxitems = 0, topk = 0, check_at_least = 0;
    uint32_t tf_min = 0, tf_est = 0, tf_max = 0;
    uint32_t nweighted = 0;   /* weighted subqueries: the denominator of the percentage scale */
    double max_possible = 0;
    uint64_t alg_bytes = 0;
    uint32_t sort_by = 0;
    uint32_t filter = 0;
    bool filter_subq = false; /* the filter counts as a matching subquery of every match */
    double bucket_max = 0;   /* finite bound of the weights, for the pruning buckets (max_possible is DBL_MAX with a weighted source) */
    bool mv_source = false;  /* a Xapiand range source is a child of the base's MultiAndPostList: its termfreqs are restated */
    bool count_only = false; /* first >= every possible match count: the MSet is empty, only counts matter */
    bool aux_subqs = false;  /* the number of matching weighted leaves varies per document (OR, AND_MAYBE) */
    bool log_raises = false; /* … and the MSet is not ordered by weight: subqueries of the best-weighted document come from the raise log */
};

/* A pinned host array and its device copy: the host fills it and one copy uploads it. */
template <class T> struct PinnedPair {
    HostBuf<T> h;
    DevBuf<T> d;
    cudaError_t alloc(size_t n) {
        const cudaError_t e = h.alloc(n);
        return e != cudaSuccess ? e : d.alloc(n);
    }
    xgm_status reserve(size_t need, size_t floor, cudaStream_t st) {
        CUDA_TRY(h.grow(need, floor, st));
        CUDA_TRY(d.grow(need, floor, st));
        return XGM_OK;
    }
    cudaError_t upload(size_t n, cudaStream_t st) const {
        return n ? cudaMemcpyAsync(d.get(), h.get(), n * sizeof(T), cudaMemcpyHostToDevice, st) : cudaSuccess;
    }
};

/* One work list of a batch: a segment per query (per query and leaf on the OR list), which the device expands
 * into work items of at most bpi driver blocks. */
struct WorkList {
    PinnedPair<XgmWorkItem> seg;  /* segments, in the order the expansion reads them */
    PinnedPair<uint32_t> levels;  /* level starts of a level-ordered expansion */
    DevBuf<XgmWorkItem> d_exp;    /* expanded + interleaved work items (device only) */
    uint32_t nseg = 0, nstarts = 0, nitems = 0; /* nstarts: entries of `levels` in use */
    /* the segments expand to n work items: room for them on the device */
    xgm_status set_items(uint64_t n, cudaStream_t st) {
        if (n >= 0xffffffffull) return fail(XGM_E_INVALID, "too many work items in one batch");
        nitems = (uint32_t)n;
        CUDA_TRY(d_exp.grow(n, 65536, st));
        return XGM_OK;
    }
    /* the segments, `extra` rows stored after them, and the level starts */
    cudaError_t upload(uint32_t extra, cudaStream_t st) const {
        cudaError_t e = seg.upload((size_t)nseg + extra, st);
        return e != cudaSuccess ? e : levels.upload(nstarts, st);
    }
};

/* The OR list: one level-ordered expansion per leaf position */
struct OrList : WorkList {
    struct Group { uint32_t seg_off, level_off, nlevels, out_off, total; };
    std::vector<Group> groups;
};

/* The bitmap AND list.  In range-major order its segments are followed by runs of segments that share a driver
 * list, and the device expands it per (range, run). */
struct BmList : WorkList {
    bool range_mode = false;
    uint32_t nranges = 1, nruns = 0;
    DevBuf<uint32_t> d_rng; /* per (range, run) first block, item count, output offset */
    PinnedPair<uint32_t> rng_total; /* [0] = number of items, counted on the device */
};

/* A batch's segments as planned, one vector per work list */
struct PlannedSegments { std::vector<XgmWorkItem> and_list, or_list, bm_list; };

struct xgm_searcher {
    const xgm_index* ix = nullptr;
    int device = 0; /* ix->device, kept so that freeing the searcher never reads an index already closed */
    uint32_t max_batch = 0, max_topk = 0, match_cap = 0;
    Stream stream; /* declared before the buffers and events: destroyed after them */
    Event ev0, ev1, ev2;
    Event ev_in, ev_done; /* hand-over between the copy stream and the shared compute stream */
    /* XGM_TRACE=1: one stderr line per batch with its host and GPU timeline (see trace_line) */
    Event tr_h2d, tr_out;
    std::chrono::steady_clock::time_point tr_submit, tr_planned, tr_launched, tr_async;
    bool shared_compute = true;
    /* pinned host staging */
    PinnedPair<XgmDevQuery> queries;
    HostBuf<double> h_out_w;
    HostBuf<uint32_t> h_out_d;
    HostBuf<uint64_t> h_out_k;
    HostBuf<XgmDevResult> h_info;
    PinnedPair<XgmRaise> raise;  /* raise logs of the batch (copied to the host only when a query asked for them) */
    HostBuf<XgmQState> h_qstate; /* per-query state after the batch (raise-log lengths) */
    bool any_raise = false;
    uint32_t keep_cap = 0;
    size_t ctrl_bytes = 0;
    /* device */
    WorkList and_list; /* general AND kernel */
    OrList or_list;
    BmList bm_list;    /* bitmap AND kernel */
    uint32_t bpi = 16;
    uint32_t range_bits = 16; /* XGM_RANGE_BITS: 2^16 docids per range (DESIGN.md §3.1) */
    DevBuf<uint32_t> d_topk_list; /* [max_batch] queries left to the CTA-per-query top-k kernel */
    DevBuf<unsigned char> d_ctrl; /* [XGM_CTRL_HDR B work counters][nq x XgmQState][nq x XGM_NBINS x u32] */
    DevBuf<double> d_match_w;
    DevBuf<uint32_t> d_match_d;
    DevBuf<uint64_t> d_match_k;
    DevBuf<double> d_pool_w;
    DevBuf<uint32_t> d_pool_d;
    DevBuf<uint64_t> d_pool_k;
    uint32_t pool_total = 0;
    double* d_out_w = nullptr;
    uint32_t* d_out_d = nullptr;
    uint64_t* d_out_k = nullptr;
    XgmDevResult* d_info = nullptr;
    DevBuf<unsigned char> d_slab; /* d_out_w | d_out_d | d_info | d_out_k in one allocation: one all-gather moves a shard's MSets */
    size_t slab_bytes = 0, slab_off_d = 0, slab_off_info = 0, slab_off_k = 0;
    /* last batch */
    std::vector<PlannedQuery> plan;
    uint32_t nq = 0;
    bool pending = false, any_sort = false;
    xgm_batch_stats stats{};
    XgmGrids grids{};
    bool any_or_fast = false, any_or_slow = false;
    PinnedPair<uint32_t> tileq;   /* queries of the batch answered by the bitmap-union kernel */
    uint32_t ntileq = 0;
    bool device_only = false;     /* results stay on the device (xgm_searcher_set_results_on_device) */
    uint32_t bpi_override = 0;    /* XGM_BPI: driver blocks per work item for batches >= 256 (default 16) */
    bool or_tile = true;          /* XGM_OR_TILE=0: keep every fast OR query in the one-launch kernel */
    bool or_general = false;      /* XGM_OR_KERNEL=1: every OR query on the general xgm_or_kernel */
    XgmKernelParams params;
    /* xgm_search_submit_async: a worker thread plans and enqueues the batch while the caller scatters the
     * results of an earlier one */
    std::thread worker;
    std::mutex mu;
    std::condition_variable cv;
    enum { JOB_NONE = 0, JOB_QUEUED, JOB_RUNNING, JOB_DONE } job = JOB_NONE;
    bool worker_exit = false;
    const xgm_query* job_queries = nullptr;
    uint32_t job_nq = 0;
    xgm_status job_status = XGM_OK;
    char job_err[512] = "";
};

/* Block until the worker (if any) has planned and enqueued the batch handed to xgm_search_submit_async;
 * its status and error text become the caller's. */
static xgm_status join_async(xgm_searcher* s) {
    std::unique_lock<std::mutex> lk(s->mu);
    if (s->job == xgm_searcher::JOB_NONE) return XGM_OK;
    s->cv.wait(lk, [&] { return s->job == xgm_searcher::JOB_DONE; });
    s->job = xgm_searcher::JOB_NONE;
    if (s->job_status != XGM_OK) {
        s->pending = false;
        return fail(s->job_status, "%s", s->job_err);
    }
    return XGM_OK;
}

extern "C" void xgm_searcher_free(xgm_searcher* s) {
    if (!s) return;
    if (s->worker.joinable()) {
        {
            std::unique_lock<std::mutex> lk(s->mu);
            s->cv.wait(lk, [&] { return s->job == xgm_searcher::JOB_NONE || s->job == xgm_searcher::JOB_DONE; });
            s->worker_exit = true;
        }
        s->cv.notify_all();
        s->worker.join();
    }
    cudaSetDevice(s->device); /* the members free on the searcher's device */
    if (s->stream.get()) cudaStreamSynchronize(s->stream.get());
    delete s;
}

extern "C" xgm_status xgm_searcher_new(const xgm_index* ix, uint32_t max_batch, uint32_t max_topk, xgm_searcher** out) {
    if (!ix || !out || max_batch == 0 || max_topk == 0) return fail(XGM_E_INVALID, "bad arguments");
    if (max_topk > XGM_MAX_TOPK) return fail(XGM_E_INVALID, "max_topk %u > %u", max_topk, XGM_MAX_TOPK);
    if (max_batch >= (1u << 25)) return fail(XGM_E_INVALID, "max_batch %u too large", max_batch);
    CUDA_TRY(cudaSetDevice(ix->device));
    std::unique_ptr<xgm_searcher, void (*)(xgm_searcher*)> s(new xgm_searcher(), xgm_searcher_free);
    s->ix = ix; s->device = ix->device; s->max_batch = max_batch; s->max_topk = max_topk;
    /* candidates a query may buffer before its pruning threshold settles (~k(1+ln(M/k)) arrive above
     * a rising threshold) and how many of them the top-k kernel can hold in shared memory */
    s->match_cap = std::min<uint32_t>(65536, std::max<uint32_t>(XGM_KEEP_CAP_MAX, 32 * max_topk));
    s->keep_cap = 2048; /* a power of two (the top-k kernel sorts in place): 2048, 4096 or XGM_KEEP_CAP_MAX */
    while (s->keep_cap < XGM_KEEP_CAP_MAX && s->keep_cap < 8 * max_topk) s->keep_cap <<= 1;
    CUDA_TRY(s->stream.create(cudaStreamNonBlocking));
    CUDA_TRY(s->ev0.create(cudaEventDefault)); CUDA_TRY(s->ev1.create(cudaEventDefault)); CUDA_TRY(s->ev2.create(cudaEventDefault));
    CUDA_TRY(s->ev_in.create(cudaEventDisableTiming));
    CUDA_TRY(s->ev_done.create(cudaEventDisableTiming));
    if (g_trace) {
        CUDA_TRY(s->tr_h2d.create(cudaEventDefault)); CUDA_TRY(s->tr_out.create(cudaEventDefault));
        if (!g_tr_base) {
            CUDA_TRY(cudaEventCreate(&g_tr_base));
            CUDA_TRY(cudaEventRecord(g_tr_base, s->stream.get()));
            CUDA_TRY(cudaEventSynchronize(g_tr_base));
            g_tr_t0 = std::chrono::steady_clock::now();
        }
    }
    if (const char* e = getenv("XGM_SHARED_COMPUTE")) s->shared_compute = atoi(e) != 0;
    if (const char* e = getenv("XGM_RANGE_BITS")) s->range_bits = (uint32_t)std::min(31, std::max(0, atoi(e)));
    CUDA_TRY(s->bm_list.rng_total.alloc(16));
    CUDA_TRY(cudaMemset(s->bm_list.rng_total.d.get(), 0, 64));
    s->bm_list.rng_total.h.get()[0] = 0;
    {
        std::lock_guard<std::mutex> lk(ix->launch_mu);
        if (!ix->compute_stream.get()) CUDA_TRY(ix->compute_stream.create(cudaStreamNonBlocking));
    }
    size_t nq = max_batch, ns = (size_t)max_batch * max_topk, nm = (size_t)max_batch * s->match_cap;
    CUDA_TRY(s->queries.alloc(nq));
    CUDA_TRY(s->h_out_w.alloc(ns)); CUDA_TRY(s->h_out_d.alloc(ns));
    CUDA_TRY(s->h_out_k.alloc(ns)); CUDA_TRY(s->h_info.alloc(nq));
    CUDA_TRY(s->raise.alloc(nq * XGM_RAISE_LOG));
    CUDA_TRY(s->h_qstate.alloc(nq));
    CUDA_TRY(s->tileq.alloc(nq));
    if (const char* e = getenv("XGM_OR_TILE")) s->or_tile = atoi(e) != 0;
    if (const char* e = getenv("XGM_OR_KERNEL")) s->or_general = atoi(e) == 1;
    if (const char* e = getenv("XGM_BPI")) s->bpi_override = (uint32_t)std::min(32, std::max(0, atoi(e)));
    s->ctrl_bytes = XGM_CTRL_HDR + nq * sizeof(XgmQState) + nq * XGM_NBINS * 4;
    CUDA_TRY(s->d_ctrl.alloc(s->ctrl_bytes));
    CUDA_TRY(s->d_topk_list.alloc(nq));
    CUDA_TRY(s->d_match_w.alloc(nm)); CUDA_TRY(s->d_match_d.alloc(nm)); CUDA_TRY(s->d_match_k.alloc(nm));
    {
        auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
        s->slab_off_d = up(ns * 8);
        s->slab_off_info = s->slab_off_d + up(ns * 4);
        s->slab_off_k = s->slab_off_info + up(nq * sizeof(XgmDevResult));
        s->slab_bytes = s->slab_off_k + up(ns * 8);
        CUDA_TRY(s->d_slab.alloc(s->slab_bytes));
        s->d_out_w = reinterpret_cast<double*>(s->d_slab.get());
        s->d_out_d = reinterpret_cast<uint32_t*>(s->d_slab.get() + s->slab_off_d);
        s->d_info = reinterpret_cast<XgmDevResult*>(s->d_slab.get() + s->slab_off_info);
        s->d_out_k = reinterpret_cast<uint64_t*>(s->d_slab.get() + s->slab_off_k);
    }
    /* overflow pool: room for the tie mass of a few pathological queries per batch (doccount entries at least) */
    s->pool_total = std::max<uint32_t>(1u << 20, std::min<uint32_t>(1u << 25, 2 * ix->doccount + (1u << 16)));
    if (const char* e = getenv("XGM_POOL_ENTRIES")) s->pool_total = (uint32_t)strtoul(e, nullptr, 10);
    CUDA_TRY(s->d_pool_w.alloc(s->pool_total)); CUDA_TRY(s->d_pool_d.alloc(s->pool_total));
    CUDA_TRY(s->d_pool_k.alloc(s->pool_total));
    xgm_status st = s->and_list.seg.reserve(4096, 4096, s->stream.get());
    if (st == XGM_OK) st = s->or_list.seg.reserve(4096, 4096, s->stream.get());
    if (st == XGM_OK) st = s->bm_list.seg.reserve(4096, 4096, s->stream.get());
    if (st != XGM_OK) return st;
    CUDA_TRY(xgm_kernel_grids(ix->sm_count, s->keep_cap, s->grids));
    *out = s.release();
    return XGM_OK;
}

extern "C" void* xgm_searcher_stream(xgm_searcher* s) { return s ? (void*)s->stream.get() : nullptr; }

/* ComparePostListTermFreqAscending on (tf, original index) — same std::partial_sort_copy call as
 * MultiAndPostList's constructor (multiandpostlist.h:126-131) so ties land identically (libstdc++). */
struct TfIdx { uint32_t tf, idx; };
static inline bool tf_less(const TfIdx& a, const TfIdx& c) { return a.tf < c.tf; }

/* Heap::make/pop/replace of src/xapian/common/heap.h (libc++-style sift-down) replayed on
 * (termfreq, node) pairs exactly as OrContext::postlist does (queryinternal.cc:440-489). */
struct OrEnt { uint32_t tf; int node; };
static inline bool or_cmp(const OrEnt& a, const OrEnt& b) { return a.tf > b.tf; }
static void or_sift_down(OrEnt* first, long len, long start) {
    long child = start;
    if (len < 2 || (len - 2) / 2 < child) return;
    child = 2 * child + 1;
    if (child + 1 < len && or_cmp(first[child], first[child + 1])) ++child;
    if (or_cmp(first[child], first[start])) return;
    OrEnt top = first[start];
    do {
        first[start] = first[child];
        start = child;
        if ((len - 2) / 2 < child) break;
        child = 2 * child + 1;
        if (child + 1 < len && or_cmp(first[child], first[child + 1])) ++child;
    } while (!or_cmp(first[child], top));
    first[start] = top;
}

struct OrTree { int lch[2 * XGM_MAX_TERMS], rch[2 * XGM_MAX_TERMS]; int root; };

static void build_or_tree(const uint32_t* tf, uint32_t n, OrTree& tr) {
    OrEnt h[XGM_MAX_TERMS];
    for (uint32_t i = 0; i < n; ++i) { h[i].tf = tf[i]; h[i].node = (int)i; }
    long len = n;
    for (long s = (len - 2) / 2; s >= 0; --s) or_sift_down(h, len, s);
    int next = (int)n;
    for (;;) {
        int r = h[0].node;
        uint32_t rtf = h[0].tf;
        std::swap(h[0], h[len - 1]);
        or_sift_down(h, len - 1, 0);
        --len;
        int node = next++;
        tr.lch[node] = h[0].node;
        tr.rch[node] = r;
        if (len == 1) { tr.root = node; break; }
        h[0].node = node;
        h[0].tf += rtf;
        or_sift_down(h, len, 0);
    }
}

/* Termfreq (min, max, estimate) of a PostList */
struct TfNode { uint32_t mn, mx, est; };

/* MultiAndPostList::get_termfreq_{min,max,est} (matcher/multiandpostlist.cc:55-105) over the children ch[0 .. n) in
 * the order given: the wrapping sum of the minimums, the least maximum and the scaled product of the estimates */
static TfNode and_node(const TfNode* ch, uint32_t n, uint32_t doccount) {
    uint32_t sum = ch[0].mn;
    if (sum) {
        for (uint32_t i = 1; i < n; ++i) {
            const uint32_t old = sum;
            sum += ch[i].mn;
            if (sum >= old && sum <= doccount) { sum = 0; break; }
            sum -= doccount;
        }
    }
    const double dbsize = doccount;
    uint32_t mx = ch[0].mx;
    double r = ch[0].est;
    for (uint32_t i = 1; i < n; ++i) {
        mx = std::min(mx, ch[i].mx);
        r = (r * ch[i].est) / dbsize;
    }
    return TfNode{sum, mx, doccount ? (uint32_t)(r + 0.5) : 0};
}

static void or_postfix(const OrTree& tr, int x, uint32_t n, const uint32_t* label, XgmDevQuery& dq) {
    if (x < (int)n) { dq.prog[dq.prog_len++] = (int8_t)(label ? label[x] : (uint32_t)x); return; }
    or_postfix(tr, tr.lch[x], n, label, dq);
    or_postfix(tr, tr.rch[x], n, label, dq);
    dq.prog[dq.prog_len++] = -1;
}

/* The OrContext::postlist tree over leaves with termfreqs tf[0 .. n) and max weights w[] (none: 0), folded
 * bottom-up: termfreqs by OrPostList::get_termfreq_min/max/est (matcher/orpostlist.cc:80-83,353-384), max weight
 * left + right (OrPostList::recalc_maxweight, orpostlist.cc:105-111).  With dq, the tree also becomes dq->prog,
 * the device's postfix program: left subtree, right subtree, -1, with leaf i written as label[i] (i without labels). */
struct OrFold { TfNode tf; double maxw; };
static OrFold or_fold(const uint32_t* tf, const double* w, uint32_t n, uint32_t doccount,
                      const uint32_t* label = nullptr, XgmDevQuery* dq = nullptr) {
    OrTree tr;
    tr.root = 0; /* a single leaf is the whole tree */
    if (n > 1) build_or_tree(tf, n, tr);
    OrFold v[2 * XGM_MAX_TERMS];
    for (uint32_t i = 0; i < n; ++i) v[i] = OrFold{TfNode{tf[i], tf[i], tf[i]}, w ? w[i] : 0.0};
    const double dbsize = doccount;
    for (int x = (int)n; x <= tr.root; ++x) { /* internal nodes are created children-first */
        const OrFold l = v[tr.lch[x]], r = v[tr.rch[x]];
        uint32_t mx = l.tf.mx + r.tf.mx;
        if (mx > doccount || mx < l.tf.mx) mx = doccount;
        const double a = l.tf.est, b = r.tf.est;
        const uint32_t est = dbsize == 0.0 ? 0 : (uint32_t)(a + b - (a * b / dbsize) + 0.5);
        v[x] = OrFold{TfNode{std::max(l.tf.mn, r.tf.mn), mx, est}, l.maxw + r.maxw};
    }
    if (dq) {
        dq->prog_len = 0;
        or_postfix(tr, tr.root, n, label, *dq);
    }
    return v[tr.root];
}

/* BM25Weight::init (bm25weight.cc:46-130) via Weight::init_ (weight.cc:59-83); host-side because it
 * needs log() and runs once per term per query. */
static double bm25_termweight(uint32_t N, uint32_t tf, uint32_t wqf, double factor, double k1, double k3) {
    double tw = ((double)(N - tf) + 0.5) / ((double)tf + 0.5);
    if (tw < 2) tw = tw * 0.5 + 1;
    double w = std::log(tw) * factor;
    if (k3 != 0) {
        double wqf_double = wqf;
        w *= (k3 + 1) * wqf_double / (k3 + wqf_double);
    }
    w *= (k1 + 1);
    return w;
}

/* BM25Weight::get_maxpart bm25weight.cc:183-207 */
static double bm25_maxpart(double termweight, double len_factor, double k1, double b, double min_normlen,
                           uint32_t wdf_ub, uint32_t doclen_lb) {
    double denom = k1;
    if (k1 != 0.0 && b != 0.0) {
        uint32_t m = std::max(wdf_ub, doclen_lb);
        double normlen_lb = std::max(m * len_factor, min_normlen);
        denom *= (normlen_lb * b + (1 - b));
    }
    double wdf_max = wdf_ub;
    denom += wdf_max;
    return termweight * (wdf_max / denom);
}

/* A query's leaves as the planner sees them: the nterms base terms, then the FILTER, AND_NOT and AND_MAYBE groups */
struct PlanTerms {
    uint32_t n, nfilter, nnot, nmaybe, ngroups;
    uint32_t ids[XGM_MAX_TERMS]; /* 0xffffffffu: not in this index */
    uint32_t ltf[XGM_MAX_TERMS]; /* termfreq in this index (0 if absent) */
    /* BM25 parameters and the base terms' weights */
    uint32_t N;
    double k1, k3, b, mnl, len_factor;
    double tw[XGM_MAX_TERMS], maxpart[XGM_MAX_TERMS];
    uint32_t nweighted; /* base terms with a nonzero factor */
};

/* Checks the query's shape and arguments and looks up its leaves.  Anything but XGM_OK declines the query. */
static xgm_status resolve_terms(const xgm_index* ix, const xgm_query& q, PlanTerms& t) {
    if (q.nterms == 0 || q.nterms > XGM_MAX_TERMS) return XGM_E_UNIMPLEMENTED;
    if (q.op != XGM_OP_AND && q.op != XGM_OP_OR) return XGM_E_UNIMPLEMENTED;
    const bool groups = q.nfilter || q.nnot || q.nmaybe;
    if (groups) {
        /* OP_FILTER with boolean terms / OP_AND_NOT / OP_AND_MAYBE around an AND (or single-term) base, the first
         * two also around an OR base; optional leaves on an OR base or a value-range filter on top are left to the
         * reference */
        const bool or_base = q.op == XGM_OP_OR && q.nterms != 1;
        if ((or_base && q.nmaybe) || q.filter != XGM_FILTER_NONE ||
            (uint64_t)q.nterms + q.nfilter + q.nnot + q.nmaybe > XGM_MAX_TERMS)
            return XGM_E_UNIMPLEMENTED;
    }
    if (q.sort_by > XGM_SORT_REL_VAL || q.filter > XGM_FILTER_MULTI_RANGE) return XGM_E_INVALID;
    if ((q.filter && q.filter_slot >= XGM_MAX_SLOTS) || (q.sort_by && q.sort_slot >= XGM_MAX_SLOTS)) return XGM_E_INVALID;
    if (q.revision != 0 && q.revision != ix->revision) return XGM_E_STALE;
    if ((q.filter && !ix->slot_exact[q.filter_slot] && ix->d_voff[q.filter_slot].get()) ||
        (q.sort_by && !ix->slot_exact[q.sort_slot] && ix->d_voff[q.sort_slot].get()))
        return XGM_E_UNIMPLEMENTED; /* values longer than 8 bytes: their keys do not decide the comparison */
    /* a weighted range source: a child of the AND (or of a single term) without groups, with a factor >= 0 */
    if (q.filter_weighted && (q.filter != XGM_FILTER_MULTI_RANGE || (q.op != XGM_OP_AND && q.nterms != 1) || groups ||
                              q.filter_factor < 0.0))
        return XGM_E_UNIMPLEMENTED;
    t.n = q.nterms; t.nfilter = q.nfilter; t.nnot = q.nnot; t.nmaybe = q.nmaybe;
    t.ngroups = q.nfilter + q.nnot + q.nmaybe;
    for (uint32_t j = 0; j < t.n + t.ngroups; ++j) {
        uint32_t id = 0xffffffffu;
        if (q.term_ids) id = q.term_ids[j];
        else if (q.terms && q.terms[j]) {
            uint32_t len = q.term_lens ? q.term_lens[j] : (uint32_t)strlen(q.terms[j]);
            if (!lookup_term(ix, q.terms[j], len, &id)) id = 0xffffffffu;
        } else return XGM_E_INVALID;
        if (id != 0xffffffffu && id >= ix->terms.size()) return XGM_E_INVALID;
        for (uint32_t i = 0; i < j; ++i)
            if (t.ids[i] == id && id != 0xffffffffu) return XGM_E_UNIMPLEMENTED; /* repeated leaf */
        t.ids[j] = id;
        t.ltf[j] = id == 0xffffffffu ? 0 : ix->terms[id].termfreq;
    }
    return XGM_OK;
}

/* Weight::init_ of leaf j: its BM25 termweight and maxpart */
static void term_weight(const xgm_index* ix, const xgm_query& q, const PlanTerms& t, uint32_t j, double factor,
                        double& tw, double& maxpart) {
    const uint32_t gtf = q.stats ? q.stats->termfreq[j] : t.ltf[j];
    tw = bm25_termweight(t.N, gtf, q.wqf ? q.wqf[j] : 1, factor, t.k1, t.k3);
    const uint32_t wub = t.ids[j] == 0xffffffffu ? 0 : ix->terms[t.ids[j]].wdf_ub;
    maxpart = bm25_maxpart(tw, t.len_factor, t.k1, t.b, t.mnl, wub, ix->doclen_lb);
}

/* The BM25 parameters and the base terms' weights.  A negative factor, or a zero one in an OR of several leaves,
 * declines the query. */
static xgm_status weigh_terms(const xgm_index* ix, const xgm_query& q, PlanTerms& t) {
    t.k1 = q.k1; t.k3 = q.k3; t.b = q.b; t.mnl = q.min_normlen;
    if (t.k1 == 0 && t.k3 == 0 && t.b == 0 && t.mnl == 0) { t.k1 = 1; t.k3 = 1; t.b = 0.5; t.mnl = 0.5; }
    /* BM25Weight's constructor (weight.h:639-646): k1, k3 < 0 become 0 and b is clamped to [0, 1], so a caller's
     * out-of-range value weighs as the reference weighs it.  The MaxScore bounds rely on it too: outside that range
     * the length term k1 * (normlen * b + 1 - b) can be negative and a posting can outweigh get_maxpart. */
    t.k1 = std::max(t.k1, 0.0); t.k3 = std::max(t.k3, 0.0); t.b = std::min(std::max(t.b, 0.0), 1.0);
    t.N = q.stats ? q.stats->collection_size : ix->doccount;
    const uint64_t tl = q.stats ? q.stats->total_length : ix->total_length;
    t.len_factor = 0;
    if (!(t.b == 0 || t.k1 == 0)) {
        double avg = t.N == 0 ? 0.0 : (double)tl / t.N;
        t.len_factor = avg != 0 ? 1 / avg : 0;
    }
    t.nweighted = 0;
    for (uint32_t j = 0; j < t.n; ++j) {
        const double factor = q.factors ? q.factors[j] : 1.0;
        if (factor < 0.0 || (factor == 0.0 && q.op == XGM_OP_OR && t.n > 1)) return XGM_E_UNIMPLEMENTED;
        term_weight(ix, q, t, j, factor, t.tw[j], t.maxpart[j]);
        if (factor == 0.0) { t.tw[j] = 0.0; t.maxpart[j] = 0.0; } /* no Weight object: not a counted subquery */
        else ++t.nweighted;
    }
    return XGM_OK;
}

/* Device slot of leaf `id` (0xffffffffu: not in this index) with its weight pair.  A boolean leaf has (0.0, 0.0); the
 * AND kernels skip it altogether (XgmDevQuery::unweighted). */
static void put_term(const xgm_index* ix, XgmDevTerm& d, uint32_t id, double termweight, double maxpart) {
    d.termweight = termweight;
    d.maxpart = maxpart;
    d.bm_off = XGM_NO_BITMAP; d.rk_off = 0;
    d.blk_begin = 0; d.nblocks = 0;
    if (id != 0xffffffffu) {
        const TermInfo& tinf = ix->terms[id];
        d.blk_begin = tinf.blk_begin; d.nblocks = tinf.nblocks;
        d.bm_off = tinf.bm_off; d.rk_off = tinf.rk_off;
    }
}

/* The AND_NOT terms from slot on, as boolean leaves: only those in this index (the others exclude nothing).
 * Returns the next free slot. */
static uint32_t put_excluded(const xgm_index* ix, const PlanTerms& t, XgmDevQuery& dq, uint32_t slot) {
    const uint32_t nb = t.n + t.nfilter;
    for (uint32_t j = nb; j < nb + t.nnot; ++j)
        if (t.ltf[j] != 0) { put_term(ix, dq.terms[slot++], t.ids[j], 0.0, 0.0); ++dq.nnot; }
    return slot;
}

/* Termfreq bounds of the groups around a base with bounds cur: MultiAnd(base, AND of the FILTER terms), then
 * AndNot(…, OR of the AND_NOT terms).  AND_MAYBE keeps its left side's. */
static TfNode group_bounds(const xgm_index* ix, const PlanTerms& t, TfNode cur) {
    const uint32_t doccount = ix->doccount;
    if (t.nfilter) {
        /* QueryFilter::postlist: MultiAndPostList of [base, Query(OP_AND, boolean terms)] */
        const uint32_t* ftf = t.ltf + t.n;
        TfNode f{ftf[0], ftf[0], ftf[0]};
        if (t.nfilter > 1) {
            TfNode fin[XGM_MAX_TERMS], fo[XGM_MAX_TERMS];
            for (uint32_t j = 0; j < t.nfilter; ++j) fin[j] = TfNode{ftf[j], ftf[j], ftf[j]};
            std::partial_sort_copy(fin, fin + t.nfilter, fo, fo + t.nfilter,
                                   [](const TfNode& a, const TfNode& c) { return a.est < c.est; });
            f = and_node(fo, t.nfilter, doccount);
        }
        /* the pair by ascending estimate, the base first on a tie */
        const TfNode ch[2] = {f.est < cur.est ? f : cur, f.est < cur.est ? cur : f};
        cur = and_node(ch, 2, doccount);
    }
    if (t.nnot) {
        /* AndNotPostList::get_termfreq_min/max/est, matcher/andnotpostlist.cc:30-62 */
        const TfNode rr = or_fold(t.ltf + t.n + t.nfilter, nullptr, t.nnot, doccount).tf;
        const TfNode a = cur;
        cur.mn = a.mn <= rr.mx ? 0 : a.mn - rr.mx;
        cur.mx = std::min(doccount - rr.mn, a.mx);
        if (doccount == 0) cur.est = 0;
        else {
            double e = a.est;
            e = (e * (double)(doccount - rr.est)) / (double)doccount;
            cur.est = (uint32_t)(e + 0.5);
        }
    }
    return cur;
}

/* Largest expected share of driver postings whose coarse bit in terms[1] is set, 1 - (1 - tf / lastdocid)^8, for
 * which the bitmap AND kernel tests the coarse bit first (DESIGN.md §6: chosen by measurement on C2 and C5). */
#define XGM_COARSE_PASS_MAX 0.1

/* The range of OP_FILTER(base, range) as a MultiAndPostList child.  The source of a Xapiand range
 * (MultipleValueRange) has termfreqs (min, est, max) = (0, value_freq, value_freq) (range.cc:457-464,
 * api/postingsource.cc:201-214).  A stock OP_VALUE_RANGE has max = value_freq and min = value_freq when the range
 * covers the slot's value bounds, 0 otherwise (valuerangepostlist.cc:40-54,145-148); its string-fraction estimate
 * (valuerangepostlist.cc:70-130) is not restated: value_freq stands in for it and finish_info flags the bounds. */
static bool stock_range_covers_slot(const xgm_index* ix, const xgm_query& q) {
    const uint32_t s = q.filter_slot;
    return q.filter == XGM_FILTER_VALUE_RANGE && ix->slot_freq[s] != 0 && q.range_lo <= ix->slot_first_min[s] &&
           ix->slot_first_max[s] <= q.range_hi;
}

static TfNode range_child(const xgm_index* ix, const xgm_query& q) {
    const uint32_t vf = ix->slot_freq[q.filter_slot];
    return TfNode{stock_range_covers_slot(ix, q) ? vf : 0u, vf, vf};
}

/* An AND base: one MultiAndPostList over the base terms and, for a value range, the range; the FILTER terms join
 * the required lists as boolean leaves, then the AND_NOT and AND_MAYBE terms follow. */
static void plan_and_route(const xgm_index* ix, const xgm_query& q, const PlanTerms& t, PlannedQuery& pq,
                           XgmDevQuery& dq) {
    const uint32_t n = t.n;
    /* the range takes part in the MultiAndPostList like a term (a weighted one only as a Xapiand range's source) */
    const bool has_range = q.filter != XGM_FILTER_NONE;
    const bool mv_source = q.filter == XGM_FILTER_MULTI_RANGE;
    const bool src_weighted = mv_source && q.filter_weighted;
    const double src_w = src_weighted ? (q.filter_factor != 0.0 ? q.filter_factor : 1.0) : 0.0;
    /* its children sorted by get_termfreq_est with the very call of multiandpostlist.h:126-131 */
    const uint32_t nch = n + (has_range ? 1u : 0u);
    const TfNode src = has_range ? range_child(ix, q) : TfNode{0, 0, 0};
    TfIdx in[XGM_MAX_TERMS + 1], outv[XGM_MAX_TERMS + 1];
    for (uint32_t j = 0; j < n; ++j) in[j] = TfIdx{t.ltf[j], j};
    if (has_range) in[n] = TfIdx{src.est, n};
    std::partial_sort_copy(in, in + nch, outv, outv + nch, tf_less);
    /* MultiAndPostList::recalc_maxweight (multiandpostlist.cc:167-177) and termfreqs over the children in that
     * order: base term order[i], or the source at src_pos */
    uint32_t order[XGM_MAX_TERMS], src_pos = XGM_NO_SRC, k = 0;
    TfNode ch[XGM_MAX_TERMS + 1];
    double mp = 0, mp_real = 0;
    for (uint32_t c = 0; c < nch; ++c) {
        const uint32_t j = outv[c].idx;
        if (j == n) {
            src_pos = k;
            ch[c] = src;
            mp += src_weighted ? src_w * DBL_MAX : 0.0;
            mp_real += src_w;
        } else {
            order[k++] = j;
            ch[c] = TfNode{t.ltf[j], t.ltf[j], t.ltf[j]};
            mp += t.maxpart[j];
            mp_real += t.maxpart[j];
        }
    }
    pq.max_possible = nch == 1 ? t.maxpart[0] : mp;
    pq.bucket_max = nch == 1 ? t.maxpart[0] : mp_real;
    const TfNode cur = group_bounds(ix, t, and_node(ch, nch, ix->doccount));
    pq.tf_min = cur.mn; pq.tf_max = cur.mx; pq.tf_est = cur.est;
    pq.mv_source = mv_source;
    if (src_weighted) { dq.src_pos = src_pos; dq.src_weight = src_w; }
    dq.route = XGM_ROUTE_AND;
    dq.nterms = n + t.nfilter;
    /* required lists: the base (its own MultiAndPostList order, which fixes the order of the weight sum) merged with
     * the boolean filter terms by ascending termfreq */
    TfIdx fin[XGM_MAX_TERMS];
    for (uint32_t j = 0; j < t.nfilter; ++j) fin[j] = TfIdx{t.ltf[n + j], n + j};
    std::stable_sort(fin, fin + t.nfilter, tf_less);
    uint32_t slot = 0, bi = 0, fi = 0, tf1 = 0;
    while (bi < n || fi < t.nfilter) {
        const bool base = fi >= t.nfilter || (bi < n && t.ltf[order[bi]] <= fin[fi].tf);
        const uint32_t j = base ? order[bi++] : fin[fi++].idx;
        if (slot == 1) tf1 = t.ltf[j];
        if (!base || (q.factors && q.factors[j] == 0.0)) dq.unweighted |= 1u << slot;
        put_term(ix, dq.terms[slot++], t.ids[j], base ? t.tw[j] : 0.0, base ? t.maxpart[j] : 0.0);
    }
    /* The bitmap AND kernel probes terms[1] for every driver posting.  Where a coarse bit (8 docids) is rarely set,
     * testing it first leaves few fine-word loads; where it is mostly set, the second load only adds latency. */
    if (dq.nterms >= 2 && ix->lastdocid != 0) {
        const double pass = 1.0 - std::pow(1.0 - std::min(1.0, (double)tf1 / ix->lastdocid), 8.0);
        dq.probe_coarse = pass <= XGM_COARSE_PASS_MAX ? 1u : 0u;
    }
    slot = put_excluded(ix, t, dq, slot);
    if (t.nmaybe) {
        /* AndMaybePostList: termfreqs are the left's; recalc_maxweight = pl_max + r_max where r is the
         * OrContext tree over the optional leaves (matcher/andmaybepostlist.cc:69-75); prog names them in
         * query order */
        const uint32_t mb = n + t.nfilter + t.nnot;
        double mtw[XGM_MAX_TERMS], mmax[XGM_MAX_TERMS];
        for (uint32_t j = 0; j < t.nmaybe; ++j) term_weight(ix, q, t, mb + j, 1.0, mtw[j], mmax[j]);
        pq.max_possible = pq.max_possible + or_fold(t.ltf + mb, mmax, t.nmaybe, ix->doccount, nullptr, &dq).maxw;
        pq.bucket_max = pq.max_possible;
        for (uint32_t j = 0; j < t.nmaybe; ++j) put_term(ix, dq.terms[slot++], t.ids[mb + j], mtw[j], mmax[j]);
        dq.nmaybe = t.nmaybe;
        pq.aux_subqs = true;
    }
    /* weighted subqueries, for the percentage scale (a weighted source excludes groups) */
    pq.nweighted = t.nweighted + (src_weighted ? 1u : 0u) + t.nmaybe;
}

/* An OR base of several leaves: a Huffman-shaped tree of binary OrPostLists, built from the leaves in query order
 * (OrContext::postlist, queryinternal.cc:440-489).  On the device the leaves are stored in ascending-termfreq order
 * (position = ownership priority); the program refers to positions. */
static void plan_or_route(const xgm_index* ix, const xgm_query& q, const PlanTerms& t, PlannedQuery& pq,
                          XgmDevQuery& dq) {
    const uint32_t n = t.n;
    TfIdx in[XGM_MAX_TERMS];
    for (uint32_t j = 0; j < n; ++j) in[j] = TfIdx{t.ltf[j], j};
    std::stable_sort(in, in + n, tf_less);
    uint32_t posof[XGM_MAX_TERMS];
    for (uint32_t i = 0; i < n; ++i) posof[in[i].idx] = i;
    const OrFold f = or_fold(t.ltf, t.maxpart, n, ix->doccount, posof, &dq);
    /* QueryFilter / QueryAndNot above the OrPostList tree: the filter's boolean terms, a value range and the excluded
     * terms weigh nothing (MultiAndPostList::get_weight adds +0.0, AndNotPostList returns the left's weight), so a
     * match keeps the tree's weight; the counts follow the same bound arithmetic as around an AND base.  A value
     * range comes without groups: QueryFilter::postlist's MultiAndPostList of [tree, range] (queryinternal.cc:
     * 2271-2283), its two children by ascending estimate. */
    TfNode cur = f.tf;
    if (q.filter != XGM_FILTER_NONE) {
        const TfNode src = range_child(ix, q);
        const TfNode ch[2] = {src.est < cur.est ? src : cur, src.est < cur.est ? cur : src};
        cur = and_node(ch, 2, ix->doccount);
    }
    cur = group_bounds(ix, t, cur);
    pq.tf_min = cur.mn; pq.tf_max = cur.mx; pq.tf_est = cur.est;
    pq.mv_source = q.filter == XGM_FILTER_MULTI_RANGE;
    pq.max_possible = f.maxw;
    pq.bucket_max = pq.max_possible;
    pq.nweighted = t.nweighted; /* every leaf: a zero factor was declined */
    dq.route = XGM_ROUTE_OR;
    dq.nterms = n;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t j = in[i].idx;
        put_term(ix, dq.terms[i], t.ids[j], t.tw[j], t.maxpart[j]);
    }
    /* terms[n .. n + or_nreq) must hold the document, terms[n + or_nreq .. + nnot) must not */
    for (uint32_t j = 0; j < t.nfilter; ++j) put_term(ix, dq.terms[n + j], t.ids[n + j], 0.0, 0.0);
    dq.or_nreq = t.nfilter;
    put_excluded(ix, t, dq, n + t.nfilter);
}

/* Plans query qi of a batch into pq and dq and adds its segments; its outcome is pq.status. */
static void plan_query(xgm_searcher* s, const xgm_query& q, uint32_t qi, PlannedQuery& pq, XgmDevQuery& dq,
                       PlannedSegments& segs) {
    const xgm_index* ix = s->ix;
    pq = PlannedQuery();
    memset(&dq, 0, offsetof(XgmDevQuery, terms)); /* the term slots in use are written in full by put_term */
    PlanTerms t;
    pq.status = resolve_terms(ix, q, t);
    if (pq.status != XGM_OK) return;
    /* Enquire::Internal::get_mset clamping, api/enquire.cc:420-426 */
    uint32_t docs = ix->doccount;
    uint32_t first = std::min(q.first, docs);
    uint32_t maxitems = std::min(q.maxitems, docs - first);
    uint32_t cal = std::min(q.check_at_least, docs);
    cal = std::max(cal, first + maxitems);
    pq.first = first; pq.maxitems = maxitems; pq.topk = first + maxitems; pq.check_at_least = cal;
    pq.sort_by = q.sort_by; pq.filter = q.filter;
    /* a stock range covering every value of a slot that every document has is matched by the all-documents list
     * (QueryValueRange::postlist, queryinternal.cc:1116-1124), an unweighted leaf: no matching subquery */
    pq.filter_subq = q.filter != XGM_FILTER_NONE &&
                     !(stock_range_covers_slot(ix, q) && ix->slot_freq[q.filter_slot] == ix->doccount);
    pq.status = weigh_terms(ix, q, t);
    if (pq.status != XGM_OK) return;

    dq.op = q.op; dq.nweighted = t.nweighted;
    dq.topk = pq.topk; dq.check_at_least = cal;
    dq.len_factor = t.len_factor; dq.k1 = t.k1; dq.b = t.b; dq.one_minus_b = 1 - t.b; dq.min_normlen = t.mnl;
    dq.filter = q.filter; dq.filter_slot = q.filter_slot; dq.range_lo = q.range_lo; dq.range_hi = q.range_hi;
    dq.sort_by = q.sort_by; dq.sort_slot = q.sort_slot; dq.sort_reverse = q.sort_reverse; dq.sort_use_max = q.sort_use_max;
    dq.sort_missing = q.sort_missing_key;
    dq.src_pos = XGM_NO_SRC; dq.src_weight = 0.0;
    if (q.op == XGM_OP_AND || t.n == 1) plan_and_route(ix, q, t, pq, dq);
    else plan_or_route(ix, q, t, pq, dq);

    /* algorithmic bytes, SURVEY.md §8(d): compressed columns + 16 B per block header of every query
     * term (full lists, no credit for skipping) + 16 B per result; 4 B per candidate added at wait() */
    for (uint32_t j = 0; j < t.n + t.ngroups; ++j)
        if (t.ids[j] != 0xffffffffu) pq.alg_bytes += ix->terms[t.ids[j]].bytes;
    pq.alg_bytes += 16ull * pq.topk;

    /* `first` at or beyond the largest possible match count: ProtoMSet never fills (protomset.h:497-505),
     * the MSet is empty and all three bounds equal the exact match count — count on the device only.  Where the
     * number of matching subqueries varies per document, percent_scale_factor still needs that of the first
     * best-weighted document (ProtoMSet saw every match): keep that one document, in relevance order — nothing is
     * returned, so the order asked for does not matter — and read its count as for any relevance-ordered query. */
    if (pq.first >= pq.tf_max && cal != 0) {
        pq.count_only = true;
        const bool varies = dq.route == XGM_ROUTE_OR || pq.aux_subqs;
        dq.topk = varies ? 1u : 0u;
        if (varies) dq.sort_by = XGM_SORT_REL;
    } else if (pq.topk > s->max_topk) { pq.status = XGM_E_INVALID; return; }
    /* pruning buckets: linear in the primary sort key (weight, or the sort value for VAL sorts) */
    if (dq.sort_by == XGM_SORT_REL || dq.sort_by == XGM_SORT_REL_VAL) {
        dq.bucket_scale = pq.bucket_max > 0 ? (double)XGM_NBINS / pq.bucket_max : 0.0;
    } else {
        dq.bucket_key_min = ix->slot_min[q.sort_slot];
        dq.bucket_scale = (double)XGM_NBINS / ((double)(ix->slot_max[q.sort_slot] - ix->slot_min[q.sort_slot]) + 1.0);
    }

    /* percent_scale_factor needs the number of subqueries matching the best-WEIGHTED document: when that varies
     * per document and the order is not by weight alone, have the kernels log the running-maximum matches */
    dq.log_raises = (dq.route == XGM_ROUTE_OR || pq.aux_subqs) && dq.sort_by != XGM_SORT_REL ? 1u : 0u;
    pq.log_raises = dq.log_raises != 0;
    if (cal == 0) return; /* bounds only, matcher.cc:437-461 */
    /* a list every match is in is absent (an AND's terms, the FILTER terms on either base): the MSet is empty */
    for (uint32_t j = dq.route == XGM_ROUTE_AND ? 0 : t.n; j < t.n + t.nfilter; ++j)
        if (t.ltf[j] == 0) return;
    pq.on_device = true;
    /* one segment per (query[, leaf]); the device expands segments into work items (xgm_expand_items_kernel) */
    if (dq.route == XGM_ROUTE_AND) {
        /* every list but the driver has a membership bitmap → lean bitmap kernel */
        bool all_bm = dq.nterms >= 2;
        for (uint32_t i = 1; i < dq.nterms + dq.nnot; ++i) all_bm = all_bm && dq.terms[i].bm_off != XGM_NO_BITMAP;
        std::vector<XgmWorkItem>& dst = all_bm ? segs.bm_list : segs.and_list;
        if (dq.terms[0].nblocks) dst.push_back(XgmWorkItem{qi, dq.terms[0].nblocks, 0, 0});
    } else {
        bool fastor = t.n <= 5 && t.ngroups == 0 && !s->or_general;
        for (uint32_t leaf = 0; leaf < t.n; ++leaf) fastor = fastor && dq.terms[leaf].bm_off != XGM_NO_BITMAP;
        /* relevance order, no predicate, results wanted: multi-leaf documents by bitmap union first */
        const bool tile = s->or_tile && q.filter == XGM_FILTER_NONE && q.sort_by == XGM_SORT_REL && dq.topk != 0;
        dq.or_fast = !fastor ? XGM_OR_FAST_GENERAL : tile ? XGM_OR_FAST_TILE : XGM_OR_FAST_OR3;
        for (uint32_t leaf = 0; leaf < t.n; ++leaf)
            if (dq.terms[leaf].nblocks) segs.or_list.push_back(XgmWorkItem{qi, dq.terms[leaf].nblocks, 0, leaf});
    }
}

/* Level starts of segments sorted by descending length: level k holds the k-th item of every segment that has one,
 * i.e. a prefix of the sorted segments.  Writes the nlev + 1 starts to lv and returns the number of items. */
static uint64_t level_starts(const XgmWorkItem* v, size_t n, uint32_t nlev, uint32_t bpi, uint32_t* lv) {
    uint64_t run = 0;
    size_t alive = n;
    for (uint32_t k = 0; k < nlev; ++k) {
        while (alive > 0 && (v[alive - 1].b0 + bpi - 1) / bpi <= k) --alive;
        lv[k] = (uint32_t)run;
        run += alive;
    }
    lv[nlev] = (uint32_t)run;
    return run;
}

/* Level order: the general AND list, and the bitmap AND list of batches under 256 queries */
static xgm_status order_levels(WorkList& L, std::vector<XgmWorkItem>& v, uint32_t bpi, cudaStream_t st) {
    xgm_status r = L.seg.reserve(v.size(), 4096, st);
    if (r != XGM_OK) return r;
    uint64_t run = 0;
    L.nstarts = 0;
    if (!v.empty()) {
        std::sort(v.begin(), v.end(), [](const XgmWorkItem& a, const XgmWorkItem& b) { return a.b0 > b.b0; });
        const uint32_t maxlev = (v[0].b0 + bpi - 1) / bpi;
        r = L.levels.reserve((size_t)maxlev + 1, 1024, st);
        if (r != XGM_OK) return r;
        run = level_starts(v.data(), v.size(), maxlev, bpi, L.levels.h.get());
        L.nstarts = maxlev + 1;
        std::copy(v.begin(), v.end(), L.seg.h.get());
    }
    L.nseg = (uint32_t)v.size();
    return L.set_items(run, st);
}

/* OR list: leaf-major groups (all queries' rarest leaves first: by the time the frequent, low-weight leaves come up
 * the thresholds have risen and MaxScore skips them wholesale), level order inside each group so that one query's
 * items are spread in time and its threshold settles early */
static xgm_status order_or_groups(OrList& L, std::vector<XgmWorkItem>& v, uint32_t bpi, cudaStream_t st) {
    xgm_status r = L.seg.reserve(v.size(), 4096, st);
    if (r != XGM_OK) return r;
    std::stable_sort(v.begin(), v.end(), [](const XgmWorkItem& a, const XgmWorkItem& b) { return a.pad < b.pad; });
    size_t nstarts = 0;
    for (size_t a = 0; a < v.size();) {
        size_t b = a;
        while (b < v.size() && v[b].pad == v[a].pad) ++b;
        std::sort(v.begin() + a, v.begin() + b, [](const XgmWorkItem& x, const XgmWorkItem& y) { return x.b0 > y.b0; });
        nstarts += (v[a].b0 + bpi - 1) / bpi + 1;
        a = b;
    }
    r = L.levels.reserve(nstarts, 1024, st);
    if (r != XGM_OK) return r;
    L.groups.clear();
    uint64_t run = 0;
    size_t lvpos = 0;
    for (size_t a = 0; a < v.size();) {
        size_t b = a;
        while (b < v.size() && v[b].pad == v[a].pad) ++b;
        OrList::Group g;
        g.seg_off = (uint32_t)a; g.level_off = (uint32_t)lvpos;
        g.nlevels = (v[a].b0 + bpi - 1) / bpi;
        g.out_off = (uint32_t)run;
        const uint64_t n = level_starts(v.data() + a, b - a, g.nlevels, bpi, L.levels.h.get() + lvpos);
        g.total = (uint32_t)n;
        run += n;
        lvpos += (size_t)g.nlevels + 1;
        L.groups.push_back(g);
        a = b;
    }
    std::copy(v.begin(), v.end(), L.seg.h.get());
    L.nseg = (uint32_t)v.size();
    L.nstarts = (uint32_t)lvpos;
    return L.set_items(run, st);
}

/* Range-major order of the bitmap AND list (batches of 256 queries or more), expanded on the device
 * (xgm_range_*_kernel).  Segments sorted by driver list (terms[0]), ties by query index.  Up to XGM_BM_RUN
 * consecutive segments with the same driver form a run, and the run's items serve all of its queries: the AND
 * kernel decodes the driver's blocks once per range and probes them for each query.  The runs follow the segments
 * in the upload as {first segment, #driver blocks, the driver's first header, #queries}.  The host only bounds the
 * number of items: every range can add one partial item per run. */
static xgm_status order_driver_runs(xgm_searcher* s, std::vector<XgmWorkItem>& v, uint32_t bpi) {
    BmList& L = s->bm_list;
    xgm_status r = L.seg.reserve(2 * v.size(), 4096, s->stream.get()); /* segments, then at most as many runs */
    if (r != XGM_OK) return r;
    L.nranges = (s->ix->lastdocid >> s->range_bits) + 1;
    const XgmDevQuery* hq = s->queries.h.get();
    auto drv = [hq](const XgmWorkItem& a) { return hq[a.query].terms[0].blk_begin; };
    std::sort(v.begin(), v.end(), [&](const XgmWorkItem& a, const XgmWorkItem& b) {
        return drv(a) != drv(b) ? drv(a) < drv(b) : a.query < b.query;
    });
    XgmWorkItem* h = L.seg.h.get();
    const size_t nseg = v.size();
    uint64_t run = 0;
    for (size_t i = 0; i < nseg; ++i) {
        h[i] = v[i];
        XgmWorkItem* last = h + nseg + L.nruns - 1;
        if (L.nruns != 0 && last->b1 == drv(v[i]) && last->pad < XGM_BM_RUN) {
            ++last->pad;
            continue;
        }
        h[nseg + L.nruns++] = XgmWorkItem{(uint32_t)i, v[i].b0, drv(v[i]), 1u};
        run += (v[i].b0 + bpi - 1) / bpi;
    }
    /* most work first within each range (queries x driver blocks), so that the batch does not end on a long item */
    std::stable_sort(h + nseg, h + nseg + L.nruns, [](const XgmWorkItem& a, const XgmWorkItem& b) {
        return (uint64_t)a.pad * a.b0 > (uint64_t)b.pad * b.b0;
    });
    run += (uint64_t)L.nruns * L.nranges;
    const size_t need = (size_t)L.nranges * L.nruns * 3; /* first blocks, counts, offsets */
    CUDA_TRY(L.d_rng.grow(need, 0, s->stream.get()));
    L.nseg = (uint32_t)nseg;
    L.nstarts = 0;
    return L.set_items(run, s->stream.get());
}

static cudaError_t expand_levels(const WorkList& L, uint32_t bpi, cudaStream_t cs, uint32_t& launches) {
    if (!L.nitems) return cudaSuccess;
    ++launches;
    return xgm_launch_expand(L.seg.d.get(), L.nitems, L.levels.d.get(), L.nstarts - 1, bpi, L.d_exp.get(), cs);
}

static cudaError_t expand_or_groups(const OrList& L, uint32_t bpi, cudaStream_t cs, uint32_t& launches) {
    for (const auto& g : L.groups) {
        cudaError_t e = xgm_launch_expand(L.seg.d.get() + g.seg_off, g.total, L.levels.d.get() + g.level_off, g.nlevels,
                                          bpi, L.d_exp.get() + g.out_off, cs);
        if (e != cudaSuccess) return e;
        ++launches;
    }
    return cudaSuccess;
}

static cudaError_t expand_driver_runs(const BmList& L, const XgmBlockHdr* hdr, uint32_t range_bits, uint32_t bpi,
                                      cudaStream_t cs, uint32_t& launches) {
    const size_t n = (size_t)L.nranges * L.nruns;
    launches += 3;
    return xgm_launch_expand_ranges(L.seg.d.get() + L.nseg, L.nruns, hdr, L.nranges, range_bits, bpi, L.d_rng.get(),
                                    L.d_rng.get() + n, L.d_rng.get() + 2 * n, L.rng_total.d.get(), L.d_exp.get(), cs);
}

/* The match kernels of one pass (p.pass) over the batch's work lists */
static xgm_status launch_match(xgm_searcher* s, const XgmKernelParams& p, cudaStream_t cs) {
    uint32_t& launches = s->stats.kernel_launches;
    const XgmGrids& g = s->grids;
    if (s->bm_list.nitems) { CUDA_TRY(xgm_launch_and_bm(p, g.and_bm, cs)); ++launches; }
    if (s->and_list.nitems) { CUDA_TRY(xgm_launch_and(p, g.and_, cs)); ++launches; }
    if (s->or_list.nitems && s->any_or_fast) { CUDA_TRY(xgm_launch_or3(p, g.or3, 0, cs)); ++launches; }
    if (s->or_list.nitems && s->any_or_slow) { CUDA_TRY(xgm_launch_or(p, g.or_, cs)); ++launches; }
    if (s->ntileq) { /* documents with >= 2 leaves by bitmap union, then the single-leaf ones against the threshold */
        CUDA_TRY(xgm_launch_or_tile(p, g.or_tile, cs));
        CUDA_TRY(xgm_launch_or3(p, g.or3, 1, cs));
        launches += 2;
    }
    return XGM_OK;
}

static xgm_status launch_batch(xgm_searcher* s) {
    XgmKernelParams& p = s->params;
    /* batches that fill the GPU on their own run their kernels on the index's FIFO compute stream; small
     * ones (concurrent single queries of many host threads) stay on the searcher's stream and share the SMs */
    const bool shared = s->shared_compute && s->nq >= 256;
    cudaStream_t cs = shared ? s->ix->compute_stream.get() : s->stream.get();
    std::unique_lock<std::mutex> lk(s->ix->launch_mu, std::defer_lock);
    if (shared) {
        CUDA_TRY(cudaEventRecord(s->ev_in.get(), s->stream.get()));
        lk.lock(); /* one batch's launches stay contiguous in the shared stream */
        CUDA_TRY(cudaStreamWaitEvent(cs, s->ev_in.get(), 0));
    }
    CUDA_TRY(cudaMemsetAsync(s->d_ctrl.get(), 0, XGM_CTRL_HDR + (size_t)s->max_batch * sizeof(XgmQState), cs));
    CUDA_TRY(cudaMemsetAsync(p.hist, 0, (size_t)s->nq * XGM_NBINS * 4, cs));
    s->stats.kernel_launches = 0;
    p.pass = 0;
    uint32_t& launches = s->stats.kernel_launches;
    CUDA_TRY(expand_levels(s->and_list, s->bpi, cs, launches));
    CUDA_TRY(expand_or_groups(s->or_list, s->bpi, cs, launches));
    CUDA_TRY(s->bm_list.range_mode ? expand_driver_runs(s->bm_list, p.hdr, s->range_bits, s->bpi, cs, launches)
                                   : expand_levels(s->bm_list, s->bpi, cs, launches));
    CUDA_TRY(cudaEventRecord(s->ev0.get(), cs));
    xgm_status st = launch_match(s, p, cs);
    if (st != XGM_OK) return st;
    CUDA_TRY(cudaEventRecord(s->ev1.get(), cs));
    CUDA_TRY(xgm_launch_topk(p, s->nq, s->grids.topk, launches, cs));
    /* second pass: only queries whose candidate buffer overflowed do any work (device-side flag) */
    XgmKernelParams p2 = p;
    p2.pass = 1;
    st = launch_match(s, p2, cs);
    if (st != XGM_OK) return st;
    CUDA_TRY(xgm_launch_topk(p2, s->nq, s->grids.topk, launches, cs));
    CUDA_TRY(cudaEventRecord(s->ev2.get(), cs));
    if (shared) {
        CUDA_TRY(cudaEventRecord(s->ev_done.get(), cs));
        lk.unlock();
        CUDA_TRY(cudaStreamWaitEvent(s->stream.get(), s->ev_done.get(), 0));
    }
    return XGM_OK;
}

static xgm_status submit_impl(xgm_searcher* s, const xgm_query* queries, uint32_t nq) {
    const auto t_submit0 = std::chrono::steady_clock::now();
    CUDA_TRY(cudaSetDevice(s->ix->device));
    const cudaStream_t stream = s->stream.get();
    XgmDevQuery* const hq = s->queries.h.get();
    s->plan.resize(nq);
    s->nq = nq;
    PlannedSegments segs;
    segs.and_list.reserve(4096);
    /* work granularity: enough items to balance ~grid*8 warps, at most 32 driver blocks per item.  Finding it from
     * the driver block counts would mean planning twice, so it is a fixed small granularity scaled by batch size. */
    uint32_t bpi = nq >= 256 ? 12 : (nq >= 16 ? 4 : 1); /* 12: scripts/sweep_bm.py, 8..32 x range widths 2^17..2^20 */
    if (s->bpi_override && nq >= 256) bpi = s->bpi_override; /* XGM_BPI: measurement aid */
    s->any_sort = false;
    uint64_t alg = 0;
    /* Planning (term lookup, Weight::init_, evaluation order, work items) is independent per query:
     * large batches are planned by a few host threads, each into its own work lists. */
    int T = 1;
    if (nq >= 512) T = PlannerPool::get().threads();
    if (T <= 1) {
        for (uint32_t i = 0; i < nq; ++i) plan_query(s, queries[i], i, s->plan[i], hq[i], segs);
    } else {
        std::vector<PlannedSegments> ts(T);
        PlannerPool::get().run(T, [&](int t) {
            uint32_t a = (uint32_t)((uint64_t)nq * t / T), b = (uint32_t)((uint64_t)nq * (t + 1) / T);
            ts[t].bm_list.reserve((size_t)(b - a));
            for (uint32_t i = a; i < b; ++i) plan_query(s, queries[i], i, s->plan[i], hq[i], ts[t]);
        });
        for (int t = 0; t < T; ++t) {
            segs.and_list.insert(segs.and_list.end(), ts[t].and_list.begin(), ts[t].and_list.end());
            segs.or_list.insert(segs.or_list.end(), ts[t].or_list.begin(), ts[t].or_list.end());
            segs.bm_list.insert(segs.bm_list.end(), ts[t].bm_list.begin(), ts[t].bm_list.end());
        }
    }
    const auto t_planned = std::chrono::steady_clock::now();
    for (uint32_t i = 0; i < nq; ++i) {
        if (s->plan[i].sort_by || hq[i].route == XGM_ROUTE_OR || s->plan[i].aux_subqs) s->any_sort = true; /* keys/aux needed on the host */
        alg += s->plan[i].alg_bytes;
    }
    /* segments → each list's pinned staging, in the order the device expands them */
    s->bpi = bpi;
    BmList& bm = s->bm_list;
    bm.range_mode = !segs.bm_list.empty() && nq >= 256 && s->range_bits != 0;
    bm.nruns = 0;
    xgm_status st = order_levels(s->and_list, segs.and_list, bpi, stream);
    if (st == XGM_OK) st = order_or_groups(s->or_list, segs.or_list, bpi, stream);
    if (st == XGM_OK) st = bm.range_mode ? order_driver_runs(s, segs.bm_list, bpi) : order_levels(bm, segs.bm_list, bpi, stream);
    if (st != XGM_OK) return st;
    const auto t_interleaved = std::chrono::steady_clock::now();
    s->stats = xgm_batch_stats{};
    s->stats.algorithmic_bytes = alg;
    s->stats.work_items = s->and_list.nitems + s->or_list.nitems + bm.nitems;
    s->stats.h2d_bytes = (uint64_t)nq * sizeof(XgmDevQuery) + (uint64_t)(s->and_list.nseg + s->or_list.nseg + bm.nseg + bm.nruns) * sizeof(XgmWorkItem);
    s->stats.d2h_bytes = (uint64_t)nq * sizeof(XgmDevResult) + (uint64_t)nq * s->max_topk * (8 + 4 + (s->any_sort ? 8 : 0));
    XgmKernelParams& p = s->params;
    fill_index_params(s->ix, p);
    p.queries = s->queries.d.get(); p.items = s->and_list.d_exp.get(); p.nitems = s->and_list.nitems; p.nq = nq;
    p.items_or = s->or_list.d_exp.get(); p.nitems_or = s->or_list.nitems;
    p.items_bm = bm.d_exp.get(); p.nitems_bm = bm.nitems;
    p.nitems_bm_dev = bm.range_mode ? bm.rng_total.d.get() : nullptr;
    p.bm_segs = bm.range_mode ? bm.seg.d.get() : nullptr;
    p.work_counter = reinterpret_cast<uint32_t*>(s->d_ctrl.get());
    p.qstate = reinterpret_cast<XgmQState*>(s->d_ctrl.get() + XGM_CTRL_HDR);
    p.hist = reinterpret_cast<uint32_t*>(s->d_ctrl.get() + XGM_CTRL_HDR + (size_t)s->max_batch * sizeof(XgmQState));
    p.topk_list = s->d_topk_list.get();
    p.match_cap = s->match_cap; p.keep_cap = s->keep_cap;
    p.pool_total = s->pool_total; p.pool_w = s->d_pool_w.get(); p.pool_d = s->d_pool_d.get(); p.pool_k = s->d_pool_k.get();
    p.match_w = s->d_match_w.get(); p.match_d = s->d_match_d.get(); p.match_k = s->d_match_k.get();
    p.out_stride = s->max_topk; p.out_w = s->d_out_w; p.out_d = s->d_out_d; p.out_k = s->d_out_k; p.out_info = s->d_info;
    p.raise_log = s->raise.d.get();
    s->any_raise = false;
    for (uint32_t i = 0; i < nq; ++i) s->any_raise |= s->plan[i].log_raises;
    s->any_or_fast = s->any_or_slow = false;
    s->ntileq = 0;
    for (uint32_t i = 0; i < nq; ++i)
        if (hq[i].route == XGM_ROUTE_OR && s->plan[i].on_device) {
            if (hq[i].or_fast == XGM_OR_FAST_TILE) s->tileq.h.get()[s->ntileq++] = i;
            else if (hq[i].or_fast == XGM_OR_FAST_OR3) s->any_or_fast = true;
            else s->any_or_slow = true;
        }
    p.tileq = s->tileq.d.get(); p.ntileq = s->ntileq;
    CUDA_TRY(s->tileq.upload(s->ntileq, stream));
    CUDA_TRY(s->queries.upload(nq, stream));
    CUDA_TRY(s->and_list.upload(0, stream));
    CUDA_TRY(s->or_list.upload(0, stream));
    CUDA_TRY(bm.upload(bm.nruns, stream)); /* the runs follow the segments */
    if (g_trace) { s->tr_submit = t_submit0; s->tr_planned = t_interleaved; CUDA_TRY(cudaEventRecord(s->tr_h2d.get(), stream)); }
    st = launch_batch(s);
    if (st != XGM_OK) return st;
    size_t ns = (size_t)nq * s->max_topk;
    if (s->device_only) { /* the caller reads the result slab on the device (multi-GPU exchange + merge) */
        s->stats.d2h_bytes = 0;
        s->pending = true;
        s->stats.host_plan_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_submit0).count();
        return XGM_OK;
    }
    CUDA_TRY(cudaMemcpyAsync(s->h_info.get(), s->d_info, (size_t)nq * sizeof(XgmDevResult), cudaMemcpyDeviceToHost, stream));
    if (bm.range_mode) CUDA_TRY(cudaMemcpyAsync(bm.rng_total.h.get(), bm.rng_total.d.get(), 4, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaMemcpyAsync(s->h_out_w.get(), s->d_out_w, ns * 8, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaMemcpyAsync(s->h_out_d.get(), s->d_out_d, ns * 4, cudaMemcpyDeviceToHost, stream));
    if (s->any_sort) CUDA_TRY(cudaMemcpyAsync(s->h_out_k.get(), s->d_out_k, ns * 8, cudaMemcpyDeviceToHost, stream));
    if (s->any_raise) {
        CUDA_TRY(cudaMemcpyAsync(s->raise.h.get(), s->raise.d.get(), (size_t)nq * XGM_RAISE_LOG * sizeof(XgmRaise), cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaMemcpyAsync(s->h_qstate.get(), s->d_ctrl.get() + XGM_CTRL_HDR, (size_t)nq * sizeof(XgmQState), cudaMemcpyDeviceToHost, stream));
    }
    s->pending = true;
    s->stats.host_plan_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_submit0).count();
    if (g_trace) { CUDA_TRY(cudaEventRecord(s->tr_out.get(), stream)); s->tr_launched = std::chrono::steady_clock::now(); }
    if (getenv("XGM_DEBUG_TIMING"))
        fprintf(stderr, "xgm submit: plan %.3f ms, interleave %.3f ms, enqueue %.3f ms (T=%d, items %zu)\n",
                std::chrono::duration<float, std::milli>(t_planned - t_submit0).count(),
                std::chrono::duration<float, std::milli>(t_interleaved - t_planned).count(),
                std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_interleaved).count(), T,
                (size_t)s->and_list.nitems + s->or_list.nitems + bm.nitems);
    return XGM_OK;
}

static void finish_info(const PlannedQuery& pq, const XgmDevResult* dr, const uint64_t* keys, bool is_or,
                        xgm_mset_info* o, const XgmRaise* raises = nullptr, uint32_t nraise = 0) {
    memset(o, 0, sizeof(*o));
    o->first = pq.first;
    o->status = pq.status;
    o->max_possible = pq.max_possible;
    if (pq.status != XGM_OK) return;
    uint32_t lb = pq.tf_min, est = pq.tf_est, ub = pq.tf_max;
    uint32_t size = 0, known = 0;
    double max_w = 0;
    if (pq.on_device) {
        size = dr->n; known = dr->known; o->exact_matches = dr->exact;
        max_w = dr->max_w;
        /* ProtoMSet::finalise, protomset.h:484-612 (no collapser / decider / percent cut-off) */
        if (pq.count_only) { size = 0; lb = est = ub = dr->exact; }
        else if (size != pq.topk) lb = est = ub = size;
        else if (known < pq.check_at_least) lb = est = ub = known;
        else { lb = std::max(lb, known); est = std::max(est, known); }
        /* The kernel counts "among the first max(check_at_least, k+1) or fewer than k earlier matches are
         * greater", which is ProtoMSet's count when check_at_least <= k+1 (min_weight rises at the heap build)
         * or is never reached.  In between, the reference's min_weight only starts rising at the first
         * replacement after known_matching_docs reached check_at_least (protomset.h:377-398), so it counts
         * more: our count is then a lower bound — flag the bounds. */
        if (pq.check_at_least > pq.topk + 1 && known < dr->exact && !pq.count_only && pq.sort_by == XGM_SORT_REL_VAL)
            o->flags |= XGM_MSET_BOUNDS_APPROX; /* relevance-then-value still uses the simple counting rule */
        if (dr->flags & (XGM_RES_LOST | XGM_RES_PENDING)) o->status = XGM_E_UNIMPLEMENTED; /* lost or pending: pathological tie mass */
        /* a count-only query keeps one document only for the percentage scale: its bounds are the exact count */
        if ((dr->flags & XGM_RES_APPROX) && !pq.count_only) o->flags |= XGM_MSET_BOUNDS_APPROX;
        if (dr->flags & XGM_RES_SKIPPED) o->flags |= XGM_MSET_BOUNDS_APPROX | XGM_MSET_COUNT_LOWER_BOUND;
        /* with a stock value range the reference's estimate folds in ValueRangePostList::get_termfreq_est
         * (valuerangepostlist.cc:70-130), which is not restated (range_child) */
        if (pq.filter && !pq.mv_source && size == pq.topk && known >= pq.check_at_least) o->flags |= XGM_MSET_BOUNDS_APPROX;
    } else if (pq.check_at_least != 0) {
        lb = est = ub = 0; /* empty result set: !full() branch */
    } else if (pq.filter && !pq.mv_source) {
        o->flags |= XGM_MSET_BOUNDS_APPROX; /* bounds only, with a stock value range's estimate as above */
    }
    o->matches_lower_bound = o->uncollapsed_lower_bound = lb;
    o->matches_estimated = o->uncollapsed_estimated = est;
    o->matches_upper_bound = o->uncollapsed_upper_bound = ub;
    o->max_attained = max_w;
    o->n = size > pq.first ? size - pq.first : 0;
    if ((size != 0 || (pq.count_only && pq.on_device && dr->exact != 0)) && max_w != 0.0) {
        /* ProtoMSet::finalise_percentages protomset.h:466-471: AND → every subquery matched */
        /* AND: every leaf matches; OR ranked by relevance on the device (count-only queries included): leaves
         * matching the first ranked document */
        uint32_t subqs = dr->max_subqs;
        if (is_or && (pq.sort_by == XGM_SORT_REL || pq.count_only) && keys) subqs = (uint32_t)keys[0];
        if (pq.log_raises) {
            /* ProtoMSet::update_max_weight: the FIRST document in docid order that attains the maximum */
            if (!raises || nraise > XGM_RAISE_LOG) { o->status = XGM_E_UNIMPLEMENTED; return; }
            unsigned long long mb;
            memcpy(&mb, &max_w, 8);
            uint32_t best = 0xffffffffu;
            for (uint32_t i = 0; i < nraise; ++i)
                if (raises[i].wbits == mb && raises[i].docid < best) { best = raises[i].docid; subqs = raises[i].subqs; }
            if (best == 0xffffffffu) { o->status = XGM_E_UNIMPLEMENTED; return; }
        }
        /* a value-range / posting-source filter counts as a matching subquery (ValueRangePostList /
         * ExternalPostList::count_matching_subqs return 1) without being one of the total weighted leaves
         * (api/queryinternal.cc:1097-1098) */
        if (pq.filter_subq) subqs += 1;
        double percent_scale = (double)subqs / (double)pq.nweighted;
        percent_scale /= max_w;
        o->percent_scale_factor = percent_scale * 100.0;
    }
}

extern "C" xgm_status xgm_search_submit(xgm_searcher* s, const xgm_query* queries, uint32_t nq) {
    if (!s || !queries || nq == 0) return fail(XGM_E_INVALID, "bad arguments");
    if (nq > s->max_batch) return fail(XGM_E_INVALID, "batch %u > max_batch %u", nq, s->max_batch);
    if (s->pending) return fail(XGM_E_INVALID, "previous batch not waited for");
    return submit_impl(s, queries, nq);
}

static void worker_main(xgm_searcher* s) {
    for (;;) {
        const xgm_query* queries;
        uint32_t nq;
        {
            std::unique_lock<std::mutex> lk(s->mu);
            s->cv.wait(lk, [&] { return s->worker_exit || s->job == xgm_searcher::JOB_QUEUED; });
            if (s->worker_exit) return;
            s->job = xgm_searcher::JOB_RUNNING;
            queries = s->job_queries;
            nq = s->job_nq;
        }
        g_err[0] = 0;
        const xgm_status st = submit_impl(s, queries, nq);
        {
            std::lock_guard<std::mutex> lk(s->mu);
            s->job_status = st;
            snprintf(s->job_err, sizeof(s->job_err), "%s", g_err);
            s->job = xgm_searcher::JOB_DONE;
        }
        s->cv.notify_all();
    }
}

extern "C" xgm_status xgm_search_submit_async(xgm_searcher* s, const xgm_query* queries, uint32_t nq) {
    if (!s || !queries || nq == 0) return fail(XGM_E_INVALID, "bad arguments");
    if (nq > s->max_batch) return fail(XGM_E_INVALID, "batch %u > max_batch %u", nq, s->max_batch);
    if (s->pending) return fail(XGM_E_INVALID, "previous batch not waited for");
    if (!s->worker.joinable()) s->worker = std::thread(worker_main, s);
    {
        std::lock_guard<std::mutex> lk(s->mu);
        s->job_queries = queries;
        s->job_nq = nq;
        s->job_status = XGM_OK;
        s->job = xgm_searcher::JOB_QUEUED;
        s->pending = true;
        if (g_trace) s->tr_async = std::chrono::steady_clock::now();
    }
    s->cv.notify_all();
    return XGM_OK;
}

extern "C" xgm_status xgm_search_launched(xgm_searcher* s) {
    if (!s) return fail(XGM_E_INVALID, "null argument");
    if (!s->pending) return fail(XGM_E_INVALID, "no batch submitted");
    return join_async(s);
}

extern "C" xgm_status xgm_searcher_set_results_on_device(xgm_searcher* s, int on) {
    if (!s) return fail(XGM_E_INVALID, "null argument");
    if (s->pending) return fail(XGM_E_INVALID, "a batch is in flight");
    s->device_only = on != 0;
    return XGM_OK;
}

/* XGM_TRACE=1: host times (ms since the searcher was created: async hand-over, worker start, planned, enqueued,
 * wait entered, worker joined, stream drained, scattered) and GPU times on the same origin (plan on the device,
 * match kernels begin / end, top-k end, results on the host).  A measurement aid; nothing reads it back. */
static void trace_line(xgm_searcher* s, std::chrono::steady_clock::time_point wait_in,
                       std::chrono::steady_clock::time_point joined, std::chrono::steady_clock::time_point synced) {
    auto ms = [&](std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(t - g_tr_t0).count(); };
    float g[5] = {0, 0, 0, 0, 0};
    cudaEventElapsedTime(&g[0], g_tr_base, s->tr_h2d.get());
    cudaEventElapsedTime(&g[1], g_tr_base, s->ev0.get());
    cudaEventElapsedTime(&g[2], g_tr_base, s->ev1.get());
    cudaEventElapsedTime(&g[3], g_tr_base, s->ev2.get());
    cudaEventElapsedTime(&g[4], g_tr_base, s->tr_out.get());
    fprintf(stderr, "XGMTRACE s=%p nq=%u host async=%.3f start=%.3f planned=%.3f enq=%.3f wait=%.3f joined=%.3f synced=%.3f done=%.3f "
            "gpu h2d=%.3f k0=%.3f k1=%.3f k2=%.3f out=%.3f second_pass=%u\n", (void*)s, s->nq, ms(s->tr_async), ms(s->tr_submit), ms(s->tr_planned),
            ms(s->tr_launched), ms(wait_in), ms(joined), ms(synced), ms(std::chrono::steady_clock::now()), g[0], g[1], g[2], g[3], g[4], s->stats.second_pass_queries);
}

extern "C" xgm_status xgm_search_wait(xgm_searcher* s, uint32_t* docids, double* weights, uint64_t* sort_keys,
                                      uint32_t stride, xgm_mset_info* info) {
    if (!s || (!info && !s->device_only)) return fail(XGM_E_INVALID, "null argument");
    if (!s->pending) return fail(XGM_E_INVALID, "no batch submitted");
    const auto tr_wait_in = std::chrono::steady_clock::now();
    {
        xgm_status jst = join_async(s);
        if (jst != XGM_OK) return jst;
    }
    const auto tr_joined = std::chrono::steady_clock::now();
    CUDA_TRY(cudaSetDevice(s->ix->device));
    cudaError_t e = cudaStreamSynchronize(s->stream.get());
    s->pending = false;
    if (e != cudaSuccess) return fail(XGM_E_CUDA, "batch failed: %s", cudaGetErrorString(e));
    if (s->device_only) return XGM_OK; /* nothing was copied: the results are in the device slab */
    cudaEventElapsedTime(&s->stats.match_kernel_ms, s->ev0.get(), s->ev1.get());
    cudaEventElapsedTime(&s->stats.topk_kernel_ms, s->ev1.get(), s->ev2.get());
    const auto t_wait0 = std::chrono::steady_clock::now();
    if (s->bm_list.range_mode) s->stats.work_items = (uint64_t)s->and_list.nitems + s->or_list.nitems + s->bm_list.rng_total.h.get()[0];
    s->stats.second_pass_queries = 0;
    for (uint32_t i = 0; i < s->nq; ++i) {
        const PlannedQuery& pq = s->plan[i];
        const size_t off = (size_t)i * s->max_topk;
        const XgmDevResult& dr = s->h_info.get()[i];
        if (pq.status == XGM_OK && pq.on_device && (dr.flags & XGM_RES_SECOND_PASS)) s->stats.second_pass_queries++;
        finish_info(pq, &dr, s->any_sort ? s->h_out_k.get() + off : nullptr,
                    s->queries.h.get()[i].route == XGM_ROUTE_OR || pq.aux_subqs, &info[i],
                    s->any_raise ? s->raise.h.get() + (size_t)i * XGM_RAISE_LOG : nullptr, s->any_raise ? s->h_qstate.get()[i].nraise : 0u);
        if (pq.status == XGM_OK && pq.on_device) s->stats.algorithmic_bytes += 4ull * dr.exact;
        uint32_t n = info[i].n;
        if (n > stride) return fail(XGM_E_INVALID, "stride %u too small for %u results", stride, n);
        if (n && docids && weights) {
            memcpy(docids + (size_t)i * stride, s->h_out_d.get() + off + pq.first, (size_t)n * 4);
            memcpy(weights + (size_t)i * stride, s->h_out_w.get() + off + pq.first, (size_t)n * 8);
            if (sort_keys && pq.sort_by) memcpy(sort_keys + (size_t)i * stride, s->h_out_k.get() + off + pq.first, (size_t)n * 8);
        }
    }
    s->stats.host_wait_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_wait0).count();
    if (g_trace) trace_line(s, tr_wait_in, tr_joined, t_wait0);
    return XGM_OK;
}

extern "C" xgm_status xgm_search_batch(xgm_searcher* s, const xgm_query* queries, uint32_t nq, uint32_t* docids,
                                       double* weights, uint64_t* sort_keys, uint32_t stride, xgm_mset_info* info) {
    xgm_status st = xgm_search_submit(s, queries, nq);
    if (st != XGM_OK) return st;
    return xgm_search_wait(s, docids, weights, sort_keys, stride, info);
}

extern "C" xgm_status xgm_search(xgm_searcher* s, const xgm_query* query, uint32_t* docids, double* weights,
                                 uint64_t* sort_keys, uint32_t capacity, xgm_mset_info* info) {
    return xgm_search_batch(s, query, 1, docids, weights, sort_keys, capacity, info);
}

extern "C" xgm_status xgm_search_replay(xgm_searcher* s) {
    if (!s || s->nq == 0) return fail(XGM_E_INVALID, "no resident batch");
    if (s->pending) return fail(XGM_E_INVALID, "previous batch not waited for");
    CUDA_TRY(cudaSetDevice(s->ix->device));
    return launch_batch(s);
}

extern "C" xgm_status xgm_search_device_results(xgm_searcher* s, void** weights, void** docids, void** counts, uint32_t* stride) {
    if (!s) return fail(XGM_E_INVALID, "null argument");
    if (weights) *weights = s->d_out_w;
    if (docids) *docids = s->d_out_d;
    if (counts) *counts = s->d_info;
    if (stride) *stride = s->max_topk;
    return XGM_OK;
}

extern "C" xgm_status xgm_search_device_slab(xgm_searcher* s, void** base, uint64_t* bytes, uint64_t* off_docids,
                                             uint64_t* off_counts, uint32_t* stride) {
    if (!s) return fail(XGM_E_INVALID, "null argument");
    if (base) *base = s->d_slab.get();
    if (bytes) *bytes = s->slab_bytes;
    if (off_docids) *off_docids = s->slab_off_d;
    if (off_counts) *off_counts = s->slab_off_info;
    if (stride) *stride = s->max_topk;
    return XGM_OK;
}

extern "C" xgm_status xgm_search_device_slab_keys(xgm_searcher* s, uint64_t* off_keys) {
    if (!s || !off_keys) return fail(XGM_E_INVALID, "null argument");
    *off_keys = s->slab_off_k;
    return XGM_OK;
}

extern "C" xgm_status xgm_search_last_stats(xgm_searcher* s, xgm_batch_stats* out) {
    if (!s || !out) return fail(XGM_E_INVALID, "null argument");
    if (!s->pending && s->nq) {
        cudaEventSynchronize(s->ev2.get());
        cudaEventElapsedTime(&s->stats.match_kernel_ms, s->ev0.get(), s->ev1.get());
        cudaEventElapsedTime(&s->stats.topk_kernel_ms, s->ev1.get(), s->ev2.get());
    }
    *out = s->stats;
    return XGM_OK;
}

extern "C" xgm_status xgm_index_copy_doclengths(const xgm_index* ix, uint32_t first_docid, uint32_t n, uint32_t* out) {
    if (!ix || (n && !out)) return fail(XGM_E_INVALID, "null argument");
    if ((uint64_t)first_docid + n > (uint64_t)ix->lastdocid + 1) return fail(XGM_E_INVALID, "docid range beyond lastdocid");
    CUDA_TRY(cudaSetDevice(ix->device));
    if (n) CUDA_TRY(cudaMemcpy(out, ix->d_doclen.get() + first_docid, (size_t)n * 4, cudaMemcpyDeviceToHost));
    return XGM_OK;
}

/* ------------------------------------------------------------------ multi-shard merge */

extern "C" void xgm_unshard(uint32_t* docids, uint32_t n, uint32_t shard, uint32_t nshards) {
    /* unshard(), src/xapian/backends/multi.h:66-70 */
    for (uint32_t i = 0; i < n; ++i) docids[i] = (docids[i] - 1) * nshards + shard + 1;
}

namespace {
struct MItem { double w; uint32_t d; uint64_t k; };
struct MCmp {
    uint32_t sort_by, reverse;
    bool operator()(const MItem& a, const MItem& b) const {
        if (sort_by == XGM_SORT_VAL_REL || sort_by == XGM_SORT_VAL) {
            if (a.k > b.k) return reverse != 0;
            if (a.k < b.k) return reverse == 0;
            if (sort_by == XGM_SORT_VAL) return a.d < b.d;
        }
        if (a.w > b.w) return true;
        if (a.w < b.w) return false;
        if (sort_by == XGM_SORT_REL_VAL) {
            if (a.k > b.k) return reverse != 0;
            if (a.k < b.k) return reverse == 0;
        }
        return a.d < b.d;
    }
};
}

/* Matcher::merge_mset (matcher.cc:653-782) + MSet::Internal::merge_stats (api/mset.cc:376-395). The
 * reference pops a heap of per-shard cursors under mcmp; under a strict total order that equals
 * merging the sorted runs, done here with std::merge-style selection. */
extern "C" xgm_status xgm_merge_msets(const uint32_t* const* docids, const double* const* weights,
                                      const uint64_t* const* sort_keys, const xgm_mset_info* infos, uint32_t nparts,
                                      uint32_t first, uint32_t maxitems, uint32_t sort_by, uint32_t sort_reverse,
                                      uint32_t* out_docids, double* out_weights, uint64_t* out_sort_keys,
                                      xgm_mset_info* out_info) {
    if (!docids || !weights || !infos || !out_info || (maxitems && (!out_docids || !out_weights)))
        return fail(XGM_E_INVALID, "null argument");
    xgm_mset_info o;
    memset(&o, 0, sizeof(o));
    std::vector<MItem> all;
    for (uint32_t p = 0; p < nparts; ++p) {
        const xgm_mset_info& m = infos[p];
        o.matches_lower_bound += m.matches_lower_bound; o.matches_estimated += m.matches_estimated;
        o.matches_upper_bound += m.matches_upper_bound;
        o.uncollapsed_lower_bound += m.uncollapsed_lower_bound; o.uncollapsed_estimated += m.uncollapsed_estimated;
        o.uncollapsed_upper_bound += m.uncollapsed_upper_bound;
        o.exact_matches += m.exact_matches;
        o.max_possible = std::max(o.max_possible, m.max_possible);
        if (m.max_attained > o.max_attained) { o.max_attained = m.max_attained; o.percent_scale_factor = m.percent_scale_factor; }
        if (m.status != XGM_OK) o.status = m.status;
        o.flags |= m.flags;
        for (uint32_t i = 0; i < m.n; ++i)
            all.push_back(MItem{weights[p][i], docids[p][i], (sort_keys && sort_keys[p]) ? sort_keys[p][i] : 0ull});
    }
    MCmp cmp{sort_by, sort_reverse};
    std::sort(all.begin(), all.end(), cmp);
    size_t n = all.size() > first ? all.size() - first : 0;
    n = std::min<size_t>(n, maxitems);
    for (size_t i = 0; i < n; ++i) {
        out_docids[i] = all[first + i].d;
        out_weights[i] = all[first + i].w;
        if (out_sort_keys) out_sort_keys[i] = all[first + i].k;
    }
    o.n = (uint32_t)n;
    o.first = first;
    *out_info = o;
    return XGM_OK;
}

/* The relevance-order entry points below: no orders, no keys, first = 0, maxitems = k. */
static XgmMergeArgs rel_merge_args(uint32_t nparts, uint32_t nq, uint32_t stride, uint32_t k, void* out_w, void* out_d,
                                   void* out_n) {
    XgmMergeArgs a{};
    a.nparts = nparts; a.nq = nq; a.stride = stride; a.first = 0; a.maxitems = k;
    a.out_w = static_cast<double*>(out_w); a.out_d = static_cast<uint32_t*>(out_d); a.out_n = static_cast<uint32_t*>(out_n);
    return a;
}

extern "C" xgm_status xgm_merge_topk_device(const void* gw, const void* gd, const void* ginfo, uint32_t nparts, uint32_t nq,
                                            uint32_t stride, uint32_t k, void* out_w, void* out_d, void* out_n,
                                            void* cuda_stream) {
    if (!gw || !gd || !ginfo || !out_w || !out_d || !out_n || nparts == 0 || nq == 0 || k == 0 || k > stride)
        return fail(XGM_E_INVALID, "bad arguments");
    if (xgm_merge_smem_bytes(nparts, k, false) > XGM_MERGE_MAX_SMEM || nparts > XGM_MERGE_MAX_PARTS)
        return fail(XGM_E_INVALID, "nparts*k too large for the merge kernel");
    XgmMergeArgs a = rel_merge_args(nparts, nq, stride, k, out_w, out_d, out_n);
    a.gw = static_cast<const double*>(gw); a.gd = static_cast<const uint32_t*>(gd);
    a.ginfo = static_cast<const XgmDevResult*>(ginfo);
    a.part_w = (size_t)nq * stride * 8; a.part_d = (size_t)nq * stride * 4; a.part_info = (size_t)nq * sizeof(XgmDevResult);
    CUDA_TRY(xgm_launch_merge(a, static_cast<cudaStream_t>(cuda_stream)));
    return XGM_OK;
}

/* Checks of a gathered slab layout shared by both slab entry points: 8-byte aligned offsets, regions in slab order
 * (weights | docids | records | keys when off_keys != 0) each large enough for nq*stride records. */
static xgm_status check_slab_layout(uint64_t slab_bytes, uint64_t off_docids, uint64_t off_counts, uint64_t off_keys,
                                    bool keys, uint32_t nq, uint32_t stride) {
    if ((slab_bytes | off_docids | off_counts | off_keys) & 7) return fail(XGM_E_INVALID, "slab offsets must be 8-byte aligned");
    const uint64_t ns = (uint64_t)nq * stride, end_counts = off_counts + (uint64_t)nq * sizeof(XgmDevResult);
    if (off_docids < ns * 8 || off_counts < off_docids + ns * 4 || slab_bytes < end_counts ||
        (keys && (off_keys < end_counts || slab_bytes < off_keys + ns * 8)))
        return fail(XGM_E_INVALID, "slab layout too small for nq*stride records");
    return XGM_OK;
}

extern "C" xgm_status xgm_merge_topk_device_slab(const void* gathered, uint64_t slab_bytes, uint64_t off_docids,
                                                 uint64_t off_counts, uint32_t nparts, uint32_t nq, uint32_t stride,
                                                 uint32_t k, void* out_w, void* out_d, void* out_n, void* cuda_stream) {
    if (!gathered || !out_w || !out_d || !out_n || nparts == 0 || nq == 0 || k == 0 || k > stride)
        return fail(XGM_E_INVALID, "bad arguments");
    xgm_status st = check_slab_layout(slab_bytes, off_docids, off_counts, 0, false, nq, stride);
    if (st != XGM_OK) return st;
    if (xgm_merge_smem_bytes(nparts, k, false) > XGM_MERGE_MAX_SMEM || nparts > XGM_MERGE_MAX_PARTS)
        return fail(XGM_E_INVALID, "nparts*k too large for the merge kernel");
    const unsigned char* g = static_cast<const unsigned char*>(gathered);
    XgmMergeArgs a = rel_merge_args(nparts, nq, stride, k, out_w, out_d, out_n);
    a.gw = reinterpret_cast<const double*>(g); a.gd = reinterpret_cast<const uint32_t*>(g + off_docids);
    a.ginfo = reinterpret_cast<const XgmDevResult*>(g + off_counts);
    a.part_w = a.part_d = a.part_info = slab_bytes;
    CUDA_TRY(xgm_launch_merge(a, static_cast<cudaStream_t>(cuda_stream)));
    return XGM_OK;
}

extern "C" xgm_status xgm_merge_mset_device_slab(const void* gathered, uint64_t slab_bytes, uint64_t off_docids,
                                                 uint64_t off_counts, uint64_t off_keys, const uint8_t* orders,
                                                 uint32_t nparts, uint32_t nq, uint32_t stride, uint32_t first,
                                                 uint32_t maxitems, void* out_weights, void* out_docids,
                                                 void* out_keys, void* out_counts, void* cuda_stream) {
    if (!gathered || !out_weights || !out_docids || !out_keys || !out_counts || nparts == 0 || nq == 0 || maxitems == 0 ||
        (uint64_t)first + maxitems > stride)
        return fail(XGM_E_INVALID, "bad arguments");
    xgm_status st = check_slab_layout(slab_bytes, off_docids, off_counts, off_keys, true, nq, stride);
    if (st != XGM_OK) return st;
    /* the limit counts the keys whether or not the orders read them */
    if (xgm_merge_smem_bytes(nparts, (uint64_t)first + maxitems, true) > XGM_MERGE_MAX_SMEM || nparts > XGM_MERGE_MAX_PARTS)
        return fail(XGM_E_INVALID, "nparts*(first+maxitems) too large for the merge kernel");
    const unsigned char* g = static_cast<const unsigned char*>(gathered);
    XgmMergeArgs a{};
    a.gw = reinterpret_cast<const double*>(g); a.gd = reinterpret_cast<const uint32_t*>(g + off_docids);
    a.gk = orders ? reinterpret_cast<const uint64_t*>(g + off_keys) : nullptr; /* no orders: relevance, no keys */
    a.ginfo = reinterpret_cast<const XgmDevResult*>(g + off_counts);
    a.part_w = a.part_d = a.part_k = a.part_info = slab_bytes;
    a.orders = orders;
    a.nparts = nparts; a.nq = nq; a.stride = stride; a.first = first; a.maxitems = maxitems;
    a.out_w = static_cast<double*>(out_weights); a.out_d = static_cast<uint32_t*>(out_docids);
    a.out_k = static_cast<uint64_t*>(out_keys); a.out_n = static_cast<uint32_t*>(out_counts);
    CUDA_TRY(xgm_launch_merge(a, static_cast<cudaStream_t>(cuda_stream)));
    return XGM_OK;
}
