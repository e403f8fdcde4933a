/* xgm_kernels.cu — sm_90a (H100) kernels of the matcher hot path.
 *
 *   xgm_and_kernel          decode + warp-galloping intersection + fused BM25 (reference:
 *                           GlassPostList::next/skip_to glass_postlist.cc:768-991, MultiAndPostList::
 *                           find_next_match multiandpostlist.cc:179-206, get_weight :149-159,
 *                           BM25Weight::get_sumpart bm25weight.cc:170-181, doclen fetch postlisttree.h:184-195)
 *   xgm_and_bm3_kernel      the same AND when every list but the driver has a membership bitmap
 *   xgm_or_kernel           owner-leaf union with the reference's tree-order sum (OrPostList, orpostlist.cc:93-204)
 *   xgm_or3_kernel          the same OR for at most five leaves, all with bitmaps
 *   xgm_or_tile_kernel      documents with two or more leaves of such an OR, by bitmap union
 *   xgm_topk_small_kernel   ProtoMSet top-k + match counting (protomset.h:295-400,484-683; msetcmp.cc:54-98):
 *   xgm_topk_kernel         a warp per query with a handful of matches, a CTA per query otherwise
 *   xgm_merge_kernel        merge of the per-shard top-k lists (Matcher::merge_mset)
 *   xgm_coarse_kernel       the coarse bitmaps (a bit per 8 docids) from the membership bitmaps, at index upload
 *   xgm_decode_kernel       round-trip decode of one term (index self-check)
 *   xgm_expand_items_kernel work items of a level-ordered list from its segments
 *   xgm_range_{count,scan,fill}_kernel   work items of the range-major bitmap AND list
 *
 * Integer/pointer work: no tensor cores. Packed blocks are staged global→shared with the bulk-copy
 * engine (cp.async.bulk + mbarrier, SASS UBLKCP), deltas are undone with a warp prefix sum, every
 * f64 operation of BM25 is an explicit round-to-nearest intrinsic so nothing is contracted into an
 * FMA and the weights are bit-identical to the reference's x86-64 build.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "xgm_device.h"

#define FULL 0xffffffffu

/* cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute and one process may drive several
 * GPUs through the C-ABI (an xgm_index carries its device): remember the opted-in size per (kernel, device). */
#define XGM_MAX_DEVICES 64
static cudaError_t optin_smem(const void* fn, int which, size_t bytes) {
    static size_t have[2][XGM_MAX_DEVICES]; /* raised monotonically; racing threads set the same or a larger value */
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    if (dev < 0 || dev >= XGM_MAX_DEVICES) return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (bytes <= have[which][dev]) return cudaSuccess;
    e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) have[which][dev] = bytes;
    return e;
}

/* ------------------------------------------------------------------ PTX helpers */

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
/* on shared-space addresses (hot loops precompute them: no generic→shared conversion per call) */
__device__ __forceinline__ void mbar_expect_tx_a(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s_a(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait_a(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "XGM_WAITA:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra XGM_DONEA;\n"
        "bra XGM_WAITA;\n"
        "XGM_DONEA:\n"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) { mbar_expect_tx_a(smem_u32(bar), bytes); }
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    bulk_g2s_a(smem_u32(dst), src, bytes, smem_u32(bar));
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) { mbar_wait_a(smem_u32(bar), parity); }

/* ------------------------------------------------------------------ block decode */

#define STAGE_WORDS 132 /* 128 packed words at 32 bits + slack for the funnel-shift's high word; 16B multiple */

__device__ __forceinline__ uint32_t bitmask(uint32_t bits) { return bits >= 32 ? 0xffffffffu : ((1u << bits) - 1u); }

__device__ __forceinline__ uint32_t unpack_sm(const uint32_t* st, uint32_t idx, uint32_t bits, uint32_t mask) {
    uint32_t o = idx * bits;
    uint32_t wi = o >> 5, sh = o & 31;
    return __funnelshift_r(st[wi], st[wi + 1], sh) & mask;
}

/* random access into a packed global block (rare path: only for surviving documents) */
__device__ __forceinline__ uint32_t unpack_gl(const uint4* col, uint32_t off16, uint32_t idx, uint32_t bits) {
    if (bits == 0) return 0;
    const uint32_t* base = reinterpret_cast<const uint32_t*>(col + off16);
    uint32_t o = idx * bits;
    uint32_t wi = o >> 5, sh = o & 31;
    uint32_t lo = __ldg(base + wi);
    uint32_t hi = (sh + bits > 32) ? __ldg(base + wi + 1) : 0u;
    return __funnelshift_r(lo, hi, sh) & bitmask(bits);
}

/* Stage one packed block (16*bits bytes) into the warp's shared buffer with the bulk-copy engine. */
__device__ __forceinline__ void stage_block(const uint4* col, uint32_t off16, uint32_t bits, uint32_t* st,
                                            uint64_t* bar, uint32_t& phase, uint32_t lane) {
    __syncwarp();
    if (bits == 0) return;
    if (lane == 0) {
        mbar_expect_tx(bar, bits * 16u);
        bulk_g2s(st, col + off16, bits * 16u, bar);
    }
    mbar_wait(bar, phase);
    phase ^= 1u;
}

/* Decode the 128 docids of a staged block: lane l gets postings 4l..4l+3 (ascending). */
__device__ __forceinline__ void decode_docids(const uint32_t* st, uint32_t bits, uint32_t first, uint32_t lane,
                                              uint32_t d[4]) {
    uint32_t v0 = 0, v1 = 0, v2 = 0, v3 = 0;
    if (bits) {
        uint32_t mask = bitmask(bits);
        v0 = unpack_sm(st, 4 * lane + 0, bits, mask);
        v1 = unpack_sm(st, 4 * lane + 1, bits, mask);
        v2 = unpack_sm(st, 4 * lane + 2, bits, mask);
        v3 = unpack_sm(st, 4 * lane + 3, bits, mask);
    }
    /* docid_i = docid_{i-1} + v_i + 1, docid_0 = first */
    uint32_t s0 = v0 + (lane ? 1u : 0u);
    uint32_t s1 = s0 + v1 + 1u;
    uint32_t s2 = s1 + v2 + 1u;
    uint32_t s3 = s2 + v3 + 1u;
    uint32_t t = s3;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t n = __shfl_up_sync(FULL, t, o);
        if ((int)lane >= o) t += n;
    }
    uint32_t base = first + (t - s3);
    d[0] = base + s0;
    d[1] = base + s1;
    d[2] = base + s2;
    d[3] = base + s3;
}

/* ------------------------------------------------------------------ BM25 */

/* BM25Weight::get_sumpart, bm25weight.cc:170-181, operation for operation:
 *   normlen = max(len * len_factor, min_normlen)
 *   denom   = k1 * (normlen * b + (1 - b)) + wdf
 *   return termweight * (wdf / denom)                                            */
__device__ __forceinline__ double bm25_sumpart(double termweight, const XgmDevQuery* q, uint32_t wdf, uint32_t len) {
    double normlen = __dmul_rn((double)len, q->len_factor);
    normlen = normlen < q->min_normlen ? q->min_normlen : normlen;
    double wdf_d = (double)wdf;
    double t = __dadd_rn(__dmul_rn(normlen, q->b), q->one_minus_b);
    double denom = __dadd_rn(__dmul_rn(q->k1, t), wdf_d);
    return __dmul_rn(termweight, __ddiv_rn(wdf_d, denom));
}

/* ------------------------------------------------------------------ skip-table search */

/* Largest block index i in [cur, n) with hdr[i].first <= target (sentinel at hdr[n]); returns cur
 * when hdr[cur].first > target (caller checks bh.first).  Also returns that block's header and the
 * first docid of the following block.  Warp-galloping: one coalesced look at the next 32 headers
 * (the common case of a leapfrog moving forward), then a 32-ary search over the rest of the list. */
__device__ __forceinline__ uint32_t warp_seek(const XgmBlockHdr* __restrict__ hdr, uint32_t cur, uint32_t n,
                                              uint32_t target, uint32_t lane, XgmBlockHdr& bh, uint32_t& next_first) {
    const uint32_t i = cur + lane;
    uint4 hv = make_uint4(XGM_SENTINEL, 0u, 0u, 0u);
    if (i <= n) hv = __ldg(reinterpret_cast<const uint4*>(hdr + i));
    const uint32_t cnt = __popc(__ballot_sync(FULL, hv.x <= target));
    if (cnt < 32) {
        const uint32_t src = cnt ? cnt - 1 : 0;
        bh.first = __shfl_sync(FULL, hv.x, src);
        bh.doc_off = __shfl_sync(FULL, hv.y, src);
        bh.tf_off = __shfl_sync(FULL, hv.z, src);
        bh.meta = __shfl_sync(FULL, hv.w, src);
        next_first = __shfl_sync(FULL, hv.x, src + 1);
        return cur + src;
    }
    uint32_t lo = cur + 31, hi = n; /* hdr[lo].first <= target < hdr[hi].first */
    while (hi - lo > 1) {
        const uint32_t step = (hi - lo + 31) / 32;
        uint32_t pidx = lo + (lane + 1) * step;
        if (pidx > hi) pidx = hi;
        const uint32_t fp = __ldg(&hdr[pidx].first);
        const uint32_t c = __popc(__ballot_sync(FULL, fp <= target));
        uint32_t nlo = lo + c * step, nhi = lo + (c + 1) * step;
        if (nlo > hi) nlo = hi;
        if (nhi > hi) nhi = hi;
        lo = nlo;
        hi = nhi;
    }
    const uint4 h = __ldg(reinterpret_cast<const uint4*>(hdr + lo));
    bh.first = h.x; bh.doc_off = h.y; bh.tf_off = h.z; bh.meta = h.w;
    next_first = __ldg(&hdr[lo + 1].first);
    return lo;
}

/* ------------------------------------------------------------------ value-slot predicates (C5) */

__device__ __forceinline__ bool doc_passes_filter(const XgmKernelParams& p, const XgmDevQuery* q, uint32_t did) {
    if (q->filter == 0) return true;
    const XgmDevSlot& s = p.slots[q->filter_slot];
    if (!s.voff) return false;
    uint32_t a = __ldg(&s.voff[did]), b = __ldg(&s.voff[did + 1]);
    if (a == b) return false;
    if (q->filter == 1) { /* stock OP_VALUE_RANGE on the (first) value, valuerangepostlist.cc:132-151 */
        uint64_t v = __ldg(&s.vals[a]);
        return v >= q->range_lo && v <= q->range_hi;
    }
    /* MultipleValueRange::insideRange, src/multivalue/range.cc:351-368: first value >= lo must be <= hi */
    for (uint32_t i = a; i < b; ++i) {
        uint64_t v = __ldg(&s.vals[i]);
        if (v >= q->range_lo) return v <= q->range_hi;
    }
    return false;
}

__device__ __forceinline__ uint64_t doc_sort_key(const XgmKernelParams& p, const XgmDevQuery* q, uint32_t did) {
    const XgmDevSlot& s = p.slots[q->sort_slot];
    if (!s.voff) return q->sort_missing;
    uint32_t a = __ldg(&s.voff[did]), b = __ldg(&s.voff[did + 1]);
    if (a == b) return q->sort_missing; /* no value: "" for Enquire's value sorts, "\xff" / "\0" for Xapiand's SerialiseKey */
    return __ldg(&s.vals[q->sort_use_max ? b - 1 : a]);
}

/* ------------------------------------------------------------------ match emission + top-k pruning */

/* Monotone bucket of a match under the query's primary sort key: a higher bucket always ranks
 * before a lower one, so once at least topk matches sit in buckets >= b*, anything below b* can never
 * enter the MSet (the parallel analogue of ProtoMSet's rising min_weight, protomset.h:377-398). */
__device__ __forceinline__ uint32_t match_bucket(const XgmDevQuery* q, double w, uint64_t key) {
    if (q->sort_by == 0 || q->sort_by == 3) {
        double x = w * q->bucket_scale;
        uint32_t b = x >= (double)(XGM_NBINS - 1) ? XGM_NBINS - 1 : (uint32_t)x;
        return b;
    }
    /* monotone in the key: the slot's [smallest, largest] key mapped linearly, anything outside clamped */
    double x = key > q->bucket_key_min ? (double)(key - q->bucket_key_min) * q->bucket_scale : 0.0;
    uint32_t b = x >= (double)(XGM_NBINS - 1) ? XGM_NBINS - 1 : (uint32_t)x;
    return q->sort_reverse ? b : (XGM_NBINS - 1 - b);
}

/* b* and the match count rise under other warps' atomics while a launch runs: every read goes to memory */
__device__ __forceinline__ uint32_t live_bstar(const XgmQState* st) {
    return *reinterpret_cast<const volatile uint32_t*>(&st->bstar);
}
__device__ __forceinline__ uint32_t live_total(const XgmQState* st) {
    return *reinterpret_cast<const volatile uint32_t*>(&st->total);
}

/* ---- MaxScore bounds (the parallel form of OrPostList's w_min checks, orpostlist.cc:113-155) */

/* Only a query ranked by weight alone, with a top-k to fill, can drop a match by a bound on its weight. */
__device__ __forceinline__ bool prunes_by_weight(const XgmDevQuery* q) {
    return q->sort_by == 0 && q->topk != 0;
}

/* Bucket of an upper bound ub.  A bound adds get_maxpart values in leaf order while the weight it bounds is summed
 * in the OrPostList tree's order, and the two round differently: the slack keeps a bound that a document attains
 * from landing one bucket below the document's own weight. */
__device__ __forceinline__ uint32_t bound_bucket(const XgmDevQuery* q, double ub) {
    return match_bucket(q, ub * (1.0 + 1e-12), 0);
}

/* init + the get_maxpart bounds of the leaves whose bit is set in mask, added in ascending leaf order */
__device__ __forceinline__ double maxpart_sum(const XgmDevQuery* q, uint32_t mask, double init) {
    for (uint32_t i = 0; i < q->nterms; ++i)
        if (mask >> i & 1u) init += q->terms[i].maxpart;
    return init;
}

/* Bound on the weight of an owner leaf (termweight tw, get_maxpart maxpart) within one of its blocks (header word
 * meta): its weight at the block's largest wdf in the shortest document, increasing in wdf and decreasing in length.
 * A saturated header byte means a wdf of 255 or more, where only the leaf's own bound holds. */
__device__ __forceinline__ double owner_block_bound(const XgmKernelParams& p, const XgmDevQuery* q, uint32_t meta,
                                                    double tw, double maxpart) {
    const uint32_t mw = XGM_HDR_MAXWDF(meta);
    return mw == 255u ? maxpart : bm25_sumpart(tw, q, mw, p.doclen_lb);
}

/* MaxScore at work-item granularity: a document owned by leaf `drv` contains no rarer leaf, so its weight is bounded
 * by the get_maxpart sum of leaves drv..n-1.  Once the top-k threshold b* is above that bound — and at least
 * check_at_least matches have been counted, as ProtoMSet requires before min_weight may rise
 * (protomset.h:185-194) — nothing the item owns can enter the MSet: it is skipped without decoding a block, and the
 * query is marked as having skipped matches.  Work items are ordered rarest leaf first, so the frequent
 * (low-weight) leaves, which hold most of the union, are usually skipped wholesale. */
__device__ __forceinline__ bool skip_owned_item(const XgmKernelParams& p, const XgmDevQuery* q, uint32_t qi,
                                                uint32_t drv, uint32_t lane) {
    XgmQState* st = &p.qstate[qi];
    const uint32_t bstar = live_bstar(st);
    if (bstar == 0 || live_total(st) < q->check_at_least) return false;
    if (bound_bucket(q, maxpart_sum(q, ~((1u << drv) - 1u), 0.0)) >= bstar) return false;
    if (lane == 0) st->skipped = 1u;
    return true;
}

/* ---- work lists: each kernel claims its items from work counter slot + pass (XGM_WC_*, xgm_device.h) */

/* The second pass, when no query of the batch re-runs: the kernel has nothing to do. */
__device__ __forceinline__ bool nothing_to_rerun(const XgmKernelParams& p) {
    return p.pass != 0 && *reinterpret_cast<volatile uint32_t*>(p.work_counter + XGM_WC_RERUN) == 0;
}

/* Claim the next of nitems work items of counter `slot` in this pass; false once they are all taken.  Warp-uniform. */
__device__ __forceinline__ bool claim_item(const XgmKernelParams& p, uint32_t slot, uint32_t nitems, uint32_t lane,
                                           uint32_t& item) {
    uint32_t i = 0;
    if (lane == 0) i = atomicAdd(p.work_counter + slot + p.pass, 1u);
    item = __shfl_sync(FULL, i, 0);
    return item < nitems;
}

/* Query qi runs in this pass: every query in the first, only those marked for re-running in the second. */
__device__ __forceinline__ bool runs_this_pass(const XgmKernelParams& p, uint32_t qi) {
    return p.pass == 0 || p.qstate[qi].rerun != 0;
}

/* A match whose weight is at least the running maximum: append it to the query's raise log (format.h) */
__device__ __forceinline__ void log_raise(const XgmKernelParams& p, uint32_t qi, unsigned long long wb, uint32_t did, uint32_t subqs) {
    const uint32_t slot = atomicAdd(&p.qstate[qi].nraise, 1u);
    if (slot < XGM_RAISE_LOG) {
        XgmRaise r;
        r.wbits = wb; r.docid = did; r.subqs = subqs;
        p.raise_log[(size_t)qi * XGM_RAISE_LOG + slot] = r;
    }
}

/* Highest bin b whose bins [b, XGM_NBINS) of histogram h hold at least `want` entries, i.e. the bin of the want-th
 * highest entry; 0 when the whole histogram holds fewer, which prunes nothing either.  32 bins per lane, a suffix scan
 * over the lanes, then a walk inside the one lane's bins.  Every lane gets the result.  Warp-converged call.  The reads
 * are volatile: other warps are still adding to a match kernel's histogram. */
__device__ __forceinline__ uint32_t bin_of_rank(const volatile uint32_t* h, uint32_t want, uint32_t lane) {
    constexpr int per = XGM_NBINS / 32;
    uint32_t mine = 0;
    for (int i = 0; i < per; ++i) mine += h[lane * per + i];
    uint32_t sfx = mine; /* entries in the bins of lanes >= lane */
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_down_sync(FULL, sfx, o);
        if ((int)lane + o < 32) sfx += t;
    }
    const uint32_t ok = __ballot_sync(FULL, sfx >= want);
    if (ok == 0) return 0;
    const uint32_t L = 31u - (uint32_t)__clz(ok); /* highest lane whose suffix reaches `want` */
    uint32_t b = L * per;
    if (lane == L) {
        /* a bounded loop: written as a while loop, this walk costs xgm_or3_kernel two registers (via raise_bstar_warp) */
        uint32_t cum = sfx - mine;
        for (int i = per - 1; i >= 0; --i) {
            cum += h[L * per + i];
            if (cum >= want) { b = L * per + i; break; }
        }
    }
    return __shfl_sync(FULL, b, L);
}

/* Highest bin with at least topk stored matches at or above it → raise the query's pruning bucket.  Warp-converged
 * call. */
__device__ __noinline__ void raise_bstar_warp(const XgmDevQuery* q, XgmQState* st, const uint32_t* hist, uint32_t lane) {
    __threadfence();
    const uint32_t nb = bin_of_rank(hist, q->topk, lane);
    if (lane == 0 && nb != 0) atomicMax(&st->bstar, nb);
}

/* Whether `stored` matches of query q are enough to raise its b*.  An OR whose union comes from the bitmap kernels
 * (or_fast OR3 or TILE) raises from topk on.  AND queries and the general OR route wait until half of what the top-k
 * kernel can rank is in use: small match sets on those routes stay unpruned, so their known_matching_docs stays
 * exact. */
__device__ __forceinline__ bool may_raise_bstar(const XgmKernelParams& p, const XgmDevQuery* q, uint32_t stored) {
    const bool bitmap_or = q->route == XGM_ROUTE_OR && q->or_fast != XGM_OR_FAST_GENERAL;
    return stored >= q->topk && (bitmap_or || stored >= p.keep_cap / 2);
}

/* Add the lanes' counts n to query qi's exact match count, in the first pass: one atomic per warp.  Warp-converged
 * call. */
__device__ __forceinline__ void count_matches(const XgmKernelParams& p, uint32_t qi, uint32_t n, uint32_t lane) {
    const uint32_t t = __reduce_add_sync(FULL, n);
    if (lane == 0 && t && p.pass == 0) atomicAdd(&p.qstate[qi].total, t);
}

/* The emission of a match, one per lane (lanes of one call may belong to different queries): count it (unless the
 * caller counts with count_matches), raise the query's best weight and log the raise, and keep it unless its bucket is
 * already below the query's pruning bucket: in the first pass in the match buffer and the histogram, in the second in
 * the query's slice of the pool.  Warp-converged call. */
__device__ __forceinline__ void emit_match_lanes(const XgmKernelParams& p, uint32_t lane, bool alive, uint32_t qi, double w,
                                                 uint32_t d, uint32_t aux, bool count = true) {
    bool crossed = false;
    /* A query with 10^5..10^6 matches would otherwise send every one of them to the same two words (total, maxw):
     * same-address atomics serialise in L2 and one such query doubled the launch time of a 4096-query batch.  The
     * lanes of one query are counted by their lowest lane, and maxw — which only rises — is read first. */
    if (p.pass == 0 && count) {
        const uint32_t grp = __match_any_sync(FULL, alive ? qi : 0xffffffffu);
        if (alive && lane == (uint32_t)__ffs(grp) - 1u) atomicAdd(&p.qstate[qi].total, (uint32_t)__popc(grp));
    }
    if (alive) {
        const XgmDevQuery* q = &p.queries[qi];
        XgmQState* st = &p.qstate[qi];
        if (p.pass == 0) {
            /* best weight over all matches (ProtoMSet::update_max_weight, protomset.h:174-183) */
            const unsigned long long wb = (unsigned long long)__double_as_longlong(w);
            if (wb >= *reinterpret_cast<volatile unsigned long long*>(&st->maxw)) {
                const unsigned long long oldmax = atomicMax(&st->maxw, wb);
                if (q->log_raises && wb >= oldmax) log_raise(p, qi, wb, d, aux);
            }
        }
        const uint64_t key = q->sort_by != 0 ? doc_sort_key(p, q, d) : 0ull;
        const uint32_t bkt = match_bucket(q, w, key);
        if (bkt >= live_bstar(st) && q->topk != 0) {
            const uint32_t idx = atomicAdd(&st->stored, 1u);
            const uint64_t kv = q->sort_by != 0 ? key : (uint64_t)aux;
            if (p.pass == 0) {
                atomicAdd(p.hist + (size_t)qi * XGM_NBINS + bkt, 1u);
                if (idx < p.match_cap) {
                    const size_t o = (size_t)qi * p.match_cap + idx;
                    p.match_w[o] = w; p.match_d[o] = d; p.match_k[o] = kv;
                }
                /* b* is recomputed whenever the stored count crosses a multiple of 256 */
                const uint32_t after = idx + 1;
                crossed = (idx >> 8) != (after >> 8) && may_raise_bstar(p, q, after);
            } else if (idx < st->pool_cap) {
                /* second pass: every match at or above the exact b* goes to the query's slice of the pool */
                const size_t o = (size_t)st->pool_off + idx;
                p.pool_w[o] = w; p.pool_d[o] = d; p.pool_k[o] = kv;
            }
        }
    }
    uint32_t m = __ballot_sync(FULL, crossed);
    while (m) {
        const uint32_t l = (uint32_t)__ffs(m) - 1u;
        m &= m - 1u;
        const uint32_t rq = __shfl_sync(FULL, qi, l);
        raise_bstar_warp(&p.queries[rq], &p.qstate[rq], p.hist + (size_t)rq * XGM_NBINS, lane);
    }
}

/* ------------------------------------------------------------------ shared per-warp scratch */

#define MATCH_WARPS 8

/* what stage_block and probe_list use */
struct __align__(16) WarpScratch {
    uint32_t stage[STAGE_WORDS];      /* packed words of the block being probed */
    uint32_t dbuf[XGM_BLOCK];         /* decoded docids of the probed block */
    uint64_t bar;                     /* completion barrier of `stage` */
};

__device__ __forceinline__ void issue_stage(const uint4* col, uint32_t off16, uint32_t bits, uint32_t* st, uint64_t* bar,
                                            uint32_t lane) {
    if (bits != 0 && lane == 0) {
        mbar_expect_tx(bar, bits * 16u);
        bulk_g2s(st, col + off16, bits * 16u, bar);
    }
}

/* Resolve the unresolved candidates of one warp against list `lh` (skip table) — the reference's
 * skip_to/check sequence of MultiAndPostList::find_next_match, multiandpostlist.cc:179-206, done for
 * 128 candidates at once.  HIT(k, pos, bh) is invoked for candidates found at position pos of block bh,
 * MISS(k) for candidates proven absent. */
template <class Hit, class Miss>
__device__ __forceinline__ uint32_t probe_list(const XgmKernelParams& p, const XgmBlockHdr* __restrict__ lh,
                                               uint32_t lnblk, uint32_t cur, WarpScratch& ws, uint32_t& phase,
                                               uint32_t lane, const uint32_t c[4], uint32_t unresolved, Hit hit,
                                               Miss miss) {
    for (;;) {
        const uint32_t m = (unresolved & 1u) ? c[0] : (unresolved & 2u) ? c[1] : (unresolved & 4u) ? c[2]
                           : (unresolved & 8u) ? c[3] : XGM_SENTINEL;
        const uint32_t tmin = __reduce_min_sync(FULL, m);
        if (tmin == XGM_SENTINEL) break;
        if (cur >= lnblk) { /* list exhausted */
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (unresolved >> k & 1u) miss(k);
            unresolved = 0;
            break;
        }
        XgmBlockHdr bh;
        uint32_t next_first;
        cur = warp_seek(lh, cur, lnblk, tmin, lane, bh, next_first);
        if (tmin < bh.first) { /* candidates below this block fall into a gap of the list */
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if ((unresolved >> k & 1u) && c[k] < bh.first) {
                    unresolved &= ~(1u << k);
                    miss(k);
                }
            continue;
        }
        uint32_t bd[4];
        stage_block(p.docs, bh.doc_off, XGM_HDR_DOC_BITS(bh.meta), ws.stage, &ws.bar, phase, lane);
        decode_docids(ws.stage, XGM_HDR_DOC_BITS(bh.meta), bh.first, lane, bd);
        const uint32_t bcount = XGM_HDR_COUNT(bh.meta);
#pragma unroll
        for (int k = 0; k < 4; ++k) ws.dbuf[4 * lane + k] = (4 * lane + k < bcount) ? bd[k] : XGM_SENTINEL;
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            if ((unresolved >> k & 1u) && c[k] < next_first) {
                const uint32_t cd = c[k];
                uint32_t pos = 0;
#pragma unroll
                for (uint32_t s = 64; s >= 1; s >>= 1)
                    if (ws.dbuf[pos + s - 1] < cd) pos += s;
                unresolved &= ~(1u << k);
                if (ws.dbuf[pos] == cd) hit(k, pos, bh);
                else miss(k);
            }
        }
        __syncwarp();
    }
    return cur;
}

/* Index of docid d in the posting list of a term that has a membership bitmap (d must be a member):
 * postings before its 256-docid group (rank directory) + set bits before it inside the group. */
__device__ __forceinline__ uint32_t bitmap_rank(const XgmKernelParams& p, const XgmDevTerm& t, uint32_t d) {
    const uint32_t* __restrict__ bm = p.bitmaps + t.bm_off;
    const uint32_t g = d >> 8, wsel = (d >> 5) & 7u;
    uint32_t r = __ldg(p.ranks + t.rk_off + g);
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(bm + g * 8));
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(bm + g * 8 + 4));
    const uint32_t ww[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
    for (uint32_t x = 0; x < 8; ++x) {
        if (x < wsel) r += __popc(ww[x]);
        else if (x == wsel) r += __popc(ww[x] & ((1u << (d & 31)) - 1u));
    }
    return r;
}

/* One lane looks docid d up in a term's posting list — for the few documents that reach scoring
 * (optional leaves of an OP_AND_MAYBE): bitmap + rank directory when the term has them, otherwise a binary
 * search over the skip table and a sequential decode inside the one block. */
__device__ __noinline__ bool lookup_posting(const XgmKernelParams& p, const XgmDevTerm& t, uint32_t d, uint32_t* wdf) {
    const XgmBlockHdr* __restrict__ h = p.hdr + t.blk_begin;
    if (t.bm_off != XGM_NO_BITMAP) {
        const uint32_t w = __ldg(p.bitmaps + t.bm_off + (d >> 5));
        if (!((w >> (d & 31)) & 1u)) return false;
        const uint32_t r = bitmap_rank(p, t, d);
        const XgmBlockHdr bh = h[r >> 7];
        *wdf = unpack_gl(p.tfs, bh.tf_off, r & 127u, XGM_HDR_TF_BITS(bh.meta));
        return true;
    }
    if (t.nblocks == 0) return false;
    uint32_t lo = 0, hi = t.nblocks; /* last block whose first docid is <= d */
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (h[mid].first <= d) lo = mid; else hi = mid;
    }
    const XgmBlockHdr bh = h[lo];
    if (bh.first > d) return false;
    const uint32_t cnt = XGM_HDR_COUNT(bh.meta), bits = XGM_HDR_DOC_BITS(bh.meta);
    uint32_t docid = bh.first, pos = 0;
    while (docid < d && pos + 1 < cnt) {
        ++pos;
        docid += unpack_gl(p.docs, bh.doc_off, pos, bits) + 1u;
    }
    if (docid != d) return false;
    *wdf = unpack_gl(p.tfs, bh.tf_off, pos, XGM_HDR_TF_BITS(bh.meta));
    return true;
}

/* OrPostList::get_weight (matcher/orpostlist.cc:93-103): the tree over the leaves that hold the document, l, r or
 * l + r per node, evaluated as the postfix program q->prog built on the host (leaf >= 0, '+' = -1).  leaf(op, v)
 * returns whether leaf op holds the document and, if it does, sets v to the leaf's weight.  The result is only
 * defined when some leaf holds the document: the callers know whether one does.  DEPTH bounds the program's stack
 * (at most one slot per leaf).  Up to a depth of 8 every slot is reached by static indexing, which keeps the stack
 * in registers; deeper stacks are indexed dynamically and live in the local-memory frame. */
template <int DEPTH, class Leaf>
__device__ __forceinline__ double or_tree_weight(const XgmDevQuery* q, Leaf leaf) {
    double stk[DEPTH];
    auto set = [&](int s, double v) {
        if constexpr (DEPTH > 8) {
            stk[s] = v;
        } else {
#pragma unroll
            for (int j = 0; j < DEPTH; ++j)
                if (s == j) stk[j] = v;
        }
    };
    auto get = [&](int s) {
        if constexpr (DEPTH > 8) return stk[s];
        double v = 0.0;
#pragma unroll
        for (int j = 0; j < DEPTH; ++j)
            if (s == j) v = stk[j];
        return v;
    };
    uint32_t has = 0; /* bit s: stack slot s holds a value */
    int sp = 0;
    for (uint32_t i = 0; i < q->prog_len; ++i) {
        const int op = q->prog[i];
        if (op >= 0) {
            double v;
            if (leaf((uint32_t)op, v)) { set(sp, v); has |= 1u << sp; }
            else has &= ~(1u << sp);
            ++sp;
        } else {
            --sp;
            const bool hl = has >> (sp - 1) & 1u, hr = has >> sp & 1u;
            if (hl && hr) set(sp - 1, __dadd_rn(get(sp - 1), get(sp)));
            else if (hr) { set(sp - 1, get(sp)); has |= 1u << (sp - 1); }
        }
    }
    return stk[0];
}

/* AndMaybePostList::get_weight (matcher/andmaybepostlist.cc:59-67): the right side's weight, i.e. the
 * OrPostList tree over the optional leaves that hold docid d.  *present = how many leaves matched. */
__device__ __noinline__ double maybe_weight(const XgmKernelParams& p, const XgmDevQuery* q, uint32_t d, uint32_t dlen,
                                            uint32_t* present) {
    /* wdf is declared here, not in the lambda, so that it follows the fold's stack in the frame: with the other
     * order ptxas gives xgm_and_bm3_kernel, which calls this function, a 176-byte frame and spills instead of 160 */
    uint32_t cnt = 0, wdf;
    const uint32_t base = q->nterms + q->nnot;
    const double w = or_tree_weight<XGM_DEV_MAX_TERMS>(q, [&](uint32_t op, double& v) {
        const XgmDevTerm& t = q->terms[base + op];
        wdf = 0;
        if (!lookup_posting(p, t, d, &wdf)) return false;
        v = bm25_sumpart(t.termweight, q, wdf, dlen);
        ++cnt;
        return true;
    });
    *present = cnt;
    return cnt ? w : 0.0;
}

/* ------------------------------------------------------------------ sparse AND kernel */

struct __align__(16) AndScratch {
    WarpScratch w;
    uint32_t dstage[2][STAGE_WORDS];  /* double-buffered packed docids of the driver list */
    uint64_t dbar[2];                 /* completion barriers of `dstage` */
};

/* The planner sends every AND whose lists but the driver all have bitmaps to xgm_and_bm3_kernel: here some list
 * has none, or the query has a single term. */
__global__ void __launch_bounds__(MATCH_WARPS * 32, 3) xgm_and_kernel(const __grid_constant__ XgmKernelParams p) {
    __shared__ AndScratch scratch[MATCH_WARPS];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    AndScratch& as = scratch[warp];
    WarpScratch& ws = as.w;
    if (lane == 0) { mbar_init(&ws.bar, 1); mbar_init(&as.dbar[0], 1); mbar_init(&as.dbar[1], 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    uint32_t phase = 0, dphase0 = 0, dphase1 = 0;
    const XgmBlockHdr* __restrict__ hdr = p.hdr;

    if (nothing_to_rerun(p)) return;
    uint32_t item;
    while (claim_item(p, XGM_WC_AND, p.nitems, lane, item)) {
        const XgmWorkItem wi = p.items[item];
        if (!runs_this_pass(p, wi.query)) continue;
        const XgmDevQuery* q = &p.queries[wi.query];
        const uint32_t nterms = q->nterms, nnot = q->nnot, nweighted = q->nweighted;
        /* lane j keeps list j's skip-table cursor (required lists, then the excluded ones of an OP_AND_NOT) */
        uint32_t my_begin = 0, my_nblk = 0, my_cur = 0;
        if (lane < nterms + nnot) {
            my_begin = q->terms[lane].blk_begin;
            my_nblk = q->terms[lane].nblocks;
        }
        const uint32_t drv_begin = __shfl_sync(FULL, my_begin, 0);
        const double tw0 = q->terms[0].termweight;

        /* software pipeline over the driver list: block db+1 is in flight while db is intersected */
        XgmBlockHdr dh = hdr[drv_begin + wi.b0];
        __syncwarp();
        issue_stage(p.docs, dh.doc_off, XGM_HDR_DOC_BITS(dh.meta), as.dstage[0], &as.dbar[0], lane);
        uint32_t buf = 0;
        for (uint32_t db = wi.b0; db < wi.b1; ++db) {
            XgmBlockHdr nh = dh;
            if (db + 1 < wi.b1) {
                nh = hdr[drv_begin + db + 1];
                __syncwarp();
                issue_stage(p.docs, nh.doc_off, XGM_HDR_DOC_BITS(nh.meta), as.dstage[buf ^ 1], &as.dbar[buf ^ 1], lane);
            }
            const uint32_t dbits = XGM_HDR_DOC_BITS(dh.meta);
            if (dbits) {
                if (buf == 0) { mbar_wait(&as.dbar[0], dphase0); dphase0 ^= 1u; }
                else { mbar_wait(&as.dbar[1], dphase1); dphase1 ^= 1u; }
            }
            const uint32_t dcount = XGM_HDR_COUNT(dh.meta);
            uint32_t c[4];
            decode_docids(as.dstage[buf], dbits, dh.first, lane, c);
            uint32_t alive = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (4 * lane + k < dcount) alive |= 1u << k;

            double acc[4] = {0.0, 0.0, 0.0, 0.0};
            uint32_t dl[4] = {0, 0, 0, 0};

            if (nterms == 1) {
                /* single term: every posting matches; decode the wdf block too */
                stage_block(p.tfs, dh.tf_off, XGM_HDR_TF_BITS(dh.meta), ws.stage, &ws.bar, phase, lane);
                const uint32_t tb = XGM_HDR_TF_BITS(dh.meta);
                const uint32_t tmask = bitmask(tb);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (alive >> k & 1u) {
                        uint32_t tf = tb ? unpack_sm(ws.stage, 4 * lane + k, tb, tmask) : 0u;
                        dl[k] = __ldg(&p.doclen[c[k]]);
                        acc[k] = (q->unweighted & 1u) ? 0.0 : bm25_sumpart(tw0, q, tf, dl[k]);
                        if (q->src_pos == 0) acc[k] = __dadd_rn(q->src_weight, acc[k]);
                        else if (q->src_pos == 1) acc[k] = __dadd_rn(acc[k], q->src_weight);
                    }
                }
                __syncwarp();
            }

            for (uint32_t j = 1; j < nterms; ++j) {
                if (!__any_sync(FULL, alive != 0)) break;
                const uint32_t lbegin = __shfl_sync(FULL, my_begin, j);
                const double twj = q->terms[j].termweight;
                auto on_hit = [&](int k, uint32_t pos, const XgmBlockHdr& bh) {
                    if (j == 1) {
                        /* first confirmation: fetch doclen and the driver's own wdf lazily */
                        dl[k] = __ldg(&p.doclen[c[k]]);
                        acc[k] = 0.0;
                        if (!(q->unweighted & 1u)) {
                            uint32_t tf0 = unpack_gl(p.tfs, dh.tf_off, 4 * lane + k, XGM_HDR_TF_BITS(dh.meta));
                            acc[k] = bm25_sumpart(tw0, q, tf0, dl[k]);
                        }
                        if (q->src_pos == 0) acc[k] = __dadd_rn(q->src_weight, acc[k]);
                    }
                    if (q->src_pos == j) acc[k] = __dadd_rn(acc[k], q->src_weight);
                    /* MultiAndPostList::get_weight: result += plist[i]->get_weight(), in plist order */
                    if (!(q->unweighted >> j & 1u)) {
                        uint32_t tfj = unpack_gl(p.tfs, bh.tf_off, pos, XGM_HDR_TF_BITS(bh.meta));
                        acc[k] = __dadd_rn(acc[k], bm25_sumpart(twj, q, tfj, dl[k]));
                    }
                    if (j + 1 == nterms && q->src_pos == nterms) acc[k] = __dadd_rn(acc[k], q->src_weight);
                };
                const uint64_t bm_off = q->terms[j].bm_off;
                if (bm_off != XGM_NO_BITMAP) {
                    /* membership bitmap: the skip_to/check of the leapfrog is one word load per candidate,
                     * all four of a lane (and all 128 of the warp) in flight together */
                    const uint32_t* __restrict__ bm = p.bitmaps + bm_off;
                    uint32_t w[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) w[k] = (alive >> k & 1u) ? __ldg(bm + (c[k] >> 5)) : 0u;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        if (alive >> k & 1u) {
                            if (w[k] >> (c[k] & 31) & 1u) {
                                const uint32_t r = bitmap_rank(p, q->terms[j], c[k]);
                                on_hit(k, r & 127u, hdr[lbegin + (r >> 7)]);
                            } else {
                                alive &= ~(1u << k);
                            }
                        }
                    }
                } else {
                    const uint32_t lnblk = __shfl_sync(FULL, my_nblk, j);
                    uint32_t cur = __shfl_sync(FULL, my_cur, j);
                    cur = probe_list(p, hdr + lbegin, lnblk, cur, ws, phase, lane, c, alive, on_hit,
                                     [&](int k) { alive &= ~(1u << k); });
                    if (lane == j) my_cur = cur;
                }
            }

            /* right side of an OP_AND_NOT: a candidate found in any of these lists is dropped */
            for (uint32_t j = nterms; j < nterms + nnot; ++j) {
                if (!__any_sync(FULL, alive != 0)) break;
                const uint64_t bm_off = q->terms[j].bm_off;
                if (bm_off != XGM_NO_BITMAP) {
                    const uint32_t* __restrict__ bm = p.bitmaps + bm_off;
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if ((alive >> k & 1u) && ((__ldg(bm + (c[k] >> 5)) >> (c[k] & 31)) & 1u)) alive &= ~(1u << k);
                } else {
                    const uint32_t lbegin = __shfl_sync(FULL, my_begin, j);
                    const uint32_t lnblk = __shfl_sync(FULL, my_nblk, j);
                    uint32_t cur = __shfl_sync(FULL, my_cur, j);
                    cur = probe_list(p, hdr + lbegin, lnblk, cur, ws, phase, lane, c, alive,
                                     [&](int k, uint32_t, const XgmBlockHdr&) { alive &= ~(1u << k); }, [&](int) {});
                    if (lane == j) my_cur = cur;
                }
            }
            /* value-slot filter (OP_FILTER with a range source), applied to the survivors */
            if (q->filter) {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if ((alive >> k & 1u) && !doc_passes_filter(p, q, c[k])) alive &= ~(1u << k);
            }
            uint32_t aux[4] = {nweighted, nweighted, nweighted, nweighted};
            if (q->nmaybe) { /* OP_AND_MAYBE: res = l; if (r matches) res += r */
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (alive >> k & 1u) {
                        uint32_t opt = 0;
                        const double rw = maybe_weight(p, q, c[k], dl[k], &opt);
                        if (opt) acc[k] = __dadd_rn(acc[k], rw);
                        aux[k] += opt;
                    }
                }
            }
            count_matches(p, wi.query, __popc(alive), lane);
#pragma unroll
            for (int k = 0; k < 4; ++k) emit_match_lanes(p, lane, alive >> k & 1u, wi.query, acc[k], c[k], aux[k], false);
            dh = nh;
            buf ^= 1u;
        }
    }
}


/* ------------------------------------------------------------------ bitmap AND kernel */

/* AND of a driver list with lists that all have membership bitmaps — the common case once HBM is used
 * for bitmaps of the frequent terms.  Warp-autonomous like xgm_and_kernel, but stripped to the fast
 * path so that more warps fit an SM (the kernel is bound by the latency of the bitmap probes): a warp
 * decodes TWO driver blocks at a time (bulk copies of the next pair already in flight) and issues the 8
 * bitmap word loads of every lane together.  Of the driver postings ~1 % pass the second list's bitmap
 * and ~0.01 % are matches, so the rare work is queued: a warp keeps two queues in shared memory for its
 * whole lifetime, entries tagged with their query:
 *   stage 1  candidates confirmed by the second list       → flushed 32 at a time: remaining bitmaps
 *            (required / excluded lists), value-range predicate; the survivors — the matches — go to
 *   stage 2  matches                                       → flushed 32 at a time: rank → wdf, doc length,
 *            BM25 in MultiAndPostList order (multiandpostlist.cc:149-159), per-lane emission.
 * Both are only drained when the warp runs out of work, so every flush but the last runs on a full warp.
 * Stage-1 slots come from four ballots per iteration (lanes with a survivor + the bits of their count)
 * instead of one ballot per posting slot. */
#define BM3_WARPS 8
#define BM3_Q1CAP 288 /* < 32 left over + up to 256 new candidates per iteration */
#define BM3_Q2CAP 64

struct __align__(16) Bm3Scratch {
    uint32_t dstage[4][STAGE_WORDS]; /* packed driver blocks (bulk copies), then their decoded docids */
    uint32_t q1did[BM3_Q1CAP]; /* stage 1 belongs to the current work item (one run of queries) */
    uint16_t q1src[BM3_Q1CAP]; /* query slot << 12 | (driver block - b0) << 7 | position (b1 - b0 <= 32) */
    uint32_t q2did[BM3_Q2CAP]; /* stage 2 lives as long as the warp: entries carry their query */
    uint32_t q2src[BM3_Q2CAP]; /* index of the driver block's header in hdr[] */
    uint32_t q2qi[BM3_Q2CAP];  /* query | position in the driver block << 25 */
    uint64_t dbar[4];
};
static_assert(XGM_BM_RUN <= 16, "q1src keeps a query slot in 4 bits");
/* 4.6 KB per warp, 37 KB per CTA: with 4 CTAs per SM the shared-memory carve-out stays at 164 KB and the
 * bitmap probes keep ~90 KB of L1 (51 KB per CTA would push the carve-out to 228 KB and leave the probes
 * almost no L1). */

/* One flat loop with five states, so that each piece of code exists once and nothing is called from the hot
 * path: score 32 matches (stage 2 full, or out of work) → finish 32 candidates (stage 1 full, or the item
 * ended) → fetch the next work item → probe the decoded pair of driver blocks for the next query slot of the
 * item's run → decode the next pair.  A pair is decoded once and probed once per query of the run. */
__global__ void __launch_bounds__(BM3_WARPS * 32, 4) xgm_and_bm3_kernel(const __grid_constant__ XgmKernelParams p) {
    extern __shared__ __align__(16) unsigned char bm3_raw[];
    Bm3Scratch* scratch = reinterpret_cast<Bm3Scratch*>(bm3_raw);
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    Bm3Scratch& ws = scratch[warp];
    if (lane < 4) mbar_init(&ws.dbar[lane], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    uint32_t phases = 0; /* bits 0-3: mbarrier phase of each buffer; bits 8-16: the decoded pair's alive bits (below) */
    const XgmBlockHdr* __restrict__ hdr = p.hdr;
    const uint32_t stage_base = smem_u32(ws.dstage[0]);
    const uint32_t bar_base = stage_base + (uint32_t)offsetof(Bm3Scratch, dbar);
    if (nothing_to_rerun(p)) return;
    const uint32_t nitems_bm = p.nitems_bm_dev ? __ldg(p.nitems_bm_dev) : p.nitems_bm;
    uint32_t qn1 = 0, qn2 = 0; /* warp-uniform queue lengths */
    bool done = false;
    /* current work item: its driver blocks are hdr[drv + i], i < it_n; those from db on are left to decode */
    uint32_t drv = 0, it_n = 0, db = 0, cur = 0;
    /* the item's run: lane s holds the query of slot s and the offset of its probe bitmap (terms[1]), or'ed with 1 when
     * the query probes through the coarse bitmap first (bm_off is a multiple of 8, its low three bits are free).  run_bits: low
     * half, a bit per slot that takes part (in the second pass only the queries that re-run); high half, the slots
     * still to probe on the decoded pair, which sits in buffers cur ^ 2, cur ^ 2 + 1 */
    uint32_t slot_q = 0, run_bits = 0;
    uint64_t slot_bm = 0;
    uint2 h0 = make_uint2(0u, 0u), h1 = h0; /* (first docid, meta) of the staged pair */

    /* stage driver block blk into buffer b; only (first docid, meta) of its header stay live */
    auto issue = [&](uint32_t b, uint32_t blk) {
        const uint4 h = __ldg(reinterpret_cast<const uint4*>(hdr + drv + blk));
        const uint32_t bits = XGM_HDR_DOC_BITS(h.w);
        __syncwarp();
        if (bits != 0 && lane == 0) {
            mbar_expect_tx_a(bar_base + b * 8u, bits * 16u);
            bulk_g2s_a(stage_base + b * (STAGE_WORDS * 4u), p.docs + h.y, bits * 16u, bar_base + b * 8u);
        }
        return make_uint2(h.x, h.w);
    };

    for (;;) {
        /* ---- stage 2: score queued matches (one per lane) and emit them ---- */
        if (qn2 >= 32 || (done && qn2 != 0)) {
            const uint32_t count = min(qn2, 32u);
            qn2 -= count;
            const bool alive = lane < count;
            const uint32_t d = alive ? ws.q2did[qn2 + lane] : 0u;
            const uint32_t src = alive ? ws.q2src[qn2 + lane] : 0u;
            const uint32_t qp = alive ? ws.q2qi[qn2 + lane] : 0u;
            const uint32_t qi = qp & 0x1ffffffu, pos = qp >> 25;
            double acc = 0.0;
            uint32_t aux = 0;
            if (alive) {
                const XgmDevQuery* mq = &p.queries[qi];
                const uint32_t dlen = __ldg(&p.doclen[d]);
                const XgmBlockHdr hh = hdr[src];
                const uint32_t nterms = mq->nterms, sp = mq->src_pos, unw = mq->unweighted;
                /* MultiAndPostList::get_weight: result += plist[i]->get_weight(), in plist order
                 * (multiandpostlist.cc:149-159); a weighted range source is the child at position src_pos */
                if (sp == 0) acc = mq->src_weight;
                if (!(unw & 1u))
                    acc = __dadd_rn(acc, bm25_sumpart(mq->terms[0].termweight, mq, unpack_gl(p.tfs, hh.tf_off, pos, XGM_HDR_TF_BITS(hh.meta)), dlen));
                for (uint32_t j = 1; j < nterms; ++j) {
                    if (sp == j) acc = __dadd_rn(acc, mq->src_weight);
                    if (unw >> j & 1u) continue;
                    const uint32_t r = bitmap_rank(p, mq->terms[j], d);
                    const XgmBlockHdr bh = hdr[mq->terms[j].blk_begin + (r >> 7)];
                    const uint32_t tfj = unpack_gl(p.tfs, bh.tf_off, r & 127u, XGM_HDR_TF_BITS(bh.meta));
                    acc = __dadd_rn(acc, bm25_sumpart(mq->terms[j].termweight, mq, tfj, dlen));
                }
                if (sp == nterms) acc = __dadd_rn(acc, mq->src_weight);
                uint32_t opt = 0;
                if (mq->nmaybe) { /* OP_AND_MAYBE: res = l; if (r matches) res += r */
                    const double rw = maybe_weight(p, mq, d, dlen, &opt);
                    if (opt) acc = __dadd_rn(acc, rw);
                }
                aux = mq->nweighted + opt;
            }
            emit_match_lanes(p, lane, alive, qi, acc, d, aux);
            __syncwarp();
            continue;
        }
        const bool item_end = db >= it_n && (run_bits >> 16) == 0;
        /* ---- stage 1: finish the boolean test of queued candidates of the current item ---- */
        if (qn1 >= 32 || (item_end && qn1 != 0)) {
            __syncwarp();
            const uint32_t count = min(qn1, 32u);
            qn1 -= count;
            bool alive = lane < count;
            const uint32_t d = alive ? ws.q1did[qn1 + lane] : 0u;
            const uint32_t src = alive ? ws.q1src[qn1 + lane] : 0u;
            /* the lanes' candidates belong to different queries of the run */
            const uint32_t qi = __shfl_sync(FULL, slot_q, src >> 12);
            const XgmDevQuery* q = &p.queries[qi];
            const uint32_t nterms = q->nterms, nall = nterms + q->nnot;
            for (uint32_t j = 2; __any_sync(FULL, alive && j < nall); ++j) {
                if (alive && j < nall) {
                    const uint32_t w = __ldg(p.bitmaps + q->terms[j].bm_off + (d >> 5));
                    /* required lists must hold the docid; the right side of an OP_AND_NOT must not
                     * (AndNotPostList::next, matcher/andnotpostlist.cc:97-130) */
                    if (((w >> (d & 31)) & 1u) == (j < nterms ? 0u : 1u)) alive = false;
                }
            }
            if (alive && q->filter && !doc_passes_filter(p, q, d)) alive = false;
            const uint32_t m = __ballot_sync(FULL, alive);
            if (alive) {
                const uint32_t slot = qn2 + __popc(m & ((1u << lane) - 1u));
                ws.q2did[slot] = d;
                ws.q2src[slot] = drv + ((src >> 7) & 31u);
                ws.q2qi[slot] = qi | ((src & 127u) << 25);
            }
            qn2 += __popc(m);
            __syncwarp();
            continue;
        }
        if (done) break;
        /* ---- next work item ---- */
        if (item_end) {
            uint32_t item;
            if (!claim_item(p, XGM_WC_AND_BM, nitems_bm, lane, item)) { done = true; continue; }
            const XgmWorkItem wi = p.items_bm[item];
            const uint32_t n = p.bm_segs ? wi.pad : 1u;
            slot_q = lane >= n ? 0u : p.bm_segs ? p.bm_segs[wi.query + lane].query : wi.query;
            const bool take = lane < n && runs_this_pass(p, slot_q);
            run_bits = __ballot_sync(FULL, take);
            if (run_bits == 0) continue; /* second pass: no query of the run re-runs */
            slot_bm = take ? p.queries[slot_q].terms[1].bm_off | p.queries[slot_q].probe_coarse : 0ull;
            drv = p.queries[__shfl_sync(FULL, slot_q, 0)].terms[0].blk_begin + wi.b0;
            it_n = wi.b1 - wi.b0;
            db = 0;
            /* buffers 0 and 1 may hold the last item's pair, read by the generic proxy; the bulk copies refill them */
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            h0 = issue(0, 0);
            h1 = h0;
            if (it_n > 1) h1 = issue(1, 1);
            cur = 0; /* buffers cur, cur+1 hold the current pair; (cur^2), (cur^2)+1 the next */
            continue;
        }
        /* ---- probe the decoded pair for one query slot of the run ---- */
        if ((run_bits >> 16) != 0) {
            const uint32_t s = (uint32_t)__ffs(run_bits >> 16) - 1u;
            run_bits ^= 1u << (16 + s);
            const uint64_t sbm = __shfl_sync(FULL, slot_bm, s);
            const uint32_t* __restrict__ bm1 = p.bitmaps + (sbm & ~7ull);
            const uint32_t pb = cur ^ 2u;
            /* slot k of lane l: posting 32 (k & 3) + l of block k >> 2, as the decode step left it */
#define BM3_POSTING(k) ws.dstage[pb + ((k) >> 2)][32 * ((k) & 3) + lane]
            /* the skip_to/check of the leapfrog: one bitmap word per candidate, all loads issued together */
            uint32_t w[8];
            /* phases >> 8, bit k: this lane's slot k holds a posting; bit 8: both blocks are full (warp-uniform).  live,
             * bit k: slot k is to be tested against the fine bitmap */
            uint32_t live = (phases >> 8) & 0xffu;
            if (sbm & 1u) {
                /* sparse probe list: first the coarse words (a 32-byte sector spans 2048 docids, not 256), then the fine
                 * word only where the posting's 8-docid group holds a member.  The postings are read from shared memory
                 * in each phase (the memory clobber keeps them there), so the coarse round trip holds no more registers
                 * than the fine one: held across it they spill. */
#pragma unroll
                for (int k = 0; k < 8; ++k) w[k] = (live >> k & 1u) ? __ldg(p.coarse + (sbm >> 3) + (BM3_POSTING(k) >> 8)) : 0u;
                live = 0;
#pragma unroll
                for (int k = 0; k < 8; ++k) live |= (__funnelshift_r(w[k], 0u, BM3_POSTING(k) >> 3) & 1u) << k;
                asm volatile("" ::: "memory");
            }
            uint32_t c[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) c[k] = BM3_POSTING(k);
#undef BM3_POSTING
            if ((phases >> 16) && !(sbm & 1u)) { /* two full blocks: no per-posting predicates */
#pragma unroll
                for (int k = 0; k < 8; ++k) w[k] = __ldg(bm1 + (c[k] >> 5));
            } else {
#pragma unroll
                for (int k = 0; k < 8; ++k) w[k] = (live >> k & 1u) ? __ldg(bm1 + (c[k] >> 5)) : 0u;
            }
            uint32_t surv = 0; /* dead slots carry w = 0 */
#pragma unroll
            for (int k = 0; k < 8; ++k) surv |= (__funnelshift_r(w[k], 0u, c[k]) & 1u) << k; /* shifts by c & 31 */
            /* Queue slots without a scan: survivors are rare, so a lane's count n is 1..8 in the few lanes that
             * have one; four ballots (lanes with survivors, and the three bits of n - 1) give every lane the
             * number of survivors in the lanes below it. */
            const uint32_t B = __ballot_sync(FULL, surv != 0);
            if (B) {
                const uint32_t nm1 = (uint32_t)__popc(surv) - 1u;
                const uint32_t B0 = __ballot_sync(FULL, surv != 0 && (nm1 & 1u));
                const uint32_t B1 = __ballot_sync(FULL, surv != 0 && (nm1 & 2u));
                const uint32_t B2 = __ballot_sync(FULL, surv != 0 && (nm1 & 4u));
                if (surv) {
                    const uint32_t lt = (1u << lane) - 1u;
                    uint32_t slot = qn1 + __popc(B & lt) + __popc(B0 & lt) + 2u * __popc(B1 & lt) + 4u * __popc(B2 & lt);
                    const uint32_t rb = s << 12 | (db - 2u) << 7 | lane; /* db has moved on to the next pair */
#pragma unroll
                    for (int k = 0; k < 8; ++k)
                        if (surv >> k & 1u) {
                            ws.q1did[slot] = c[k];
                            ws.q1src[slot] = (uint16_t)(rb + ((k >> 2) << 7) + ((k & 3) << 5));
                            ++slot;
                        }
                }
                qn1 += __popc(B) + __popc(B0) + 2u * __popc(B1) + 4u * __popc(B2);
            }
            continue;
        }
        /* ---- decode the next pair of driver blocks ---- */
        {
            const bool two = db + 1 < it_n;
            /* the probes read buffers cur ^ 2 through the generic proxy; the bulk copies below refill them */
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            uint2 n0 = h0, n1 = h1;
            if (db + 2 < it_n) n0 = issue(cur ^ 2, db + 2);
            if (db + 3 < it_n) n1 = issue((cur ^ 2) + 1, db + 3);
            uint32_t c[8];
            const uint32_t cnt0 = XGM_HDR_COUNT(h0.y), cnt1 = two ? XGM_HDR_COUNT(h1.y) : 0u;
            {
                const uint32_t bits = XGM_HDR_DOC_BITS(h0.y);
                if (bits) { mbar_wait_a(bar_base + cur * 8u, (phases >> cur) & 1u); phases ^= 1u << cur; }
                decode_docids(ws.dstage[cur], bits, h0.x, lane, c);
            }
            if (two) {
                const uint32_t bits = XGM_HDR_DOC_BITS(h1.y);
                if (bits) { mbar_wait_a(bar_base + (cur + 1) * 8u, (phases >> (cur + 1)) & 1u); phases ^= 1u << (cur + 1); }
                decode_docids(ws.dstage[cur + 1], bits, h1.x, lane, c + 4);
            } else {
                c[4] = c[5] = c[6] = c[7] = 0u;
            }
            /* Interleave the postings across the lanes, through the staging buffers they were decoded from: the
             * probe step reads slot k of lane l as posting 32 (k & 3) + l of block k >> 2.  decode_docids leaves a
             * lane postings 4l..4l+3, at C2's driver density ~85 bytes of bitmap from its neighbour's, so each probe
             * load would touch ~21 cache lines per warp; interleaved, its 32 lanes are 32 consecutive postings.  (An
             * absent second block transposes its zeros.)  The buffers are not refilled before every slot of the run
             * has probed them: the next pair's decode issues into the other two. */
            __syncwarp();
            reinterpret_cast<uint4*>(ws.dstage[cur])[lane] = make_uint4(c[0], c[1], c[2], c[3]);
            reinterpret_cast<uint4*>(ws.dstage[cur + 1])[lane] = make_uint4(c[4], c[5], c[6], c[7]);
            __syncwarp();
            phases &= 0xffu;
            if (cnt0 + cnt1 == 2u * XGM_BLOCK) {
                phases |= 0x1ffu << 8;
            } else {
                /* slot k < 4 holds posting 32k + lane of the first block: the lane has (cnt + 31 - lane) / 32 of
                 * each block's cnt postings (cnt <= 128, and 0 of an absent second block) */
                const uint32_t m0 = (cnt0 + 31u - lane) >> 5, m1 = (cnt1 + 31u - lane) >> 5;
                phases |= (((1u << m0) - 1u) | (((1u << m1) - 1u) << 4)) << 8;
            }
            run_bits = (run_bits & 0xffffu) * 0x10001u; /* every slot probes the pair */
            h0 = n0;
            h1 = n1;
            cur ^= 2u;
            db += 2;
        }
    }
}

cudaError_t xgm_launch_and_bm(const XgmKernelParams& p, int grid, cudaStream_t s) {
    xgm_and_bm3_kernel<<<grid, BM3_WARPS * 32, sizeof(Bm3Scratch) * BM3_WARPS, s>>>(p);
    return cudaGetLastError();
}

/* Also opts the kernel in to its dynamic shared memory on the CURRENT device (the attribute is per device:
 * call once per searcher, after cudaSetDevice). */
int xgm_and_bm_occupancy_blocks_per_sm() {
    int n = 0;
    const size_t smem = sizeof(Bm3Scratch) * BM3_WARPS;
    cudaFuncSetAttribute(xgm_and_bm3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, xgm_and_bm3_kernel, BM3_WARPS * 32, smem);
    return n;
}

/* ------------------------------------------------------------------ OR kernel */

#define OR_WARPS 4

struct __align__(16) OrScratch {
    WarpScratch w;
    uint32_t tft[XGM_DEV_MAX_TERMS][XGM_BLOCK]; /* wdf of candidate x in leaf i, for leaves probed by decoding */
};

/* OR of leaves (OrPostList tree, orpostlist.cc:93-204).  Each document of the union is produced exactly
 * once, by the rarest leaf that contains it ("owner"): work items walk one leaf's blocks, test the other
 * leaves for the same 128 docids (membership bitmap when the leaf has one, galloping block decode
 * otherwise), drop documents owned by a rarer leaf, and evaluate the reference's tree-shaped sum (l, r
 * or l+r per node, queryinternal.cc:440-489) for the rest.
 * MaxScore pruning, the parallel form of OrPostList's w_min checks (orpostlist.cc:113-155): a document
 * whose present leaves cannot add up to the current top-k threshold (sum of their get_maxpart bounds
 * falls in a bucket below b*) is counted as a match but neither scored nor stored. */
__global__ void __launch_bounds__(OR_WARPS * 32) xgm_or_kernel(const __grid_constant__ XgmKernelParams p) {
    __shared__ OrScratch scratch[OR_WARPS];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    OrScratch& os = scratch[warp];
    WarpScratch& ws = os.w;
    if (lane == 0) mbar_init(&ws.bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    uint32_t phase = 0;
    const XgmBlockHdr* __restrict__ hdr = p.hdr;

    if (nothing_to_rerun(p)) return;
    uint32_t item;
    while (claim_item(p, XGM_WC_OR, p.nitems_or, lane, item)) {
        const XgmWorkItem wi = p.items_or[item];
        if (!runs_this_pass(p, wi.query)) continue;
        const XgmDevQuery* q = &p.queries[wi.query];
        if (q->or_fast != XGM_OR_FAST_GENERAL) continue; /* answered by xgm_or3_kernel */
        const uint32_t nterms = q->nterms;
        const uint32_t drv = wi.pad; /* driver leaf (position in ascending-termfreq order) */
        uint32_t my_begin = 0, my_nblk = 0, my_cur = 0;
        if (lane < nterms) {
            my_begin = q->terms[lane].blk_begin;
            my_nblk = q->terms[lane].nblocks;
        }
        const uint32_t drv_begin = __shfl_sync(FULL, my_begin, drv);
        const bool can_prune = prunes_by_weight(q);
        if (can_prune && skip_owned_item(p, q, wi.query, drv, lane)) continue;

        for (uint32_t db = wi.b0; db < wi.b1; ++db) {
            const XgmBlockHdr dh = hdr[drv_begin + db];
            const uint32_t dcount = XGM_HDR_COUNT(dh.meta);
            uint32_t c[4];
            stage_block(p.docs, dh.doc_off, XGM_HDR_DOC_BITS(dh.meta), ws.stage, &ws.bar, phase, lane);
            decode_docids(ws.stage, XGM_HDR_DOC_BITS(dh.meta), dh.first, lane, c);
            uint32_t owned = 0;
            uint32_t present[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                present[k] = 1u << drv;
                if (4 * lane + k < dcount) owned |= 1u << k;
            }
            __syncwarp();
            for (uint32_t j = 0; j < nterms; ++j) {
                if (j == drv) continue;
                if (!__any_sync(FULL, owned != 0)) break;
                const uint64_t bm_off = q->terms[j].bm_off;
                if (bm_off != XGM_NO_BITMAP) {
                    const uint32_t* __restrict__ bm = p.bitmaps + bm_off;
                    uint32_t w[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) w[k] = (owned >> k & 1u) ? __ldg(bm + (c[k] >> 5)) : 0u;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        if ((owned >> k & 1u) && (w[k] >> (c[k] & 31) & 1u)) {
                            if (j < drv) owned &= ~(1u << k); /* a rarer leaf owns this document */
                            else present[k] |= 1u << j;
                        }
                    }
                } else {
                    const uint32_t lbegin = __shfl_sync(FULL, my_begin, j);
                    const uint32_t lnblk = __shfl_sync(FULL, my_nblk, j);
                    uint32_t cur = __shfl_sync(FULL, my_cur, j);
                    cur = probe_list(
                        p, hdr + lbegin, lnblk, cur, ws, phase, lane, c, owned,
                        [&](int k, uint32_t pos, const XgmBlockHdr& bh) {
                            if (j < drv) {
                                owned &= ~(1u << k);
                            } else {
                                os.tft[j][4 * lane + k] = unpack_gl(p.tfs, bh.tf_off, pos, XGM_HDR_TF_BITS(bh.meta));
                                present[k] |= 1u << j;
                            }
                        },
                        [&](int) {});
                    if (lane == j) my_cur = cur;
                }
            }
            if (q->filter) {
#pragma unroll
                for (int k = 0; k < 4; ++k)
                    if ((owned >> k & 1u) && !doc_passes_filter(p, q, c[k])) owned &= ~(1u << k);
            }
            if (q->or_nreq | q->nnot) {
                /* OP_FILTER's boolean terms / OP_AND_NOT's excluded terms above the OR: a document of the union
                 * that fails them is not a match at all (neither counted nor scored) */
                const uint32_t nreq = q->or_nreq, nnot = q->nnot;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if (!(owned >> k & 1u)) continue;
                    bool keep = true;
                    uint32_t wdf_unused;
                    for (uint32_t i = 0; i < nreq && keep; ++i) keep = lookup_posting(p, q->terms[nterms + i], c[k], &wdf_unused);
                    for (uint32_t i = 0; i < nnot && keep; ++i) keep = !lookup_posting(p, q->terms[nterms + nreq + i], c[k], &wdf_unused);
                    if (!keep) owned &= ~(1u << k);
                }
            }
            /* MaxScore: can the leaves present reach the current threshold at all? */
            uint32_t skip = 0;
            if (can_prune) {
                const uint32_t bstar = live_bstar(&p.qstate[wi.query]);
                if (bstar != 0) {
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if ((owned >> k & 1u) && bound_bucket(q, maxpart_sum(q, present[k], 0.0)) < bstar) skip |= 1u << k;
                }
            }
            /* weight = fold of the tree over the leaves present (OrPostList::get_weight, orpostlist.cc:93-103) */
            double acc[4] = {0.0, 0.0, 0.0, 0.0};
            uint32_t aux[4] = {0, 0, 0, 0};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if ((owned & ~skip) >> k & 1u) {
                    const uint32_t d = c[k];
                    const uint32_t dlen = __ldg(&p.doclen[d]);
                    acc[k] = or_tree_weight<XGM_DEV_MAX_TERMS>(q, [&](uint32_t op, double& v) {
                        if (!(present[k] >> op & 1u)) return false;
                        uint32_t tf;
                        if (op == drv) {
                            tf = unpack_gl(p.tfs, dh.tf_off, 4 * lane + k, XGM_HDR_TF_BITS(dh.meta));
                        } else if (q->terms[op].bm_off != XGM_NO_BITMAP) {
                            const uint32_t r = bitmap_rank(p, q->terms[op], d);
                            const XgmBlockHdr bh = hdr[q->terms[op].blk_begin + (r >> 7)];
                            tf = unpack_gl(p.tfs, bh.tf_off, r & 127u, XGM_HDR_TF_BITS(bh.meta));
                        } else {
                            tf = os.tft[op][4 * lane + k];
                        }
                        v = bm25_sumpart(q->terms[op].termweight, q, tf, dlen);
                        return true;
                    });
                    aux[k] = __popc(present[k]);
                }
            }
            /* the documents MaxScore skipped are matches too: counted, never scored or stored */
            count_matches(p, wi.query, __popc(owned), lane);
#pragma unroll
            for (int k = 0; k < 4; ++k)
                emit_match_lanes(p, lane, (owned & ~skip) >> k & 1u, wi.query, acc[k], c[k], aux[k], false);
            __syncwarp();
        }
    }
}

/* Weight of document d of an OR query of at most OR3_MAX_LEAVES leaves (presence mask pm over leaf positions): the
 * OrPostList tree fold (or_tree_weight) with its stack in registers.  The wdf of leaf `drv` (the owner, if any:
 * drv < nterms) comes from position pos of the block whose header is hdr[src]; every other leaf is looked up through
 * its rank directory. */
#define OR3_MAX_LEAVES 5
__device__ __forceinline__ double or_score_doc(const XgmKernelParams& p, const XgmDevQuery* mq, uint32_t d, uint32_t pm,
                                               uint32_t drv, uint32_t src, uint32_t pos) {
    const XgmBlockHdr* __restrict__ hdr = p.hdr;
    const uint32_t dlen = __ldg(&p.doclen[d]);
    return or_tree_weight<OR3_MAX_LEAVES>(mq, [&](uint32_t op, double& v) {
        if (!(pm >> op & 1u)) return false;
        uint32_t tf;
        if (op == drv) {
            const XgmBlockHdr hh = hdr[src];
            tf = unpack_gl(p.tfs, hh.tf_off, pos, XGM_HDR_TF_BITS(hh.meta));
        } else {
            const uint32_t r = bitmap_rank(p, mq->terms[op], d);
            const XgmBlockHdr bh = hdr[mq->terms[op].blk_begin + (r >> 7)];
            tf = unpack_gl(p.tfs, bh.tf_off, r & 127u, XGM_HDR_TF_BITS(bh.meta));
        }
        v = bm25_sumpart(mq->terms[op].termweight, mq, tf, dlen);
        return true;
    });
}

/* ------------------------------------------------------------------ OR kernel, bitmap leaves + queued scoring */

/* Same contract as xgm_or_kernel for queries whose leaves ALL have membership bitmaps and number at most five
 * (BASELINE config C3), organised like xgm_and_bm3_kernel.  Per iteration a warp decodes one block of the
 * owner leaf (bulk copies of the next blocks in flight), issues the bitmap probes of all other leaves for its
 * 128 docids together (up to 16 independent loads per lane) and builds every document's presence mask from the
 * bits.  Ownership (no rarer leaf holds the document) and MaxScore are then register work: the bound of a
 * presence mask comes from a 32-entry table held one entry per lane (one shuffle per posting).  Documents that
 * survive are queued with their presence mask and scored 32 at a time, one per lane: wdf of the owner from its
 * block, of the other leaves through their rank directories, then the reference's OrPostList tree as a postfix
 * program (orpostlist.cc:93-103).  The queue lives as long as the warp, so scoring always runs on full warps. */
#define OR3_WARPS 8
#define OR3_QCAP 160 /* < 32 left over + up to 128 new candidates per iteration */

struct __align__(16) Or3Scratch {
    uint32_t dstage[4][STAGE_WORDS];
    uint32_t qdid[OR3_QCAP];
    uint32_t qsrc[OR3_QCAP]; /* index of the owner block's header in hdr[] */
    uint32_t qqi[OR3_QCAP];  /* query | position in the block << 25 */
    uint32_t qpm[OR3_QCAP];  /* presence mask | owner leaf << 16 */
    uint64_t dbar[4];
};

/* PHASE 0: the whole union in one launch (queries with or_fast == XGM_OR_FAST_OR3).  PHASE 1: the documents holding
 * exactly ONE leaf of the queries whose documents with two or more leaves were already produced by
 * xgm_or_tile_kernel (or_fast == XGM_OR_FAST_TILE) — see there. */
template <int PHASE>
__global__ void __launch_bounds__(OR3_WARPS * 32, 3) xgm_or3_kernel(const __grid_constant__ XgmKernelParams p) {
    extern __shared__ __align__(16) unsigned char or3_raw[];
    Or3Scratch* scratch = reinterpret_cast<Or3Scratch*>(or3_raw);
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    Or3Scratch& ws = scratch[warp];
    if (lane < 4) mbar_init(&ws.dbar[lane], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    uint32_t phases = 0;
    const XgmBlockHdr* __restrict__ hdr = p.hdr;
    const uint32_t stage_base = smem_u32(ws.dstage[0]);
    const uint32_t bar_base = stage_base + (uint32_t)offsetof(Or3Scratch, dbar);
    if (nothing_to_rerun(p)) return;
    uint32_t qn = 0; /* warp-uniform queue length */
    bool done = false;
    /* current work item: blocks [db, it_b1) of leaf it_drv of query it_query are left */
    uint32_t it_query = 0, it_b1 = 0, db = 0, it_drv = 0, drv_begin = 0, nterms = 0;
    double others = 0.0, drv_tw = 0.0, drv_maxpart = 0.0;
    uint32_t total_acc = 0; /* documents this lane owns in the current item (exact match count) */
    bool can_prune = false;
    const XgmDevQuery* q = p.queries;
    const uint32_t* bmp[OR3_MAX_LEAVES];
#pragma unroll
    for (int j = 0; j < OR3_MAX_LEAVES; ++j) bmp[j] = p.bitmaps;

    auto issue = [&](uint32_t blk) { /* stage owner block blk into buffer blk & 3 */
        const uint32_t b = blk & 3u;
        const uint4 h = __ldg(reinterpret_cast<const uint4*>(hdr + drv_begin + blk));
        const uint32_t bits = XGM_HDR_DOC_BITS(h.w);
        __syncwarp();
        if (bits != 0 && lane == 0) {
            mbar_expect_tx_a(bar_base + b * 8u, bits * 16u);
            bulk_g2s_a(stage_base + b * (STAGE_WORDS * 4u), p.docs + h.y, bits * 16u, bar_base + b * 8u);
        }
    };

    for (;;) {
        /* ---- score queued documents (one per lane) and emit them ---- */
        if (qn >= 32 || (done && qn != 0)) {
            __syncwarp();
            const uint32_t count = min(qn, 32u);
            qn -= count;
            const bool alive = lane < count;
            const uint32_t d = alive ? ws.qdid[qn + lane] : 0u;
            const uint32_t src = alive ? ws.qsrc[qn + lane] : 0u;
            const uint32_t qp = alive ? ws.qqi[qn + lane] : 0u;
            const uint32_t pmd = alive ? ws.qpm[qn + lane] : 0u;
            const uint32_t qi = qp & 0x1ffffffu, pos = qp >> 25, pm = pmd & 0xffffu, drv = pmd >> 16;
            double acc = 0.0;
            bool score = alive;
            if (alive) {
                /* before the other leaves are looked up: the owner's exact weight plus the bounds of the others
                 * already decides most documents (MaxScore at its finest grain) */
                const XgmDevQuery* mq = &p.queries[qi];
                const uint32_t bstar = prunes_by_weight(mq) ? live_bstar(&p.qstate[qi]) : 0u;
                if (bstar != 0) {
                    const XgmBlockHdr hh = hdr[src];
                    const uint32_t tf = unpack_gl(p.tfs, hh.tf_off, pos, XGM_HDR_TF_BITS(hh.meta));
                    const double own = bm25_sumpart(mq->terms[drv].termweight, mq, tf, __ldg(&p.doclen[d]));
                    if (bound_bucket(mq, maxpart_sum(mq, pm & ~(1u << drv), own)) < bstar) score = false;
                }
            }
            if (score) acc = or_score_doc(p, &p.queries[qi], d, pm, drv, src, pos);
            emit_match_lanes(p, lane, score, qi, acc, d, (uint32_t)__popc(pm), false);
            __syncwarp();
            continue;
        }
        if (done) break;
        /* ---- next work item ---- */
        if (db >= it_b1) {
            if (total_acc || it_b1) { /* close the previous item: its owned documents are matches */
                count_matches(p, it_query, total_acc, lane);
                total_acc = 0; it_b1 = 0; db = 0;
            }
            uint32_t item;
            if (!claim_item(p, PHASE ? XGM_WC_OR3_SINGLE : XGM_WC_OR3, p.nitems_or, lane, item)) { done = true; continue; }
            const XgmWorkItem wi = p.items_or[item];
            if (!runs_this_pass(p, wi.query)) continue;
            q = &p.queries[wi.query];
            if (q->or_fast != (PHASE ? XGM_OR_FAST_TILE : XGM_OR_FAST_OR3)) continue; /* another kernel's query */
            nterms = q->nterms;
            it_drv = wi.pad;
            can_prune = prunes_by_weight(q);
            if (can_prune) {
                if (PHASE) {
                    /* only single-leaf documents are left: none of this leaf can reach the threshold */
                    const uint32_t bstar = live_bstar(&p.qstate[wi.query]);
                    if (bstar != 0 && bound_bucket(q, q->terms[it_drv].maxpart) < bstar) continue;
                } else if (skip_owned_item(p, q, wi.query, it_drv, lane)) {
                    continue;
                }
            }
            it_query = wi.query; it_b1 = wi.b1; db = wi.b0;
            drv_begin = q->terms[it_drv].blk_begin;
#pragma unroll
            for (int j = 0; j < OR3_MAX_LEAVES; ++j) bmp[j] = p.bitmaps + ((uint32_t)j < nterms ? q->terms[j].bm_off : 0ull);
            /* lane m holds, for presence mask m, the sum of the get_maxpart bounds of the leaves other than the
             * owner; the owner's own bound is per block (its largest wdf is in the header) */
            others = maxpart_sum(q, lane & ~(1u << it_drv), 0.0);
            drv_tw = q->terms[it_drv].termweight;
            drv_maxpart = q->terms[it_drv].maxpart;
            for (uint32_t b = db; b < it_b1 && b < db + 3; ++b) issue(b);
            continue;
        }
        /* ---- one block of the owner leaf ---- */
        {
            if (db + 3 < it_b1) issue(db + 3);
            const uint4 h = __ldg(reinterpret_cast<const uint4*>(hdr + drv_begin + db));
            const uint32_t bits = XGM_HDR_DOC_BITS(h.w), cnt = XGM_HDR_COUNT(h.w), cur = db & 3u;
            if (bits) { mbar_wait_a(bar_base + cur * 8u, (phases >> cur) & 1u); phases ^= 1u << cur; }
            if (PHASE) {
                /* a block whose best possible single-leaf document is below the threshold is skipped whole */
                const uint32_t bs = live_bstar(&p.qstate[it_query]);
                if (bs != 0 && bound_bucket(q, owner_block_bound(p, q, h.w, drv_tw, drv_maxpart)) < bs) { ++db; continue; }
            }
            uint32_t c[4];
            decode_docids(ws.dstage[cur], bits, h.x, lane, c);
            const int nv = min(4, max(0, (int)cnt - 4 * (int)lane));
            const uint32_t valid = (1u << nv) - 1u;
            uint32_t pm[4] = {0, 0, 0, 0};
            /* membership of the 128 docids in every other leaf: all probes issued before any is used */
#pragma unroll
            for (int j = 0; j < OR3_MAX_LEAVES; ++j) {
                if ((uint32_t)j < nterms && (uint32_t)j != it_drv) {
                    uint32_t w[4];
#pragma unroll
                    for (int k = 0; k < 4; ++k) w[k] = (valid >> k & 1u) ? __ldg(bmp[j] + (c[k] >> 5)) : 0u;
#pragma unroll
                    for (int k = 0; k < 4; ++k) pm[k] |= (__funnelshift_r(w[k], 0u, c[k]) & 1u) << j;
                }
            }
            const uint32_t rarer = (1u << it_drv) - 1u;
            const uint32_t bstar = can_prune ? live_bstar(&p.qstate[it_query]) : 0u;
            /* pruning bucket of every presence mask for THIS block: the owner's bound within the block plus the others' */
            uint32_t ubbkt = XGM_NBINS;
            if (bstar != 0) ubbkt = bound_bucket(q, owner_block_bound(p, q, h.w, drv_tw, drv_maxpart) + others);
            uint32_t cand = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const uint32_t m = pm[k] | (1u << it_drv);
                pm[k] = m;
                const uint32_t bk = __shfl_sync(FULL, ubbkt, m & 31u);
                bool own;
                if (PHASE) {
                    own = (valid >> k & 1u) && m == (1u << it_drv); /* no other leaf holds the document */
                } else {
                    own = (valid >> k & 1u) && (m & rarer) == 0u; /* a rarer leaf owns the document otherwise */
                    if (own && q->filter && !doc_passes_filter(p, q, c[k])) own = false;
                    total_acc += own ? 1u : 0u;
                }
                if (own && bk >= bstar) cand |= 1u << k;
            }
            const uint32_t B = __ballot_sync(FULL, cand != 0);
            if (B) {
                const uint32_t nm1 = (uint32_t)__popc(cand) - 1u;
                const uint32_t B0 = __ballot_sync(FULL, cand != 0 && (nm1 & 1u));
                const uint32_t B1 = __ballot_sync(FULL, cand != 0 && (nm1 & 2u));
                if (cand) {
                    const uint32_t lt = (1u << lane) - 1u;
                    uint32_t slot = qn + __popc(B & lt) + __popc(B0 & lt) + 2u * __popc(B1 & lt);
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        if (cand >> k & 1u) {
                            ws.qdid[slot] = c[k];
                            ws.qsrc[slot] = drv_begin + db;
                            ws.qqi[slot] = it_query | ((4 * lane + k) << 25);
                            ws.qpm[slot] = pm[k] | (it_drv << 16);
                            ++slot;
                        }
                }
                qn += __popc(B) + __popc(B0) + 2u * __popc(B1);
            }
            ++db;
        }
    }
    if (total_acc || it_b1) count_matches(p, it_query, total_acc, lane);
}

cudaError_t xgm_launch_or3(const XgmKernelParams& p, int grid, int phase, cudaStream_t s) {
    if (phase) xgm_or3_kernel<1><<<grid, OR3_WARPS * 32, sizeof(Or3Scratch) * OR3_WARPS, s>>>(p);
    else xgm_or3_kernel<0><<<grid, OR3_WARPS * 32, sizeof(Or3Scratch) * OR3_WARPS, s>>>(p);
    return cudaGetLastError();
}

/* also opts in to the dynamic shared memory on the current device (call once per searcher) */
int xgm_or3_occupancy_blocks_per_sm() {
    int n = 0;
    const size_t smem = sizeof(Or3Scratch) * OR3_WARPS;
    cudaFuncSetAttribute(xgm_or3_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaFuncSetAttribute(xgm_or3_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, xgm_or3_kernel<0>, OR3_WARPS * 32, smem);
    return n;
}

/* ------------------------------------------------------------------ OR by bitmap union (documents with >= 2 leaves) */

/* For an OR whose leaves all have membership bitmaps the union needs no posting list at all: word w of the
 * union is the OR of word w of every leaf's bitmap — coalesced 128-byte reads per leaf and warp, 6 MB per
 * 5-leaf query over 10M documents — and its population count is the exact match count (no ownership logic).  The
 * same words give "held by two or more leaves" (two |= one & x; one |= x): those documents, a few percent of the
 * union, are the only ones scored here — presence mask from the bits, MaxScore bucket from a table held one entry
 * per lane, wdf of every present leaf through its rank directory, the reference's tree order (or_score_doc).
 * Their weights give the top-k threshold b* its level BEFORE the far more numerous single-leaf documents are
 * looked at: those are left to xgm_or3_kernel<PHASE 1>, which walks the posting lists and, knowing b*, skips
 * whole leaves and whole blocks (largest wdf of the block in its header) without decoding them.  A single-leaf
 * document in the final top-k has a weight >= the final threshold >= b* after this kernel, so nothing is lost.
 * Work item = 2048 words (65 536 docids) of one query, ordered range-major over the batch. */
#define TILE_WARPS 8
#define TILE_ITERS 64
#define TILE_QCAP 64

struct __align__(16) TileScratch {
    uint32_t qdid[TILE_QCAP];
    uint32_t qqi[TILE_QCAP];
    uint32_t qpm[TILE_QCAP];
};

__global__ void __launch_bounds__(TILE_WARPS * 32, 4) xgm_or_tile_kernel(const __grid_constant__ XgmKernelParams p) {
    __shared__ TileScratch scratch[TILE_WARPS];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    TileScratch& ws = scratch[warp];
    if (nothing_to_rerun(p)) return;
    const uint32_t nwords = (p.lastdocid >> 5) + 1u;
    const uint32_t items_per_q = (nwords + 32u * TILE_ITERS - 1u) / (32u * TILE_ITERS);
    const uint32_t nitems = items_per_q * p.ntileq;
    uint32_t qn = 0;

    auto flush = [&](uint32_t count) {
        qn -= count;
        const bool alive = lane < count;
        const uint32_t d = alive ? ws.qdid[qn + lane] : 0u;
        const uint32_t qi = alive ? ws.qqi[qn + lane] : 0u;
        const uint32_t pm = alive ? ws.qpm[qn + lane] : 0u;
        double acc = 0.0;
        if (alive) acc = or_score_doc(p, &p.queries[qi], d, pm, 0xffu, 0u, 0u);
        emit_match_lanes(p, lane, alive, qi, acc, d, (uint32_t)__popc(pm), false);
        __syncwarp();
    };

    uint32_t item;
    while (claim_item(p, XGM_WC_TILE, nitems, lane, item)) {
        const uint32_t tile = item / p.ntileq, qi = __ldg(p.tileq + (item - tile * p.ntileq));
        if (!runs_this_pass(p, qi)) continue;
        const XgmDevQuery* q = &p.queries[qi];
        const uint32_t nterms = q->nterms;
        /* the loads carry no per-leaf predicate: a missing leaf re-reads leaf 0's word (an L1 hit) and is masked */
        const uint32_t* bmp[OR3_MAX_LEAVES];
        uint32_t lm[OR3_MAX_LEAVES];
#pragma unroll
        for (int j = 0; j < OR3_MAX_LEAVES; ++j) {
            bmp[j] = p.bitmaps + q->terms[(uint32_t)j < nterms ? j : 0].bm_off;
            lm[j] = (uint32_t)j < nterms ? 0xffffffffu : 0u;
        }
        /* lane m: pruning bucket of presence mask m (sum of the get_maxpart bounds of its leaves) */
        const uint32_t ubbkt = bound_bucket(q, maxpart_sum(q, lane, 0.0));
        uint32_t total_acc = 0;
        const uint32_t w0 = tile * (32u * TILE_ITERS);
        const uint32_t iters = min((uint32_t)TILE_ITERS, (nwords - w0 + 31u) >> 5);
        /* the words of iteration it + 1 are requested before the candidates of iteration it are looked at (the
         * loads of one iteration used to be the only ones in flight); indices are clamped, not predicated */
        uint32_t w[OR3_MAX_LEAVES], wn[OR3_MAX_LEAVES];
        {
            const uint32_t word = w0 + lane;
            const uint32_t cw = min(word, nwords - 1u), vm = word < nwords ? 0xffffffffu : 0u;
#pragma unroll
            for (int j = 0; j < OR3_MAX_LEAVES; ++j) w[j] = __ldg(bmp[j] + cw) & lm[j] & vm;
        }
        for (uint32_t it = 0; it < iters; ++it) {
            const uint32_t word = w0 + it * 32u + lane;
            {
                const uint32_t nx = word + 32u;
                const uint32_t cw = min(nx, nwords - 1u), vm = (it + 1u < iters && nx < nwords) ? 0xffffffffu : 0u;
#pragma unroll
                for (int j = 0; j < OR3_MAX_LEAVES; ++j) wn[j] = __ldg(bmp[j] + cw) & lm[j] & vm;
            }
            uint32_t one = 0, two = 0;
#pragma unroll
            for (int j = 0; j < OR3_MAX_LEAVES; ++j) { two |= one & w[j]; one |= w[j]; }
            total_acc += (uint32_t)__popc(one);
            uint32_t cand = two;
            if (__any_sync(FULL, cand != 0)) {
                const uint32_t bstar = live_bstar(&p.qstate[qi]);
                do { /* one document per lane and round */
                    const bool has = cand != 0;
                    const uint32_t bit = has ? (uint32_t)__ffs(cand) - 1u : 0u;
                    cand &= cand - 1u;
                    uint32_t pm = 0;
#pragma unroll
                    for (int j = 0; j < OR3_MAX_LEAVES; ++j) pm |= (w[j] >> bit & 1u) << j;
                    const uint32_t bk = __shfl_sync(FULL, ubbkt, pm & 31u);
                    const bool ok = has && bk >= bstar;
                    const uint32_t B = __ballot_sync(FULL, ok);
                    if (B) {
                        if (ok) {
                            const uint32_t slot = qn + __popc(B & ((1u << lane) - 1u));
                            ws.qdid[slot] = (word << 5) + bit;
                            ws.qqi[slot] = qi;
                            ws.qpm[slot] = pm;
                        }
                        qn += __popc(B);
                        if (qn >= 32) { __syncwarp(); flush(32); }
                    }
                } while (__any_sync(FULL, cand != 0));
            }
#pragma unroll
            for (int j = 0; j < OR3_MAX_LEAVES; ++j) w[j] = wn[j];
        }
        count_matches(p, qi, total_acc, lane);
    }
    __syncwarp();
    if (qn) flush(qn);
}

cudaError_t xgm_launch_or_tile(const XgmKernelParams& p, int grid, cudaStream_t s) {
    xgm_or_tile_kernel<<<grid, TILE_WARPS * 32, 0, s>>>(p);
    return cudaGetLastError();
}

int xgm_or_tile_occupancy_blocks_per_sm() {
    int n = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, xgm_or_tile_kernel, TILE_WARPS * 32, 0);
    return n;
}

/* ------------------------------------------------------------------ top-k / ProtoMSet */

/* Strict total order of the reference's comparators (msetcmp.cc:54-98) with ascending docid order:
 * returns true when a ranks before b. */
__device__ __forceinline__ bool ranks_before(uint32_t sort_by, uint32_t reverse, double wa, uint32_t da, uint64_t ka,
                                             double wb, uint32_t db, uint64_t kb) {
    if (sort_by == 1 || sort_by == 2) {
        if (ka > kb) return reverse != 0;
        if (ka < kb) return reverse == 0;
        if (sort_by == 2) return da < db;
    }
    if (wa > wb) return true;
    if (wa < wb) return false;
    if (sort_by == 3) {
        if (ka > kb) return reverse != 0;
        if (ka < kb) return reverse == 0;
    }
    return da < db;
}

#define TOPK_THREADS 256
#define XGM_EXACT_COUNT_MAX 1024u /* largest match set whose ProtoMSet count is reproduced exactly */
#define XGM_KEEP_PER_THREAD 32   /* keep_cap <= 8192 = 32 * TOPK_THREADS */

/* Sort key of a match as up to five 32-bit words, most significant first, such that a larger key ranks
 * earlier under the reference's comparators (msetcmp.cc:54-98, ascending docid order):
 *   relevance:            weight bits, ~docid                      (3 words)
 *   value then relevance: value', weight bits, ~docid              (5 words)   value' = reverse ? v : ~v
 *   value:                value', ~docid                           (3 words)
 *   relevance then value: weight bits, value', ~docid              (5 words)
 * Weights are >= 0, so their IEEE bit patterns order like the values. */
__device__ __forceinline__ int match_key_words(uint32_t sort_by, uint32_t reverse, double w, uint64_t k, uint32_t d,
                                               uint32_t out[5]) {
    const uint64_t wb = (uint64_t)__double_as_longlong(w);
    const uint64_t kv = reverse ? k : ~k;
    const uint32_t nd = ~d;
    if (sort_by == 0) { out[0] = (uint32_t)(wb >> 32); out[1] = (uint32_t)wb; out[2] = nd; return 3; }
    if (sort_by == 2) { out[0] = (uint32_t)(kv >> 32); out[1] = (uint32_t)kv; out[2] = nd; return 3; }
    if (sort_by == 1) {
        out[0] = (uint32_t)(kv >> 32); out[1] = (uint32_t)kv; out[2] = (uint32_t)(wb >> 32); out[3] = (uint32_t)wb; out[4] = nd;
        return 5;
    }
    out[0] = (uint32_t)(wb >> 32); out[1] = (uint32_t)wb; out[2] = (uint32_t)(kv >> 32); out[3] = (uint32_t)kv; out[4] = nd;
    return 5;
}

/* Weights are >= +0.0 and never NaN, so their IEEE bit patterns order like the values: the ranking loops
 * compare 64-bit integers (full-rate integer pipe) instead of doubles — the FP64 compare throughput of the
 * SM is what bounded the top-k CTAs of queries with ~1000 matches. */
__device__ __forceinline__ uint64_t wbits(double w) { return (uint64_t)__double_as_longlong(w); }

/* Bitonic sort of the CTA's shared-memory candidate arrays (w, k, d), P a power of two, all TOPK_THREADS
 * threads.  BY_DOCID: ascending docid.  Otherwise the reference's relevance order: weight descending,
 * docid ascending (msetcmp.cc:54-61). */
template <bool BY_DOCID>
__device__ __forceinline__ void bitonic_sort_candidates(double* sw, uint64_t* sk, uint32_t* sd, uint32_t P, uint32_t tid) {
    for (uint32_t k = 2; k <= P; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t t = tid; t < P; t += TOPK_THREADS) {
                const uint32_t x = t ^ j;
                if (x > t) {
                    const uint32_t da = sd[t], db = sd[x];
                    const double wa = sw[t], wb = sw[x];
                    const uint64_t ba = wbits(wa), bb = wbits(wb);
                    /* true when the pair is out of order for an ascending run */
                    const bool wrong = BY_DOCID ? (da > db) : (ba < bb || (ba == bb && da > db));
                    const bool right = BY_DOCID ? (da < db) : (ba > bb || (ba == bb && da < db));
                    if (((t & k) == 0) ? wrong : right) {
                        sd[t] = db; sd[x] = da;
                        sw[t] = wb; sw[x] = wa;
                        const uint64_t ka = sk[t]; sk[t] = sk[x]; sk[x] = ka;
                    }
                }
            }
            __syncthreads();
        }
    }
}

/* One CTA per query.
 * First pass: survivors (bucket >= final b*) are compacted into shared memory and rank-sorted under
 * the reference's total order; when nothing was pruned the same pass reproduces ProtoMSet's
 * known_matching_docs (walking the matches in docid order, a match is counted iff it is among the first
 * max(check_at_least, topk+1) or fewer than topk earlier matches have a strictly greater weight —
 * protomset.h:340-400 with the `weight < min_weight → continue` of matcher.cc:496-498).
 * If candidates were lost (many warps emitted before b* could rise) the completed histogram gives the
 * exact b* and the exact number of matches at or above it; the query gets a slice of the overflow pool
 * and is flagged for a second matching pass.
 * Second pass: the slice holds every match at or above b*.  If a single bucket holds a mass of ties the
 * slice can be far larger than shared memory: an MSB-first radix select over the composite sort key
 * (8 bits per round, in global memory) finds the exact topk-th key, and only the topk winners are sorted. */
__device__ __forceinline__ void topk_one_query(const XgmKernelParams& p, const uint32_t qi) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const XgmDevQuery* q = &p.queries[qi];
    const XgmQState st = p.qstate[qi];
    if (p.pass != 0 && st.rerun == 0) return;
    double* sw = reinterpret_cast<double*>(smem_raw);
    uint64_t* sk = reinterpret_cast<uint64_t*>(sw + p.keep_cap);
    uint32_t* sd = reinterpret_cast<uint32_t*>(sk + p.keep_cap);
    __shared__ uint32_t s_known, s_n, s_hist[256], s_prefix[5], s_krem;
    const uint32_t sort_by = q->sort_by, reverse = q->sort_reverse;
    const uint32_t topk = q->topk;
    const uint32_t tid = threadIdx.x;
    if (tid == 0) { s_known = 0; s_n = 0; }
    __syncthreads();
    bool complete = false;
    uint32_t lost = 0;

    if (p.pass == 0) {
        const uint32_t stored = st.stored < p.match_cap ? st.stored : p.match_cap;
        const size_t qoff = (size_t)qi * p.match_cap;
        complete = (st.total == st.stored) && (st.stored <= p.keep_cap); /* every match is here */
        /* four independent rounds of loads in flight per thread: a dense query stores thousands of
         * candidates and one dependent round trip per 256 of them would make its CTA the launch's tail */
        for (uint32_t base = 0; base < stored; base += 4 * TOPK_THREADS) {
            double w[4];
            uint64_t k[4];
            uint32_t d[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const uint32_t i = base + u * TOPK_THREADS + tid;
                if (i < stored) {
                    w[u] = __ldcs(p.match_w + qoff + i);
                    k[u] = __ldcs(p.match_k + qoff + i);
                    d[u] = __ldcs(p.match_d + qoff + i);
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const uint32_t i = base + u * TOPK_THREADS + tid;
                const bool keep = i < stored && (complete || match_bucket(q, w[u], k[u]) >= st.bstar);
                /* one shared-memory atomic per warp, not per survivor (an unpruned query keeps everything) */
                const uint32_t m = __ballot_sync(FULL, keep);
                if (m) {
                    const uint32_t lane = tid & 31u, leader = (uint32_t)__ffs(m) - 1u;
                    uint32_t pos0 = 0;
                    if (lane == leader) pos0 = atomicAdd(&s_n, (uint32_t)__popc(m));
                    pos0 = __shfl_sync(FULL, pos0, leader);
                    if (keep) {
                        const uint32_t pos = pos0 + __popc(m & ((1u << lane) - 1u));
                        if (pos < p.keep_cap) { sw[pos] = w[u]; sd[pos] = d[u]; sk[pos] = k[u]; }
                    }
                }
            }
        }
        __syncthreads();
        if (st.stored > p.match_cap || s_n > p.keep_cap) {
            if (tid == 0) {
                const uint32_t* hist = p.hist + (size_t)qi * XGM_NBINS;
                uint32_t cum = 0, b = XGM_NBINS;
                while (b > 0 && cum < topk) { --b; cum += hist[b]; }
                if (b < st.bstar) { b = st.bstar; cum = 0; for (uint32_t i = b; i < XGM_NBINS; ++i) cum += hist[i]; }
                XgmDevResult r;
                r.n = 0; r.exact = st.total; r.known = 0; r.max_w = __longlong_as_double((long long)st.maxw);
                r.max_subqs = q->nweighted; r.pad = 0;
                /* 64-bit reservation counter: the sum over a batch of tie-mass queries cannot wrap */
                const unsigned long long off = atomicAdd(reinterpret_cast<unsigned long long*>(p.work_counter + XGM_WC_POOL), (unsigned long long)cum);
                if (cum >= topk && off + cum <= (unsigned long long)p.pool_total) {
                    p.qstate[qi].bstar = b;
                    p.qstate[qi].stored = 0;
                    p.qstate[qi].pool_off = (uint32_t)off;
                    p.qstate[qi].pool_cap = cum;
                    p.qstate[qi].rerun = 1;
                    atomicAdd(p.work_counter + XGM_WC_RERUN, 1u);
                    r.flags = XGM_RES_PENDING;
                } else {
                    r.flags = XGM_RES_LOST; /* overflow pool exhausted */
                }
                p.out_info[qi] = r;
            }
            return;
        }
    } else {
        const uint32_t n_src = st.stored < st.pool_cap ? st.stored : st.pool_cap;
        if (st.stored != st.pool_cap) lost = 1; /* cannot happen: the histogram count is exact */
        const double* gw = p.pool_w + st.pool_off;
        const uint32_t* gd = p.pool_d + st.pool_off;
        const uint64_t* gk = p.pool_k + st.pool_off;
        if (n_src <= p.keep_cap) {
            for (uint32_t i = tid; i < n_src; i += TOPK_THREADS) { sw[i] = gw[i]; sd[i] = gd[i]; sk[i] = gk[i]; }
            if (tid == 0) s_n = n_src;
            __syncthreads();
        } else {
            /* radix select: find the exact key of the topk-th best match, 8 bits per round */
            const int nwords = (sort_by == 0 || sort_by == 2) ? 3 : 5;
            if (tid < 5) s_prefix[tid] = 0;
            if (tid == 0) s_krem = topk;
            __syncthreads();
            for (int round = 0; round < nwords * 4; ++round) {
                s_hist[tid] = 0; /* TOPK_THREADS == 256 */
                __syncthreads();
                const int wi = round >> 2, sh = 24 - 8 * (round & 3);
                for (uint32_t i = tid; i < n_src; i += TOPK_THREADS) {
                    uint32_t kw[5];
                    match_key_words(sort_by, reverse, gw[i], gk[i], gd[i], kw);
                    bool ok = true;
                    for (int x = 0; x < wi; ++x) ok = ok && (kw[x] == s_prefix[x]);
                    if (ok && sh < 24) ok = (kw[wi] >> (sh + 8)) == (s_prefix[wi] >> (sh + 8));
                    if (ok) atomicAdd(&s_hist[(kw[wi] >> sh) & 255u], 1u);
                }
                __syncthreads();
                if (tid == 0) {
                    uint32_t krem = s_krem, dgt = 255;
                    for (;; --dgt) {
                        if (s_hist[dgt] >= krem || dgt == 0) break;
                        krem -= s_hist[dgt];
                    }
                    s_krem = krem;
                    s_prefix[wi] |= dgt << sh;
                }
                __syncthreads();
            }
            /* collect everything >= the selected key: exactly topk matches (keys are unique) */
            for (uint32_t i = tid; i < n_src; i += TOPK_THREADS) {
                uint32_t kw[5];
                match_key_words(sort_by, reverse, gw[i], gk[i], gd[i], kw);
                bool ge = true;
                for (int x = 0; x < nwords; ++x) {
                    if (kw[x] != s_prefix[x]) { ge = kw[x] > s_prefix[x]; break; }
                }
                if (ge) {
                    const uint32_t pos = atomicAdd(&s_n, 1u);
                    if (pos < p.keep_cap) { sw[pos] = gw[i]; sd[pos] = gd[i]; sk[pos] = gk[i]; }
                }
            }
            __syncthreads();
        }
    }

    const uint32_t kept = s_n;
    uint32_t n = kept < p.keep_cap ? kept : p.keep_cap;
    /* The exact ProtoMSet count needs all n^2 pairs; beyond XGM_EXACT_COUNT_MAX matches only the top-k is
     * produced: a shared-memory histogram of the same monotone buckets gives a threshold bucket, entries
     * below it are dropped before ranking (the bounds are then flagged approximate). */
    if (n > XGM_EXACT_COUNT_MAX && topk != 0 && topk < n) {
        complete = false;
        uint32_t* lh = reinterpret_cast<uint32_t*>(sd + p.keep_cap); /* XGM_NBINS words after the arrays */
        for (uint32_t i = tid; i < XGM_NBINS; i += TOPK_THREADS) lh[i] = 0;
        __syncthreads();
        for (uint32_t i = tid; i < n; i += TOPK_THREADS) atomicAdd(&lh[match_bucket(q, sw[i], sk[i])], 1u);
        __syncthreads();
        if (tid < 32) {
            const uint32_t b = bin_of_rank(lh, topk, tid);
            if (tid == 0) s_prefix[0] = b;
        }
        if (tid == 32) s_n = 0;
        __syncthreads();
        const uint32_t bsel = s_prefix[0];
        /* in-place compaction: read everything into registers first (n <= keep_cap <= 32 per thread) */
        double rw[XGM_KEEP_PER_THREAD]; uint64_t rk[XGM_KEEP_PER_THREAD]; uint32_t rd[XGM_KEEP_PER_THREAD];
        uint32_t cnt = 0;
        for (uint32_t i = tid, x = 0; i < n; i += TOPK_THREADS, ++x) {
            rw[x] = sw[i]; rk[x] = sk[i]; rd[x] = sd[i];
            cnt = x + 1;
        }
        __syncthreads();
        for (uint32_t x = 0; x < cnt; ++x) {
            if (match_bucket(q, rw[x], rk[x]) >= bsel) {
                const uint32_t pos = atomicAdd(&s_n, 1u);
                sw[pos] = rw[x]; sk[pos] = rk[x]; sd[pos] = rd[x];
            }
        }
        __syncthreads();
        n = s_n;
    }
    const uint32_t free_count = q->check_at_least > topk + 1 ? q->check_at_least : topk + 1;
    uint32_t known = 0;
    const size_t ooff = (size_t)qi * p.out_stride;
    if (sort_by == 0) {
        /* relevance order: weight desc, docid asc — no sort keys to compare.  The docid-order history of
         * ProtoMSet's count is only needed when the count is reported (unpruned set) and can differ from n
         * (more matches than the free_count that are counted unconditionally). */
        const bool need_counts = complete && !st.skipped && n > free_count;
        if (need_counts && n <= TOPK_THREADS) {
            /* Few survivors (the common case of a 3-term AND: 100 < n <= 256): one element per thread and one
             * pass over the others gives the rank, the docid-order position and both "earlier" counters — no
             * sort, one barrier.  The merge sort below needs ~45 barrier-separated stages for the same n. */
            const bool act = tid < n;
            const uint64_t* bw = reinterpret_cast<const uint64_t*>(sw);
            const uint64_t bi = act ? bw[tid] : 0ull;
            const uint32_t di = act ? sd[tid] : 0u;
            uint32_t rank = 0, posd = 0, gt = 0, ge = 0;
            if (act)
                for (uint32_t j = 0; j < n; ++j) {
                    const uint64_t bj = bw[j];
                    const uint32_t before = (uint32_t)(sd[j] < di), g = (uint32_t)(bj > bi), e = (uint32_t)(bj == bi);
                    posd += before;
                    gt += before & g;
                    ge += before & (g | e);
                    rank += g | (e & before);
                }
            const uint32_t cal = q->check_at_least;
            if (tid == 0) s_prefix[0] = cal <= topk + 1 ? topk : 0xffffffffu;
            __syncthreads();
            if (cal > topk + 1) {
                const uint32_t from = cal - 1 > topk ? cal - 1 : topk;
                if (act && posd >= from && ge < topk) atomicMin(&s_prefix[0], posd);
                __syncthreads();
            }
            const uint32_t r_raise = s_prefix[0];
            if (act) {
                if (rank < topk) {
                    p.out_w[ooff + rank] = sw[tid];
                    p.out_d[ooff + rank] = di;
                    p.out_k[ooff + rank] = sk[tid] & 0xffull;
                }
                if (posd <= r_raise || gt < topk) ++known;
            }
        } else if (need_counts) {
            /* 256 < n <= XGM_EXACT_COUNT_MAX.  Put the survivors in docid order first: "earlier in docid order"
             * becomes "smaller index".  Only 8-byte keys (docid << 10 | index) are sorted — 32 at a time in
             * registers (one warp, shuffles, no barrier), then log2(P / 32) merge passes in shared memory, each
             * element finding its place by one binary search in the other run — and the records are gathered
             * once.  (A bitonic sort of the 20-byte records took 55 barrier-separated passes for P = 1024 and
             * two thirds of this path's time.) */
            uint32_t P = 512;
            while (P < n) P <<= 1;
            {
                uint64_t* ksrc = reinterpret_cast<uint64_t*>(sw + P); /* the upper halves are free: 2P <= keep_cap */
                uint64_t* kdst = sk + P;
                const uint32_t lane = tid & 31u, warp = tid >> 5;
                for (uint32_t c = warp; c < P / 32u; c += TOPK_THREADS / 32u) {
                    const uint32_t i = c * 32u + lane;
                    uint64_t key = i < n ? ((uint64_t)sd[i] << 10) | i : ~0ull;
#pragma unroll
                    for (uint32_t k2 = 2; k2 <= 32; k2 <<= 1) {
#pragma unroll
                        for (uint32_t j = k2 >> 1; j > 0; j >>= 1) {
                            const uint64_t other = __shfl_xor_sync(FULL, key, j);
                            const bool keep_min = ((lane & j) == 0) == ((lane & k2) == 0);
                            key = keep_min ? (key < other ? key : other) : (key < other ? other : key);
                        }
                    }
                    ksrc[i] = key;
                }
                __syncthreads();
                const uint32_t nx = P / TOPK_THREADS; /* 2 or 4 elements per thread */
                for (uint32_t L = 32; L < P; L <<= 1) {
                    /* the searches of a thread's elements run in lockstep — fixed trip count, no branches — so
                     * that their dependent shared-memory probes overlap instead of queueing one behind the other */
                    uint64_t key[4];
                    const uint64_t* o[4];
                    uint32_t dstb[4], cnt[4];
                    bool isb[4];
#pragma unroll
                    for (uint32_t x = 0; x < 4; ++x) {
                        const uint32_t t = tid + x * TOPK_THREADS, tt = x < nx ? t : tid;
                        const uint32_t base = tt & ~(2u * L - 1u), off = tt - base;
                        key[x] = ksrc[tt];
                        isb[x] = off >= L;
                        o[x] = ksrc + base + (isb[x] ? 0u : L);
                        dstb[x] = base + (isb[x] ? off - L : off);
                        cnt[x] = 0;
                    }
                    for (uint32_t step = L >> 1; step > 0; step >>= 1) {
#pragma unroll
                        for (uint32_t x = 0; x < 4; ++x) {
                            const uint64_t e = o[x][cnt[x] + step - 1u];
                            if (isb[x] ? e <= key[x] : e < key[x]) cnt[x] += step; /* A: b's strictly smaller; B: a's not larger */
                        }
                    }
#pragma unroll
                    for (uint32_t x = 0; x < 4; ++x) {
                        const uint64_t e = o[x][cnt[x]];
                        if (isb[x] ? e <= key[x] : e < key[x]) ++cnt[x];
                        if (x < nx) kdst[dstb[x] + cnt[x]] = key[x];
                    }
                    __syncthreads();
                    uint64_t* tk_ = ksrc; ksrc = kdst; kdst = tk_;
                }
                /* gather: P / 256 <= 4 records per thread travel through registers into docid order; the
                 * per-element state of the merge below goes into the aux word: aux (8 bits) | docid-order position
                 * (11) | greater-before (11) | not-less-before (11) */
                double gw[4];
                uint64_t ga[4];
                uint32_t gd[4];
#pragma unroll
                for (uint32_t x = 0; x < 4; ++x) {
                    const uint32_t t = tid + x * TOPK_THREADS;
                    gw[x] = 0.0; ga[x] = 0; gd[x] = 0xffffffffu;
                    if (t < P) {
                        const uint64_t key = ksrc[t];
                        if (key != ~0ull) {
                            const uint32_t i = (uint32_t)key & 1023u;
                            gw[x] = sw[i]; ga[x] = sk[i] & 0xffull; gd[x] = (uint32_t)(key >> 10);
                        }
                    }
                }
                __syncthreads();
#pragma unroll
                for (uint32_t x = 0; x < 4; ++x) {
                    const uint32_t t = tid + x * TOPK_THREADS;
                    if (t < P) { sw[t] = gw[x]; sk[t] = ga[x] | ((uint64_t)t << 8); sd[t] = gd[x]; }
                }
                __syncthreads();
            }
            /* Bottom-up merge sort by (weight desc, docid asc) of the docid-ordered survivors.  While run A
             * (earlier docids) is merged with run B, every b in B learns how many a in A are strictly greater
             * ("earlier and greater", ProtoMSet's min_weight test) and how many are not smaller; the merged
             * position of an element is its index in its run plus one binary search in the other run.  After
             * log2(P) passes the array is the ranked MSet.  O(n log^2 n) instead of the n^2 pair test. */
            double* w_src = sw; double* w_dst = sw + P;
            uint64_t* k_src = sk; uint64_t* k_dst = sk + P;
            uint32_t* d_src = sd; uint32_t* d_dst = sd + P;
            const uint32_t nx = P / TOPK_THREADS;
            for (uint32_t L = 1; L < P; L <<= 1) {
                /* as above: the elements of a thread search in lockstep.  Run A counts the b's strictly greater; run
                 * B counts the a's strictly greater (its "greater before") and the a's not smaller (its place) */
                uint64_t bi[4], st8[4];
                const uint64_t* o[4];
                uint32_t dstb[4], cgt[4], cge[4], dd[4];
                bool isb[4];
#pragma unroll
                for (uint32_t x = 0; x < 4; ++x) {
                    const uint32_t t = tid + x * TOPK_THREADS, tt = x < nx ? t : tid;
                    const uint32_t base = tt & ~(2u * L - 1u), off = tt - base;
                    bi[x] = wbits(w_src[tt]);
                    st8[x] = k_src[tt];
                    dd[x] = d_src[tt];
                    isb[x] = off >= L;
                    o[x] = reinterpret_cast<const uint64_t*>(w_src) + base + (isb[x] ? 0u : L);
                    dstb[x] = base + (isb[x] ? off - L : off);
                    cgt[x] = 0; cge[x] = 0;
                }
                for (uint32_t step = L >> 1; step > 0; step >>= 1) {
#pragma unroll
                    for (uint32_t x = 0; x < 4; ++x) {
                        const uint64_t e1 = o[x][cgt[x] + step - 1u], e2 = o[x][cge[x] + step - 1u];
                        if (e1 > bi[x]) cgt[x] += step;
                        if (e2 >= bi[x]) cge[x] += step;
                    }
                }
#pragma unroll
                for (uint32_t x = 0; x < 4; ++x) {
                    if (o[x][cgt[x]] > bi[x]) ++cgt[x];
                    if (o[x][cge[x]] >= bi[x]) ++cge[x];
                    if (x < nx) {
                        const uint32_t pos = dstb[x] + (isb[x] ? cge[x] : cgt[x]);
                        if (isb[x]) st8[x] += ((uint64_t)cgt[x] << 19) + ((uint64_t)cge[x] << 30);
                        reinterpret_cast<uint64_t*>(w_dst)[pos] = bi[x];
                        d_dst[pos] = dd[x];
                        k_dst[pos] = st8[x];
                    }
                }
                /* a warp owns whole 32-element groups (t = tid + 256 x), so the passes inside a group need no CTA barrier */
                if (L < 16) __syncwarp(); else __syncthreads();
                double* tw_ = w_src; w_src = w_dst; w_dst = tw_;
                uint64_t* tk_ = k_src; k_src = k_dst; k_dst = tk_;
                uint32_t* td_ = d_src; d_src = d_dst; d_dst = td_;
            }
            /* position at which ProtoMSet first raises min_weight: the heap build (k) when check_at_least <=
             * k + 1, else the first replacement at or after check_at_least - 1 (protomset.h:377-398;
             * tests/test_protomset_count_model.py) */
            const uint32_t cal = q->check_at_least;
            if (tid == 0) s_prefix[0] = cal <= topk + 1 ? topk : 0xffffffffu;
            __syncthreads();
            if (cal > topk + 1) {
                const uint32_t from = cal - 1 > topk ? cal - 1 : topk;
                for (uint32_t t = tid; t < n; t += TOPK_THREADS) {
                    const uint64_t st8 = k_src[t];
                    const uint32_t posd = (uint32_t)(st8 >> 8) & 0x7ffu, ge = (uint32_t)(st8 >> 30) & 0x7ffu;
                    if (posd >= from && ge < topk) atomicMin(&s_prefix[0], posd);
                }
                __syncthreads();
            }
            const uint32_t r_raise = s_prefix[0];
            for (uint32_t t = tid; t < n; t += TOPK_THREADS) { /* real matches occupy the first n ranks */
                const uint64_t st8 = k_src[t];
                const uint32_t posd = (uint32_t)(st8 >> 8) & 0x7ffu, gt = (uint32_t)(st8 >> 19) & 0x7ffu;
                if (t < topk) {
                    p.out_w[ooff + t] = w_src[t];
                    p.out_d[ooff + t] = d_src[t];
                    p.out_k[ooff + t] = st8 & 0xffull;
                }
                if (posd <= r_raise || gt < topk) ++known;
            }
        } else {
            uint32_t P = 32;
            while (P < n) P <<= 1;
            if (n > TOPK_THREADS && P <= p.keep_cap) {
                /* many survivors (a mass of tied weights, or a dense query): sort instead of ranking pairs */
                for (uint32_t t = n + tid; t < P; t += TOPK_THREADS) { sd[t] = 0xffffffffu; sw[t] = 0.0; sk[t] = 0; }
                __syncthreads();
                bitonic_sort_candidates<false>(sw, sk, sd, P, tid);
                const uint32_t m = n < topk ? n : topk;
                for (uint32_t i = tid; i < m; i += TOPK_THREADS) {
                    p.out_w[ooff + i] = sw[i];
                    p.out_d[ooff + i] = sd[i];
                    p.out_k[ooff + i] = sk[i];
                }
                if (tid == 0) known = n; /* used only when n <= free_count: every match is counted */
            } else {
                /* rank only; two threads share an element when there are few (j split by parity).  The loop
                 * bound is uniform so that the pair's shuffle is executed by whole warps. */
                const uint32_t split = n <= TOPK_THREADS / 2 ? 2u : 1u;
                const uint32_t sub = tid & (split - 1u);
                for (uint32_t base = 0; base < n; base += TOPK_THREADS / split) {
                    const uint32_t i = base + tid / split;
                    const bool act = i < n;
                    const double wi = act ? sw[i] : 0.0;
                    const uint64_t bi = wbits(wi);
                    const uint64_t* bw = reinterpret_cast<const uint64_t*>(sw);
                    const uint32_t di = act ? sd[i] : 0u;
                    uint32_t rank = 0;
                    if (act)
                        for (uint32_t j = sub; j < n; j += split) {
                            const uint64_t bj = bw[j]; /* no short-circuit: branches here cost ~100 cycles a pair */
                            rank += (uint32_t)(bj > bi) | ((uint32_t)(bj == bi) & (uint32_t)(sd[j] < di));
                        }
                    if (split == 2u) rank += __shfl_xor_sync(FULL, rank, 1);
                    if (act && sub == 0u) {
                        if (rank < topk) {
                            p.out_w[ooff + rank] = wi;
                            p.out_d[ooff + rank] = di;
                            p.out_k[ooff + rank] = sk[i];
                        }
                        ++known; /* n <= free_count: every match is counted */
                    }
                }
            }
        }
    } else {
        for (uint32_t i = tid; i < n; i += TOPK_THREADS) {
            const double wi = sw[i];
            const uint32_t di = sd[i];
            const uint64_t ki = sk[i];
            uint32_t rank = 0, before = 0, greater_before = 0;
            for (uint32_t j = 0; j < n; ++j) {
                const double wj = sw[j];
                const uint32_t dj = sd[j];
                rank += ranks_before(sort_by, reverse, wj, dj, sk[j], wi, di, ki) ? 1u : 0u;
                const bool earlier = dj < di;
                before += earlier ? 1u : 0u;
                greater_before += (earlier && wj > wi) ? 1u : 0u;
            }
            if (rank < topk) {
                p.out_w[ooff + rank] = wi;
                p.out_d[ooff + rank] = di;
                p.out_k[ooff + rank] = ki;
            }
            if (sort_by == 1 || sort_by == 2 || before < free_count || greater_before < topk) ++known;
        }
    }
    atomicAdd(&s_known, known);
    __syncthreads();
    if (tid == 0) {
        XgmDevResult r;
        r.n = n < topk ? n : topk;
        r.exact = st.total;
        r.flags = 0;
        if (kept > p.keep_cap || lost) r.flags |= XGM_RES_LOST;
        if (topk == 0) {
            r.known = st.total; /* nothing is ever kept, so min_weight never rises: every match is counted */
        } else if (complete && !st.skipped) {
            r.known = s_known;
        } else {
            /* pruned run: ProtoMSet's count depends on docid-order history we did not keep; report the
             * guaranteed part and flag the bounds as approximate */
            r.known = st.total < free_count ? st.total : free_count;
            r.flags |= XGM_RES_APPROX;
        }
        if (st.skipped) r.flags |= XGM_RES_SKIPPED;
        if (p.pass != 0) r.flags |= XGM_RES_SECOND_PASS;
        r.max_w = __longlong_as_double((long long)st.maxw);
        r.max_subqs = q->nweighted;
        r.pad = 0;
        p.out_info[qi] = r;
    }
}

/* Queries whose whole match set is a handful of documents — the majority of a batch of selective ANDs (70 % of
 * BASELINE's C2 queries match <= 32 documents) — do not need a CTA, 45 KB of shared memory and a dozen barriers:
 * one warp ranks up to 64 unpruned relevance-ordered matches (two per lane, pair test against a 768-byte
 * staging area) and every one of them is counted (n <= max(check_at_least, topk + 1): protomset.h:340-376).
 * Everything else is put on topk_list for xgm_topk_kernel (XGM_WC_TOPK_FRONT entries from the front, XGM_WC_TOPK_BACK from the back). */
#define TOPK_SMALL_WARPS 8
#define TOPK_SMALL_MAX 64u
__global__ void __launch_bounds__(TOPK_SMALL_WARPS * 32) xgm_topk_small_kernel(const __grid_constant__ XgmKernelParams p) {
    __shared__ unsigned long long s_w[TOPK_SMALL_WARPS][TOPK_SMALL_MAX];
    __shared__ uint32_t s_d[TOPK_SMALL_WARPS][TOPK_SMALL_MAX];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t qi = blockIdx.x * TOPK_SMALL_WARPS + warp;
    if (qi >= p.nq) return;
    const XgmDevQuery* q = &p.queries[qi];
    const XgmQState st = p.qstate[qi];
    const uint32_t topk = q->topk, n = st.stored;
    const uint32_t free_count = q->check_at_least > topk + 1 ? q->check_at_least : topk + 1;
    const bool small = q->sort_by == 0 && topk != 0 && n == st.total && st.skipped == 0 && n <= TOPK_SMALL_MAX &&
                       n <= free_count && n <= p.match_cap;
    if (!small) {
        /* longest first: the queries whose exact count needs the sorts (more than 256 stored matches) fill the
         * list from the front, the others from the back, and the CTAs take the front first */
        if (lane == 0) {
            if (n > TOPK_THREADS) p.topk_list[atomicAdd(p.work_counter + XGM_WC_TOPK_FRONT, 1u)] = qi;
            else p.topk_list[p.nq - 1u - atomicAdd(p.work_counter + XGM_WC_TOPK_BACK, 1u)] = qi;
        }
        return;
    }
    const size_t qoff = (size_t)qi * p.match_cap, ooff = (size_t)qi * p.out_stride;
    unsigned long long bw[2] = {0ull, 0ull}, kk[2] = {0ull, 0ull};
    uint32_t dd[2] = {0u, 0u};
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const uint32_t i = lane + 32u * u;
        if (i < n) {
            bw[u] = (unsigned long long)__double_as_longlong(__ldcs(p.match_w + qoff + i));
            dd[u] = __ldcs(p.match_d + qoff + i);
            kk[u] = __ldcs(p.match_k + qoff + i);
            s_w[warp][i] = bw[u];
            s_d[warp][i] = dd[u];
        }
    }
    __syncwarp();
    uint32_t rank[2] = {0u, 0u};
    for (uint32_t j = 0; j < n; ++j) { /* weights are >= +0 and never NaN: their bit patterns order like the values */
        const unsigned long long bj = s_w[warp][j];
        const uint32_t dj = s_d[warp][j];
#pragma unroll
        for (int u = 0; u < 2; ++u) rank[u] += (uint32_t)(bj > bw[u]) | ((uint32_t)(bj == bw[u]) & (uint32_t)(dj < dd[u]));
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const uint32_t i = lane + 32u * u;
        if (i < n && rank[u] < topk) {
            p.out_w[ooff + rank[u]] = __longlong_as_double((long long)bw[u]);
            p.out_d[ooff + rank[u]] = dd[u];
            p.out_k[ooff + rank[u]] = kk[u];
        }
    }
    if (lane == 0) {
        XgmDevResult r;
        r.n = n < topk ? n : topk;
        r.exact = st.total;
        r.known = n;
        r.flags = 0;
        r.max_w = __longlong_as_double((long long)st.maxw);
        r.max_subqs = q->nweighted;
        r.pad = 0;
        p.out_info[qi] = r;
    }
}

/* CTA per query, persistent: the CTAs take the listed queries (first pass, after xgm_topk_small_kernel) or all
 * queries of the batch (no list; second pass) from a counter. */
__global__ void __launch_bounds__(TOPK_THREADS) xgm_topk_kernel(XgmKernelParams p) {
    __shared__ uint32_t s_slot;
    if (p.pass != 0 && *reinterpret_cast<volatile uint32_t*>(p.work_counter + XGM_WC_RERUN) == 0) return; /* nothing to re-run */
    const bool listed = p.topk_list != nullptr && p.pass == 0;
    const uint32_t nfront = listed ? *reinterpret_cast<volatile uint32_t*>(p.work_counter + XGM_WC_TOPK_FRONT) : p.nq;
    const uint32_t count = nfront + (listed ? *reinterpret_cast<volatile uint32_t*>(p.work_counter + XGM_WC_TOPK_BACK) : 0u);
    for (;;) {
        __syncthreads(); /* the previous query's shared state is no longer read */
        if (threadIdx.x == 0) s_slot = atomicAdd(p.work_counter + XGM_WC_TOPK + p.pass, 1u);
        __syncthreads();
        const uint32_t slot = s_slot;
        if (slot >= count) break;
        topk_one_query(p, !listed ? slot : slot < nfront ? p.topk_list[slot] : p.topk_list[p.nq - 1u - (slot - nfront)]);
    }
}

/* ------------------------------------------------------------------ multi-shard merge */

/* Matcher::merge_mset (matcher.cc:653-782) on the device, after an all-gather of the per-GPU top-k
 * records: one CTA per query merges the nparts sorted lists under (weight desc, docid asc) with docids
 * mapped through unshard() (backends/multi.h:66-70).  Every part arrives sorted in that very order
 * (unshard is monotone within a part), so the rank of a record is its index in its own part plus, for
 * every other part, the number of records there that rank before it — a binary search each. */
#define XGM_MERGE_MAX_PARTS 64
__global__ void __launch_bounds__(256) xgm_merge_kernel(const double* __restrict__ gw, const uint32_t* __restrict__ gd,
                                                        const XgmDevResult* __restrict__ ginfo, size_t part_w,
                                                        size_t part_d, size_t part_info, uint32_t nparts,
                                                        uint32_t nq, uint32_t stride, uint32_t k, double* out_w,
                                                        uint32_t* out_d, uint32_t* out_n) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* sw = reinterpret_cast<double*>(smem_raw);
    uint32_t* sd = reinterpret_cast<uint32_t*>(sw + (size_t)nparts * k);
    __shared__ uint32_t s_cnt[XGM_MERGE_MAX_PARTS];
    const uint32_t qi = blockIdx.x;
    /* part strides are in bytes: the parts are either three gathered arrays or whole result slabs */
    for (uint32_t part = threadIdx.x; part < nparts; part += blockDim.x) {
        const XgmDevResult* pi = reinterpret_cast<const XgmDevResult*>(reinterpret_cast<const unsigned char*>(ginfo) + part * part_info);
        s_cnt[part] = min(pi[qi].n, k);
    }
    __syncthreads();
    const size_t off = (size_t)qi * stride;
    for (uint32_t x = threadIdx.x; x < nparts * k; x += blockDim.x) {
        const uint32_t part = x / k, i = x - part * k;
        if (i < s_cnt[part]) {
            const double* pw = reinterpret_cast<const double*>(reinterpret_cast<const unsigned char*>(gw) + part * part_w);
            const uint32_t* pd = reinterpret_cast<const uint32_t*>(reinterpret_cast<const unsigned char*>(gd) + part * part_d);
            sw[x] = pw[off + i];
            sd[x] = (pd[off + i] - 1u) * nparts + part + 1u;
        }
    }
    __syncthreads();
    uint32_t total = 0;
    for (uint32_t part = 0; part < nparts; ++part) total += s_cnt[part];
    for (uint32_t x = threadIdx.x; x < nparts * k; x += blockDim.x) {
        const uint32_t part = x / k, i = x - part * k;
        if (i >= s_cnt[part]) continue;
        const double wi = sw[x];
        const uint32_t di = sd[x];
        uint32_t rank = i;
        for (uint32_t o = 0; o < nparts && rank < k; ++o) {
            if (o == part) continue;
            const double* ow = sw + (size_t)o * k;
            const uint32_t* od = sd + (size_t)o * k;
            uint32_t lo = 0, hi = s_cnt[o]; /* first record of part o that does not rank before (wi, di) */
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                const double wm = ow[mid];
                if (wm > wi || (wm == wi && od[mid] < di)) lo = mid + 1; else hi = mid;
            }
            rank += lo;
        }
        if (rank < k) {
            out_w[(size_t)qi * k + rank] = wi;
            out_d[(size_t)qi * k + rank] = di;
        }
    }
    if (threadIdx.x == 0) out_n[qi] = total < k ? total : k;
}

cudaError_t xgm_launch_merge(const double* gw, const uint32_t* gd, const XgmDevResult* ginfo, size_t part_w, size_t part_d,
                             size_t part_info, uint32_t nparts, uint32_t nq, uint32_t stride, uint32_t k, double* out_w, uint32_t* out_d, uint32_t* out_n,
                             cudaStream_t s) {
    if (nparts > XGM_MERGE_MAX_PARTS) return cudaErrorInvalidValue;
    size_t smem = (size_t)nparts * k * 12;
    if (smem > 48 * 1024) {
        cudaError_t e = optin_smem((const void*)xgm_merge_kernel, 0, smem);
        if (e != cudaSuccess) return e;
    }
    xgm_merge_kernel<<<nq, 256, smem, s>>>(gw, gd, ginfo, part_w, part_d, part_info, nparts, nq, stride, k, out_w, out_d, out_n);
    return cudaGetLastError();
}

/* ------------------------------------------------------------------ coarse bitmaps (index upload) */

/* Coarse word g summarises fine words 8g .. 8g + 7 (one 256-docid group): bit 4k + j is set if byte j of fine word
 * 8g + k is non-zero, i.e. bit (d >> 3) & 31 stands for docids d & ~7 .. (d & ~7) + 7. */
__global__ void __launch_bounds__(256) xgm_coarse_kernel(const uint4* __restrict__ bm, size_t ncoarse, uint32_t* __restrict__ coarse) {
    const size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ncoarse) return;
    const uint4 a = bm[2 * g], b = bm[2 * g + 1];
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    uint32_t out = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k)
#pragma unroll
        for (int j = 0; j < 4; ++j) out |= ((w[k] >> (8 * j)) & 0xffu ? 1u : 0u) << (4 * k + j);
    coarse[g] = out;
}

cudaError_t xgm_launch_coarse(const uint32_t* bitmaps, size_t ncoarse, uint32_t* coarse, cudaStream_t s) {
    if (ncoarse == 0) return cudaSuccess;
    xgm_coarse_kernel<<<(unsigned)((ncoarse + 255) / 256), 256, 0, s>>>(reinterpret_cast<const uint4*>(bitmaps), ncoarse, coarse);
    return cudaGetLastError();
}

/* ------------------------------------------------------------------ decode (round-trip check) */

__global__ void __launch_bounds__(MATCH_WARPS * 32) xgm_decode_kernel(XgmKernelParams p, uint32_t blk_begin,
                                                                      uint32_t nblocks, uint32_t* out_d,
                                                                      uint32_t* out_w) {
    __shared__ WarpScratch scratch[MATCH_WARPS];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    WarpScratch& ws = scratch[warp];
    if (lane == 0) mbar_init(&ws.bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    uint32_t phase = 0;
    for (uint32_t b = blockIdx.x * MATCH_WARPS + warp; b < nblocks; b += gridDim.x * MATCH_WARPS) {
        const XgmBlockHdr h = p.hdr[blk_begin + b];
        const uint32_t count = XGM_HDR_COUNT(h.meta);
        uint32_t d[4];
        stage_block(p.docs, h.doc_off, XGM_HDR_DOC_BITS(h.meta), ws.stage, &ws.bar, phase, lane);
        decode_docids(ws.stage, XGM_HDR_DOC_BITS(h.meta), h.first, lane, d);
        stage_block(p.tfs, h.tf_off, XGM_HDR_TF_BITS(h.meta), ws.stage, &ws.bar, phase, lane);
        const uint32_t tb = XGM_HDR_TF_BITS(h.meta);
        const uint32_t tmask = bitmask(tb);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            uint32_t idx = 4 * lane + k;
            if (idx < count) {
                out_d[(size_t)b * XGM_BLOCK + idx] = d[k];
                out_w[(size_t)b * XGM_BLOCK + idx] = tb ? unpack_sm(ws.stage, idx, tb, tmask) : 0u;
            }
        }
    }
}

/* ------------------------------------------------------------------ work-list expansion */

/* The host only sends one segment per (query[, leaf]): {query, #blocks, 0, leaf}, sorted by descending #blocks,
 * and this kernel expands them into work items of `bpi` blocks in level order (level_start[k] = number of items in
 * levels < k, nlevels >= 1): all queries' first items, then all second items, ...  The warps in flight at any
 * moment belong to many queries, so every query's pruning threshold rises early, long queries do not form a tail,
 * and concurrently running items of one query stay far apart.  The OR list is expanded one leaf group at a time,
 * rarest leaves of all queries first, for MaxScore.  The range-major bitmap AND list has its own kernels below. */
__global__ void xgm_expand_items_kernel(const XgmWorkItem* __restrict__ seg, uint32_t total,
                                        const uint32_t* __restrict__ level_start, uint32_t nlevels, uint32_t bpi,
                                        XgmWorkItem* __restrict__ out) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= total) return;
    uint32_t lo = 0, hi = nlevels; /* last level whose start is <= s */
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (level_start[mid] <= s) lo = mid; else hi = mid;
    }
    const XgmWorkItem sg = seg[s - level_start[lo]];
    XgmWorkItem w;
    w.query = sg.query;
    w.b0 = lo * bpi;
    w.b1 = min(sg.b0, w.b0 + bpi);
    w.pad = sg.pad;
    out[s] = w;
}

/* Range-major expansion (bitmap AND list, large batches).  The docid space is cut into ranges of
 * 2^range_bits documents and the work list is ordered range by range, every query's driver blocks of
 * range 0 first, then range 1, ...: at any moment all warps probe the same slice of every membership
 * bitmap (lastdocid/8 bytes per term shrink to 2^range_bits/8), which stays in the 50 MB L2 while the
 * whole batch walks over it — each bitmap is read from HBM about once per batch instead of once per query
 * that uses it.  Every query still advances through the whole batch, so thresholds rise early as with the
 * level order.  The list's unit is a run of up to XGM_BM_RUN queries with the same driver list: its items
 * serve all of them.  Three small kernels: per (range, run) the driver blocks whose first docid falls in
 * the range (two binary searches over the skip table) and their item count; an exclusive scan in
 * range-major order; the fill. */
__device__ __forceinline__ uint32_t first_block_at_or_after(const XgmBlockHdr* __restrict__ h, uint32_t nblk, uint64_t target) {
    uint32_t lo = 0, hi = nblk;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if ((uint64_t)h[mid].first < target) lo = mid + 1; else hi = mid;
    }
    return lo;
}

#define XGM_RNG_THREADS 256
__device__ __forceinline__ uint32_t block_exclusive_scan_256(uint32_t v, uint32_t* warp_sums /* [8] shared */, uint32_t* block_total) {
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(FULL, incl, o);
        if ((int)lane >= o) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    uint32_t before = 0, total = 0;
#pragma unroll
    for (uint32_t x = 0; x < XGM_RNG_THREADS / 32; ++x) {
        const uint32_t ws = warp_sums[x];
        if (x < warp) before += ws;
        total += ws;
    }
    *block_total = total;
    return before + incl - v;
}

__global__ void __launch_bounds__(XGM_RNG_THREADS) xgm_range_count_kernel(
    const XgmWorkItem* __restrict__ runs, uint32_t nruns, const XgmBlockHdr* __restrict__ hdr, uint32_t nranges,
    uint32_t range_bits, uint32_t bpi, uint32_t* __restrict__ lo_out, uint32_t* __restrict__ cnt_out,
    uint32_t* __restrict__ block_sums) {
    __shared__ uint32_t warp_sums[XGM_RNG_THREADS / 32];
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t cnt = 0;
    if (t < nranges * nruns) {
        const uint32_t j = t / nruns, r = t - j * nruns; /* range-major: consecutive threads = consecutive runs */
        const XgmWorkItem rn = runs[r]; /* b0 = #driver blocks, b1 = the driver's first header */
        const XgmBlockHdr* h = hdr + rn.b1;
        const uint32_t nblk = rn.b0;
        /* a block belongs to the range of its first docid */
        const uint32_t lo = j == 0 ? 0u : first_block_at_or_after(h, nblk, (uint64_t)j << range_bits);
        const uint32_t hi = j + 1 == nranges ? nblk : first_block_at_or_after(h, nblk, (uint64_t)(j + 1) << range_bits);
        lo_out[t] = lo;
        cnt = (hi - lo + bpi - 1) / bpi;
        cnt_out[t] = cnt;
    }
    uint32_t total;
    (void)block_exclusive_scan_256(cnt, warp_sums, &total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

/* exclusive scan of the per-block sums (a few hundred to a few thousand values), one CTA */
#define XGM_SCAN_THREADS 1024
__global__ void __launch_bounds__(XGM_SCAN_THREADS) xgm_range_scan_kernel(uint32_t* __restrict__ block_sums, uint32_t n,
                                                                         uint32_t* total) {
    __shared__ uint32_t part[XGM_SCAN_THREADS];
    const uint32_t tid = threadIdx.x;
    const uint32_t chunk = (n + XGM_SCAN_THREADS - 1) / XGM_SCAN_THREADS;
    const uint32_t a = min(n, tid * chunk), b = min(n, a + chunk);
    uint32_t sum = 0;
    for (uint32_t i = a; i < b; ++i) sum += block_sums[i];
    part[tid] = sum;
    __syncthreads();
    for (uint32_t o = 1; o < XGM_SCAN_THREADS; o <<= 1) {
        const uint32_t v = tid >= o ? part[tid - o] : 0u;
        __syncthreads();
        part[tid] += v;
        __syncthreads();
    }
    uint32_t run = part[tid] - sum;
    for (uint32_t i = a; i < b; ++i) { const uint32_t c = block_sums[i]; block_sums[i] = run; run += c; }
    if (tid == XGM_SCAN_THREADS - 1) *total = part[tid];
}

__global__ void __launch_bounds__(XGM_RNG_THREADS) xgm_range_fill_kernel(
    const XgmWorkItem* __restrict__ runs, uint32_t nruns, uint32_t nranges, uint32_t bpi, const uint32_t* __restrict__ lo_in,
    const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ block_off, XgmWorkItem* __restrict__ out) {
    __shared__ uint32_t warp_sums[XGM_RNG_THREADS / 32];
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const bool in = t < nranges * nruns;
    const uint32_t n = in ? cnt[t] : 0u;
    uint32_t total;
    const uint32_t off = block_off[blockIdx.x] + block_exclusive_scan_256(n, warp_sums, &total);
    if (!in || n == 0) return;
    const uint32_t j = t / nruns, r = t - j * nruns;
    const XgmWorkItem rn = runs[r];
    const uint32_t lo = lo_in[t];
    const uint32_t hi = j + 1 == nranges ? rn.b0 : lo_in[t + nruns];
    XgmWorkItem w;
    w.query = rn.query; /* the run's first segment */
    w.pad = rn.pad;     /* and its number of queries */
    for (uint32_t i = 0; i < n; ++i) {
        w.b0 = lo + i * bpi;
        w.b1 = min(hi, w.b0 + bpi);
        out[off + i] = w;
    }
}

cudaError_t xgm_launch_expand_ranges(const XgmWorkItem* runs, uint32_t nruns, const XgmBlockHdr* hdr, uint32_t nranges,
                                     uint32_t range_bits, uint32_t bpi, uint32_t* lo, uint32_t* cnt, uint32_t* off,
                                     uint32_t* total, XgmWorkItem* out, cudaStream_t s) {
    const uint32_t n = nranges * nruns;
    if (n == 0) return cudaSuccess;
    const uint32_t nb = (n + XGM_RNG_THREADS - 1) / XGM_RNG_THREADS; /* `off` holds the nb block sums / offsets */
    xgm_range_count_kernel<<<nb, XGM_RNG_THREADS, 0, s>>>(runs, nruns, hdr, nranges, range_bits, bpi, lo, cnt, off);
    xgm_range_scan_kernel<<<1, XGM_SCAN_THREADS, 0, s>>>(off, nb, total);
    xgm_range_fill_kernel<<<nb, XGM_RNG_THREADS, 0, s>>>(runs, nruns, nranges, bpi, lo, cnt, off, out);
    return cudaGetLastError();
}

cudaError_t xgm_launch_expand(const XgmWorkItem* seg, uint32_t total, const uint32_t* level_start, uint32_t nlevels,
                              uint32_t bpi, XgmWorkItem* out, cudaStream_t s) {
    if (total == 0) return cudaSuccess;
    xgm_expand_items_kernel<<<(total + 255) / 256, 256, 0, s>>>(seg, total, level_start, nlevels, bpi, out);
    return cudaGetLastError();
}

/* ------------------------------------------------------------------ launchers */

cudaError_t xgm_launch_and(const XgmKernelParams& p, int grid, cudaStream_t s) {
    xgm_and_kernel<<<grid, MATCH_WARPS * 32, 0, s>>>(p);
    return cudaGetLastError();
}

cudaError_t xgm_launch_or(const XgmKernelParams& p, int grid, cudaStream_t s) {
    xgm_or_kernel<<<grid, OR_WARPS * 32, 0, s>>>(p);
    return cudaGetLastError();
}

size_t xgm_topk_smem_bytes(uint32_t keep_cap) { return (size_t)keep_cap * (8 + 8 + 4) + XGM_NBINS * 4; }

cudaError_t xgm_launch_topk(const XgmKernelParams& p, uint32_t nq, cudaStream_t s) {
    size_t smem = xgm_topk_smem_bytes(p.keep_cap);
    if (smem > 48 * 1024) {
        cudaError_t e = optin_smem((const void*)xgm_topk_kernel, 1, smem);
        if (e != cudaSuccess) return e;
    }
    XgmKernelParams pp = p;
    pp.nq = nq;
    /* first pass of a real batch: the few-match queries are ranked a warp each, the rest listed for the CTAs */
    if (p.pass == 0 && nq >= 64 && p.topk_list != nullptr)
        xgm_topk_small_kernel<<<(nq + TOPK_SMALL_WARPS - 1) / TOPK_SMALL_WARPS, TOPK_SMALL_WARPS * 32, 0, s>>>(pp);
    else
        pp.topk_list = nullptr;
    static int ctas = 0; /* resident CTAs of the persistent kernel on this device class */
    if (ctas == 0) {
        int dev = 0, sms = 0, occ = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, xgm_topk_kernel, TOPK_THREADS, smem);
        ctas = sms * (occ > 0 ? occ : 1);
    }
    const uint32_t grid = nq < (uint32_t)ctas ? nq : (uint32_t)ctas;
    xgm_topk_kernel<<<grid, TOPK_THREADS, smem, s>>>(pp);
    return cudaGetLastError();
}

cudaError_t xgm_launch_decode(const XgmKernelParams& p, uint32_t blk_begin, uint32_t nblocks, uint32_t* out_d,
                              uint32_t* out_w, cudaStream_t s) {
    int grid = (int)((nblocks + MATCH_WARPS - 1) / MATCH_WARPS);
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms < 1) sms = 132; /* H100 SXM */
    if (grid > sms * 8) grid = sms * 8;
    if (grid < 1) grid = 1;
    xgm_decode_kernel<<<grid, MATCH_WARPS * 32, 0, s>>>(p, blk_begin, nblocks, out_d, out_w);
    return cudaGetLastError();
}

int xgm_and_occupancy_blocks_per_sm() {
    int n = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, xgm_and_kernel, MATCH_WARPS * 32, 0);
    return n;
}

int xgm_or_occupancy_blocks_per_sm() {
    int n = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, xgm_or_kernel, OR_WARPS * 32, 0);
    return n;
}
