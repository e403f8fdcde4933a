/* xgm.h — C-ABI of the H100-native inverted-index matcher (libxgm.so).
 *
 * This is the drop-in boundary for ONE path of Kronuz/Xapiand: everything from
 * Matcher::get_local_mset (src/xapian/matcher/matcher.cc:346-542) downward — PostList tree
 * construction, GlassPostList iteration, MultiAndPostList / OrPostList advance,
 * BM25Weight::get_sumpart, ProtoMSet top-k — for the query shapes listed below.  The reference's
 * Xapian::Enquire / MSet surface and Xapiand's DatabaseHandler::get_mset
 * (src/database/handler.cc:1414-1553) stay above it unchanged; INTEGRATION.md shows the shim a
 * maintainer adds inside Matcher::get_local_mset.
 *
 * Conventions: plain C types, no C++ exceptions cross the boundary, every entry point returns an
 * xgm_status (0 = ok).  Handles are opaque.  An xgm_index is immutable after xgm_builder_finish /
 * xgm_index_load and may be shared by any number of host threads; an xgm_searcher (stream +
 * staging buffers) must be used by one thread at a time — the same rule as one Xapian::Enquire per
 * thread (src/database/lock.h:59-75 serialises a shard checkout).
 *
 * The CUDA path is the only path: there is no CPU fallback.  Query shapes the kernels do not cover
 * return XGM_E_UNIMPLEMENTED so the shim can throw Xapian::UnimplementedError and leave the query
 * to the reference's own matcher.
 */
#ifndef XGM_H
#define XGM_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XGM_ABI_VERSION 2
#define XGM_MAX_TERMS 16u      /* leaves per query handled on the device */
#define XGM_MAX_TOPK 4096u     /* first + maxitems */

typedef enum xgm_status {
    XGM_OK = 0,
    XGM_E_INVALID = 1,        /* bad argument */
    XGM_E_UNIMPLEMENTED = 2,  /* query shape not covered → reference matcher should run it */
    XGM_E_CUDA = 3,           /* CUDA runtime failure (→ Xapian::DatabaseError) */
    XGM_E_NOMEM = 4,
    XGM_E_IO = 5,
    XGM_E_STALE = 6,          /* revision mismatch (→ Xapian::DatabaseModifiedError) */
    XGM_E_NODEVICE = 7        /* no CUDA device: this library has no CPU path */
} xgm_status;

typedef struct xgm_builder xgm_builder;
typedef struct xgm_index xgm_index;
typedef struct xgm_searcher xgm_searcher;

/* ---- error text ------------------------------------------------------------------------- */
/* Thread-local description of the last failure on the calling thread (never NULL). */
const char* xgm_last_error(void);
uint32_t xgm_abi_version(void);

/* ---- index construction ------------------------------------------------------------------
 * Replaces the read side of GlassPostList (src/xapian/backends/glass/glass_postlist.cc:722-991):
 * the shim walks the glass DB once through Database::allterms_begin / postlist_begin /
 * get_doclength / valuestream_begin and hands the flat postings over; docids/wdfs are what
 * PostingIterator::operator* / get_wdf return. */
xgm_status xgm_builder_new(xgm_builder** out);
/* doclen[docid] for docid in [0, lastdocid]; entry 0 unused; 0 for unused docids.
 * Database::get_doccount/get_lastdocid/get_total_length/get_doclength_{lower,upper}_bound. */
xgm_status xgm_builder_set_docs(xgm_builder*, uint32_t doccount, uint32_t lastdocid,
                                uint64_t total_length, uint32_t doclen_lower_bound,
                                uint32_t doclen_upper_bound, const uint32_t* doclen);
/* One term's posting list, docids strictly ascending.  wdf_upper_bound = the reference's
 * Database::get_wdf_upper_bound(term) (glass_database.cc:822-829); pass 0 to have it derived the
 * same way from (termfreq, collfreq, first wdf, max wdf over the index). */
xgm_status xgm_builder_add_term(xgm_builder*, const char* term, uint32_t term_len,
                                const uint32_t* docids, const uint32_t* wdfs, uint32_t n,
                                uint64_t collfreq, uint32_t wdf_upper_bound, uint32_t* term_id);
/* Numeric value slot: for every docid up to `nvals[docid]` (0..255) order-preserving u64 keys,
 * ascending, laid out CSR-style: keys of docid d are vals[voff[d] .. voff[d+1]).  This is the
 * decoded form of Xapiand's StringList of sortable_serialise()d numbers
 * (src/serialise_list.h:301-356, src/sortable_serialise.cc). */
xgm_status xgm_builder_add_value_slot(xgm_builder*, uint32_t slot, const uint64_t* voff /*[lastdocid+2]*/,
                                      const uint64_t* vals);
/* The same slot in the form Xapiand stores it (Document::add_value of StringList::serialise over the sorted,
 * unique serialised values, src/database/schema.cc:2958-2959, src/serialise_list.h:301-356): bytes of docid d
 * are bytes[off[d] .. off[d+1]) — empty = no value, one value = its bytes, several = '\0' then
 * (serialise_length(len), bytes)*.  Every element becomes its value key (xgm_value_key below); elements are
 * kept in stored order.  A slot holding an element longer than 8 bytes is marked inexact and queries that
 * filter or sort on it are declined (XGM_E_UNIMPLEMENTED). */
xgm_status xgm_builder_add_value_slot_serialised(xgm_builder*, uint32_t slot, const uint64_t* off /*[lastdocid+2]*/,
                                                 const unsigned char* bytes);
/* Database::get_revision (src/xapian/database.h:600) of the snapshot the postings were read from; a query
 * that names another revision gets XGM_E_STALE (→ Xapian::DatabaseModifiedError, the retry loop of
 * src/database/handler.cc:1292-1316,1333-1335).  Default 0. */
xgm_status xgm_builder_set_revision(xgm_builder*, uint64_t revision);
/* Compress into the HBM block format and upload to `device`. Consumes the builder. */
xgm_status xgm_builder_finish(xgm_builder*, int device, xgm_index** out);
void xgm_builder_free(xgm_builder*);

/* Synthetic Zipfian corpus of BASELINE.md §3 (xgm_corpus.h), shard `shard` of `nshards`
 * (interleaved docids, src/xapian/backends/multi.h:37-70), built directly into an index. */
xgm_status xgm_index_build_synthetic(uint32_t ndocs, uint32_t vocab, uint64_t seed, uint32_t nshards,
                                     uint32_t shard, int with_values, int device, int host_threads,
                                     xgm_index** out);
/* A glass database directory, read directly: `iamglass` + the B-tree of `postlist.glass` (posting lists,
 * document lengths, value streams and statistics all live there) are parsed by the library itself — no Xapian
 * code, no cursors (src/xapian/backends/glass/glass_table.h:66-300, glass_postlist.cc:677-695,
 * glass_values.cc:69-91, glass_version.cc:97-234; SURVEY.md section 8(b), (f)-3).  The index carries the
 * database's revision; value slots go in as stored (xgm_builder_add_value_slot_serialised). */
xgm_status xgm_index_open(const char* glass_path, int device, xgm_index** out);
/* Host-only helpers of the same reader: the revision and document counts of the version file (to decide
 * whether an index is stale), and a dump in the XGMFLAT1 format of `oracle/ref_runner export`, which is how
 * the reader is pinned against the reference's own iterators without a GPU. */
xgm_status xgm_glass_revision(const char* glass_path, uint64_t* revision, uint32_t* doccount, uint32_t* lastdocid);
xgm_status xgm_glass_export_flat(const char* glass_path, const char* out_path);
/* XGMFLAT1 file (oracle/ref_runner `export`: a glass DB dumped through the public iterators). */
xgm_status xgm_index_load_flat(const char* path, int device, xgm_index** out);
void xgm_index_close(xgm_index*);

typedef struct xgm_index_info {
    uint32_t doccount, lastdocid;
    uint64_t total_length;
    uint32_t doclen_lower_bound, doclen_upper_bound;
    uint32_t nterms;
    uint64_t npostings;
    uint64_t nblocks;
    uint64_t bytes_docids, bytes_wdfs, bytes_headers, bytes_doclen; /* HBM footprint by column */
    int device;
    uint64_t revision;
    uint64_t bytes_bitmaps;  /* membership bitmaps, their coarse bitmaps (a bit per 8 docids) + rank directories of the frequent terms */
    uint32_t nbitmaps;
} xgm_index_info;
xgm_status xgm_index_info_get(const xgm_index*, xgm_index_info* out);

typedef struct xgm_term_stats {
    uint32_t term_id;
    uint32_t termfreq;       /* GlassPostListTable::get_freqs glass_postlist.cc:150-192 */
    uint64_t collfreq;
    uint32_t wdf_upper_bound;
    uint64_t bytes;          /* compressed HBM bytes of this term (docids + wdfs + headers) */
} xgm_term_stats;
/* Returns XGM_OK with termfreq == 0 for an unknown term (like Database::get_termfreq). */
xgm_status xgm_term_stats_get(const xgm_index*, const char* term, uint32_t term_len, xgm_term_stats* out);
/* termfreq of n terms in one call (0 for unknown terms): phase 1 of Xapiand's two-phase scheme looks up every
 * query term of a batch on every shard before the sums are exchanged (src/database/handler.cc:1532-1538). */
xgm_status xgm_term_stats_many(const xgm_index*, uint32_t n, const char* const* terms, const uint32_t* term_lens,
                               uint32_t* termfreq);
/* Round-trip check: decode a term's posting list on the device back into flat arrays (capacity n). */
xgm_status xgm_index_decode_term(const xgm_index*, uint32_t term_id, uint32_t* docids, uint32_t* wdfs,
                                 uint32_t capacity, uint32_t* n);
/* Document lengths of docids [first_docid, first_docid + n) copied from the dense HBM column (0 for unused
 * docids) — Database::get_doclength (api/database.cc:347), for tests and tools; not on the query path. */
xgm_status xgm_index_copy_doclengths(const xgm_index*, uint32_t first_docid, uint32_t n, uint32_t* out);

/* Number of documents with a value in `slot` (Database::get_value_freq). */
xgm_status xgm_index_value_freq(const xgm_index*, uint32_t slot, uint32_t* out);

/* ---- value keys ----------------------------------------------------------------------------
 * Xapian compares slot values as byte strings (msetcmp.cc:75-85, valuerangepostlist.cc:132-151,
 * src/multivalue/range.cc:351-368).  On the device a value is its first 8 bytes, big-endian, zero padded:
 * order-preserving for every string, and one-to-one for strings of at most 8 bytes without trailing NULs —
 * which covers Xapiand's sortable_serialise() of any number whose binary exponent is below 128 in magnitude
 * (src/sortable_serialise.cc:41-212: 2 header bytes + up to 54 mantissa bits, trailing zero bytes chopped).
 * xgm_value_key returns 1 when the key is exact (len <= 8, no trailing NUL), else 0. */
int xgm_value_key(const void* bytes, size_t len, uint64_t* key);
/* Inverse for exact keys: writes the value's bytes (<= 8), returns their number. */
size_t xgm_value_key_bytes(uint64_t key, unsigned char out[8]);
/* MSetIterator::get_sort_key for Xapiand's sorter: the bytes Multi_MultiValueKeyMaker::operator()
 * (src/multivalue/keymaker.cc:704-757) builds for ONE SerialiseKey slot from the value with this key —
 * forward: the value itself; reverse: every byte subtracted from 0xff ('\0' → "\xff\0"), then "\xff\xff".
 * out needs 20 bytes; returns the length. */
size_t xgm_sort_key_bytes(uint64_t key, int reverse, unsigned char out[20]);

/* ---- queries ------------------------------------------------------------------------------ */
enum { XGM_OP_AND = 0, XGM_OP_OR = 1 };                      /* Query::OP_AND / OP_OR of LEAF_TERMs */
enum { XGM_SORT_REL = 0, XGM_SORT_VAL_REL = 1, XGM_SORT_VAL = 2, XGM_SORT_REL_VAL = 3 };
                                                              /* Enquire::Internal::sort_setting */
enum { XGM_FILTER_NONE = 0,
       XGM_FILTER_VALUE_RANGE = 1,  /* OP_FILTER(q, OP_VALUE_RANGE(slot, lo, hi)): first value in range,
                                       src/xapian/matcher/valuerangepostlist.cc */
       XGM_FILTER_MULTI_RANGE = 2   /* OP_FILTER(q, MultipleValueRange): src/multivalue/range.cc:351-368 */ };

/* Collection statistics for Weight::init_ (src/xapian/weight/weight.cc:59-83).  NULL means "this
 * index alone".  In Xapiand's two-phase scheme (src/database/handler.cc:1532-1551) the caller sums
 * them over shards (Weight::Internal::operator+=, weightinternal.cc:54-72) and passes the totals. */
typedef struct xgm_stats {
    uint32_t collection_size;
    uint64_t total_length;
    const uint32_t* termfreq;   /* one per query term, in query order */
} xgm_stats;

typedef struct xgm_query {
    uint32_t op;                 /* XGM_OP_* over the terms below */
    uint32_t nterms;             /* 1..XGM_MAX_TERMS */
    const char* const* terms;    /* term bytes; may be NULL if term_ids is given */
    const uint32_t* term_lens;   /* NULL → NUL-terminated */
    const uint32_t* term_ids;    /* optional pre-resolved ids (xgm_term_stats.term_id); UINT32_MAX = absent */
    const uint32_t* wqf;         /* NULL → 1 each */
    uint32_t first, maxitems, check_at_least;   /* Enquire::get_mset arguments */
    const xgm_stats* stats;      /* NULL → local statistics */
    double k1, k3, b, min_normlen; /* BM25Weight parameters; all 0 → defaults 1,1,0.5,0.5 (weight.h:665-667);
                                      otherwise clamped as BM25Weight's constructor does: k1, k3 < 0 → 0,
                                      b to [0, 1] (weight.h:639-646) */
    uint32_t filter, filter_slot;
    uint64_t range_lo, range_hi;
    uint32_t sort_by, sort_slot, sort_reverse, sort_use_max; /* sort_use_max: key = largest value of the slot */
    /* Term groups around the base, innermost first (SURVEY.md §8(f)-1): all three around an XGM_OP_AND or
     * single-term base, nfilter and nnot also around an XGM_OP_OR base (nmaybe there: XGM_E_UNIMPLEMENTED).  Their
     * terms follow the nterms base terms in terms / term_lens / term_ids (and stats->termfreq):
     *   nfilter  OP_FILTER(base, AND of boolean terms)   QueryFilter::postlist   api/queryinternal.cc:2270-2283
     *   nnot     OP_AND_NOT(…, OR of terms)              QueryAndNot::postlist   api/queryinternal.cc:2208-2225,
     *                                                     AndNotPostList matcher/andnotpostlist.cc
     *   nmaybe   OP_AND_MAYBE(…, OR of weighted terms)   QueryAndMaybe::postlist api/queryinternal.cc:2247-2268,
     *                                                     AndMaybePostList matcher/andmaybepostlist.cc
     * nterms + nfilter + nnot + nmaybe <= XGM_MAX_TERMS.  wqf (when given) covers all of them; the filter and
     * excluded terms carry no weight, so theirs is ignored. */
    uint32_t nfilter, nnot, nmaybe, reserved;
    /* OP_SCALE_WEIGHT factor per base term (QueryScaleWeight::postlist api/queryinternal.cc:1075-1080: the
     * product of the factors above a leaf reaches Weight::init_); NULL → 1.0 each.  A factor of 0 makes the
     * leaf unweighted (AND bases only; under an OR it is declined). */
    const double* factors;
    /* ---- ABI 2 ---- */
    uint64_t revision;           /* 0 = any; else must equal the index's revision or the query gets XGM_E_STALE */
    /* The value-range source on the WEIGHTED side: OP_AND(base, PostingSource) — what
     * MultipleValueRange::getQuery + Xapiand's query DSL build (src/multivalue/range.cc:110-125): every match
     * gets filter_factor * get_weight() = filter_factor * 1.0 (range.cc:410-414, externalpostlist.cc:86-95) at
     * the source's place in the MultiAndPostList order, and max_possible includes filter_factor * DBL_MAX
     * (api/postingsource.cc:208).  0 = the source only filters (OP_FILTER right side). */
    uint32_t filter_weighted, reserved2;
    double filter_factor;        /* used when filter_weighted; 0 is treated as 1.0 */
    uint64_t sort_missing_key;   /* key of a document without a value in sort_slot: 0 (the empty string) for
                                    Enquire::set_sort_by_value* and for Xapiand's SerialiseKey in reverse — its
                                    MIN_STR_CMPVALUE is std::string("\x00"), i.e. empty (src/multivalue/keymaker.h:54) —
                                    and xgm_value_key("\xff") for SerialiseKey forward (MAX_STR_CMPVALUE, keymaker.h:53) */
} xgm_query;

/* One query's result: the fields of MSet::Internal (src/xapian/api/msetinternal.h:58-99). */
typedef struct xgm_mset_info {
    uint32_t n;                    /* items written (after dropping `first`) */
    uint32_t first;
    uint32_t matches_lower_bound, matches_estimated, matches_upper_bound;
    uint32_t uncollapsed_lower_bound, uncollapsed_estimated, uncollapsed_upper_bound;
    uint32_t exact_matches;        /* documents matching the boolean structure */
    uint32_t status;               /* xgm_status for this query */
    uint32_t flags;                /* XGM_MSET_* */
    uint32_t reserved;
    double max_possible, max_attained, percent_scale_factor;
} xgm_mset_info;

/* ProtoMSet::known_matching_docs depends on the docid-order history of the match (SURVEY.md §7 hard
 * part 3).  It is reproduced exactly whenever the whole match set fits the searcher's candidate
 * buffer and check_at_least is at most first+maxitems+1 (Xapiand's default) or is never reached; for larger
 * match sets that were pruned on the device, or a check_at_least in between (where the reference's
 * min_weight lags, protomset.h:377-398), the lower bound / estimate are conservative (still valid
 * bounds) and this flag is set.  Docids, weights, max_possible,
 * max_attained, percent_scale_factor, the upper bound and exact_matches are always exact.
 * percent_scale_factor needs the number of subqueries matching the FIRST document in docid order that attains
 * max_attained (ProtoMSet::update_max_weight, protomset.h:174-183).  Where that document need not be among the
 * results (an OR or OP_AND_MAYBE sorted by value), the kernels keep a record of the matches that reach the running
 * best weight; a query with more such matches than that record holds (XGM_RAISE_LOG, e.g. a tie of more than 64
 * matches at the best weight) is declined with XGM_E_UNIMPLEMENTED, never answered with a guessed percentage. */
#define XGM_MSET_BOUNDS_APPROX 1u
/* OR queries only: MaxScore skipped whole posting-list segments that cannot reach the top-k (what
 * OrPostList's w_min pruning does in the reference, orpostlist.cc:113-155), so exact_matches counts only
 * the documents actually visited.  Never set when check_at_least covers the match set. */
#define XGM_MSET_COUNT_LOWER_BOUND 2u

/* ---- searching ---------------------------------------------------------------------------- */
/* A searcher is what one Xapian::Enquire is to the reference (src/xapian/api/enquire.cc:71-298; one per
 * thread, like Xapiand's one Enquire per DocMatcher, src/database/handler.cc:1250-1371): it owns a CUDA
 * stream and pinned/device staging for batches of up to max_batch queries with first+maxitems <= max_topk
 * each.  xgm_search* replace Matcher::get_local_mset (src/xapian/matcher/matcher.cc:346-542, declared in
 * matcher.h:92-108) for the query shapes listed at xgm_query. */
xgm_status xgm_searcher_new(const xgm_index*, uint32_t max_batch, uint32_t max_topk, xgm_searcher** out);
/* May run after xgm_index_close of the searcher's index (a garbage collector frees the two in any order); the
 * searcher must not search once its index is closed. */
void xgm_searcher_free(xgm_searcher*);

/* Asynchronous batch: plan on the host, copy the plan to the device, launch the kernels, start the
 * device→host copy of the results.  Returns as soon as the work is enqueued. */
xgm_status xgm_search_submit(xgm_searcher*, const xgm_query* queries, uint32_t nq);
/* Same, but the host half (planning = the host part of LocalSubMatch::open_post_list + Weight::init_,
 * matcher/localsubmatch.cc:164-309, and the launches) runs on the searcher's worker thread, so the caller
 * can scatter an earlier batch of another searcher meanwhile.  `queries` (and the term strings they point
 * to) must stay valid until xgm_search_launched or xgm_search_wait returns; planning errors are reported
 * there.  xgm_search_launched blocks until everything is enqueued on the searcher's stream — needed
 * before enqueuing dependent work (the all-gather + merge of the multi-GPU path) on that stream. */
xgm_status xgm_search_submit_async(xgm_searcher*, const xgm_query* queries, uint32_t nq);
xgm_status xgm_search_launched(xgm_searcher*);
/* Wait for the submitted batch and scatter results: docids/weights hold `stride` entries per query
 * (query i at [i*stride, i*stride + info[i].n)); sort_keys may be NULL. */
xgm_status xgm_search_wait(xgm_searcher*, uint32_t* docids, double* weights, uint64_t* sort_keys,
                           uint32_t stride, xgm_mset_info* info);
/* Convenience: submit + wait. */
xgm_status xgm_search_batch(xgm_searcher*, const xgm_query* queries, uint32_t nq, uint32_t* docids,
                            double* weights, uint64_t* sort_keys, uint32_t stride, xgm_mset_info* info);
/* Single query, like Enquire::get_mset(first, maxitems, check_at_least). */
xgm_status xgm_search(xgm_searcher*, const xgm_query* query, uint32_t* docids, double* weights,
                      uint64_t* sort_keys, uint32_t capacity, xgm_mset_info* info);

/* Device-resident variant used for throughput measurement and multi-GPU merging: the plan built by
 * the last xgm_search_submit stays resident; xgm_search_replay relaunches the kernels on it without
 * host work or copies, leaving results in device memory. */
xgm_status xgm_search_replay(xgm_searcher*);
/* Device pointers of the last batch's top-k records (first+maxitems stride = xgm_searcher max_topk):
 * weights f64[nq*max_topk], docids u32[nq*max_topk], counts u32[nq] */
xgm_status xgm_search_device_results(xgm_searcher*, void** weights, void** docids, void** counts,
                                     uint32_t* stride);
/* The same three arrays live in ONE device allocation ("result slab": weights at offset 0, docids at
 * *off_docids, counts at *off_counts, *bytes in total), so that a shard's MSets travel in a single
 * all-gather (north_star: "a single NCCL all-gather of per-GPU top-k"; the exchange that replaces
 * handler.cc:1540-1556's per-shard prepared MSets). */
xgm_status xgm_search_device_slab(xgm_searcher*, void** base, uint64_t* bytes, uint64_t* off_docids,
                                  uint64_t* off_counts, uint32_t* stride);
/* The slab's fourth region, after the per-query records: the records' sort keys u64[nq*max_topk] at *off_keys
 * (256-byte aligned like the other regions), what xgm_search_wait returns as sort_keys for a value-sorted query.
 * A relevance-ordered query's keys there are unspecified. */
xgm_status xgm_search_device_slab_keys(xgm_searcher*, uint64_t* off_keys);
/* Multi-GPU use: leave the batch's results in the device slab only — xgm_search_submit* then skips the
 * device→host copies and xgm_search_wait only synchronises (its output arguments may be NULL).  The caller
 * exchanges and merges the slabs on the device and copies the merged MSets itself. */
xgm_status xgm_searcher_set_results_on_device(xgm_searcher*, int on);
/* CUDA stream of the searcher (cudaStream_t as void*) and timing/roofline counters of the last batch. */
void* xgm_searcher_stream(xgm_searcher*);
typedef struct xgm_batch_stats {
    uint64_t algorithmic_bytes;   /* SURVEY.md §8(d): sum over query terms of column bytes + 16*blocks, + 4*candidates + 16*k */
    uint64_t postings;            /* sum of termfreqs over the batch */
    uint32_t work_items;
    uint32_t kernel_launches;
    float match_kernel_ms;        /* CUDA-event time of the decode+intersect+score kernel(s) */
    float topk_kernel_ms;
    uint64_t h2d_bytes, d2h_bytes; /* bytes the batch moved over PCIe (plan in, results out) */
    float host_plan_ms;           /* host time inside xgm_search_submit (planning + enqueue) */
    float host_wait_ms;           /* host time inside xgm_search_wait after the stream drained (result scatter) */
    uint32_t second_pass_queries; /* queries whose candidate buffer overflowed and were matched a second time */
    uint32_t reserved;
} xgm_batch_stats;
xgm_status xgm_search_last_stats(xgm_searcher*, xgm_batch_stats* out);

/* ---- multi-shard merge (Matcher::merge_mset, src/xapian/matcher/matcher.cc:653-782) --------
 * parts: nparts per-shard results for the same query, docids already unsharded
 * (Xapian's unshard(), src/xapian/backends/multi.h:66-70, is applied by xgm_unshard). */
void xgm_unshard(uint32_t* docids, uint32_t n, uint32_t shard, uint32_t nshards);
xgm_status xgm_merge_msets(const uint32_t* const* docids, const double* const* weights,
                           const uint64_t* const* sort_keys, const xgm_mset_info* infos, uint32_t nparts,
                           uint32_t first, uint32_t maxitems, uint32_t sort_by, uint32_t sort_reverse,
                           uint32_t* out_docids, double* out_weights, uint64_t* out_sort_keys,
                           xgm_mset_info* out_info);
/* Device-side merge after an all-gather of per-GPU top-k records: gathered weights/docids hold
 * nparts*nq*stride records laid out [part][query][rank], gathered_counts the per-part result records
 * (the buffer xgm_search_device_results returns as `counts`, 32 bytes per query, first u32 = n);
 * local docids are unsharded on the fly (part p = shard p of nparts). Outputs: [nq][k] weights and
 * docids, [nq] counts. Relevance order (xgm_merge_mset_device_slab takes every order).  A query that any part lost (its shard's overflow pool could
 * not take a tie mass: xgm_search_wait reports XGM_E_UNIMPLEMENTED for it) gets count UINT32_MAX and no
 * records, never a merge without that shard's documents; the other queries are unaffected.  A query declined
 * because of its shape is declined on every shard alike and merges with count 0.
 * Limits: k <= stride, nparts <= 64, nparts * k * 12 <= 200 KiB (the kernel's shared memory). */
xgm_status xgm_merge_topk_device(const void* gathered_weights, const void* gathered_docids,
                                 const void* gathered_counts, uint32_t nparts, uint32_t nq, uint32_t stride,
                                 uint32_t k, void* out_weights, void* out_docids, void* out_counts,
                                 void* cuda_stream);
/* Same merge over nparts gathered result slabs (xgm_search_device_slab layout, slab p at
 * gathered + p*slab_bytes). */
xgm_status xgm_merge_topk_device_slab(const void* gathered, uint64_t slab_bytes, uint64_t off_docids,
                                      uint64_t off_counts, uint32_t nparts, uint32_t nq, uint32_t stride,
                                      uint32_t k, void* out_weights, void* out_docids, void* out_counts,
                                      void* cuda_stream);
/* The merge of gathered result slabs under each query's own order, with first > 0: Matcher::merge_mset under
 * Multi_MultiValueKeyMaker's comparator, as xgm_merge_msets does on the host.  off_keys is the slab's keys region
 * (xgm_search_device_slab_keys).  orders: device u8[nq], bits 0-1 the query's XGM_SORT_*, bit 2 its sort_reverse;
 * NULL orders every query by relevance and reads no keys.  The comparator, ties broken by ascending docid:
 *   XGM_SORT_VAL      key, docid (the weight is not compared);   XGM_SORT_VAL_REL  key, weight, docid;
 *   XGM_SORT_REL_VAL  weight, key, docid;                         XGM_SORT_REL      weight, docid.
 * Keys compare as unsigned 64-bit integers, ascending, or descending under reverse, which flips only the key.
 * Weights compare descending.  Each part gives its first min(n, first + maxitems) records (so every shard is
 * searched for ranks [0, first + maxitems)); merged ranks [first, first + maxitems) are written to
 * out_weights/out_docids/out_keys [nq][maxitems] and out_counts [nq] holds min(max(total - first, 0), maxitems).
 * Keys are written for queries whose order compares them; the rows of other queries in out_keys are not written.
 * A part that lost the query (as for xgm_merge_topk_device) or an order byte above 7 gives that query count
 * UINT32_MAX and no records; nothing is written past a count.  Each part must arrive sorted in its query's order,
 * as the searcher leaves it.
 * Limits: maxitems >= 1, first + maxitems <= stride, nparts <= 64,
 * nparts * (first + maxitems) * 20 <= 200 KiB (the kernel's shared memory); 8-byte aligned offsets, regions
 * weights | docids | records | keys in that order, each holding nq*stride records. */
xgm_status xgm_merge_mset_device_slab(const void* gathered, uint64_t slab_bytes, uint64_t off_docids,
                                      uint64_t off_counts, uint64_t off_keys, const uint8_t* orders,
                                      uint32_t nparts, uint32_t nq, uint32_t stride, uint32_t first,
                                      uint32_t maxitems, void* out_weights, void* out_docids,
                                      void* out_keys, void* out_counts, void* cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* XGM_H */
