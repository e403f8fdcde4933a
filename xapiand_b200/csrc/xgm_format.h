/* xgm_format.h — HBM index layout and device-side query descriptors (shared by host and kernels).
 *
 * Posting lists (the reference's GlassPostList chunks, glass_postlist.cc:677-695: ~2000-byte chunks
 * of vbyte (docid delta-1, wdf) pairs behind a B-tree) are re-laid-out for the GPU as three columns:
 *
 *   hdr[]   one 16-byte XgmBlockHdr per block of up to 128 postings, all terms back to back, each
 *           term followed by one sentinel header (first = 0xFFFFFFFF) so "first docid of the next
 *           block" is always readable — that is the skip table the warp-galloping search walks.
 *   docs[]  per block 128 x doc_bits bits: delta-1 between consecutive docids (slot 0 = 0, the first
 *           docid lives in the header), little-endian bit-packed, value i at bit i*doc_bits.  A block
 *           is 16*doc_bits bytes, so every block starts 16-byte aligned (cp.async.bulk granularity).
 *   tfs[]   per block 128 x tf_bits bits of wdf, same packing, separate column: the intersection
 *           only touches it for documents that survive.
 *   bitmaps[]/ranks[]  optional per-term membership bitmap (bit d = docid d has the term) plus a rank
 *           directory (postings before every 256-docid group), kept for terms frequent enough that the
 *           bitmap costs at most XGM_BITMAP_K bits per posting.  HBM is plentiful (80 GB) and the
 *           leapfrog of an AND is at heart a membership test: probing a bitmap replaces decoding the
 *           longer lists entirely; the rank directory gives the posting's index, hence its wdf.
 *   coarse[] next to every bitmap, one bit per 8 docids (built on the device at upload): coarse word
 *           bm_off / 8 + (d >> 8) covers the 256-docid group of docid d, bit (d >> 3) & 31 is set if any
 *           of its 8 docids is in the list.  A bitmap is 8 words per group, so bm_off is a multiple of 8.
 *   doclen[] dense u32 per docid (the reference keeps a second vbyte stream under key "\0\xe0",
 *           glass_postlist.cc:194-205,994-1021).
 */
#ifndef XGM_FORMAT_H
#define XGM_FORMAT_H
#include <stdint.h>

#define XGM_BLOCK 128u
#define XGM_SENTINEL 0xFFFFFFFFu
#define XGM_DEV_MAX_TERMS 16u
#define XGM_NBINS 1024u  /* histogram bins of the top-k pruning threshold */

struct XgmBlockHdr {
    uint32_t first;    /* docid of the block's first posting */
    uint32_t doc_off;  /* offset of the packed docid deltas, in 16-byte units into docs[] */
    uint32_t tf_off;   /* offset of the packed wdfs, in 16-byte units into tfs[] */
    uint32_t meta;     /* doc_bits | tf_bits << 8 | (count-1) << 16 | min(255, largest wdf in the block) << 24 */
};

#define XGM_HDR_DOC_BITS(m) ((m) & 0xffu)
#define XGM_HDR_TF_BITS(m) (((m) >> 8) & 0xffu)
#define XGM_HDR_COUNT(m) ((((m) >> 16) & 0xffu) + 1u)
#define XGM_HDR_MAXWDF(m) ((m) >> 24) /* 255 = "255 or more": use the term's own bound */

#define XGM_NO_BITMAP 0xFFFFFFFFFFFFFFFFull
#define XGM_NO_SRC 0xFFFFFFFFu

struct XgmDevTerm {
    uint32_t blk_begin;   /* index of the term's first header in hdr[] */
    uint32_t nblocks;     /* real blocks (the sentinel sits at blk_begin + nblocks) */
    double termweight;    /* BM25Weight::init result, bm25weight.cc:46-130 (computed on the host) */
    uint64_t bm_off;      /* membership bitmap of the term (u32 words into bitmaps[]), XGM_NO_BITMAP if none */
    uint64_t rk_off;      /* its rank directory (u32 entries into ranks[]): postings before each 256-docid group */
    double maxpart;       /* BM25Weight::get_maxpart: upper bound of the term's contribution (MaxScore pruning) */
};

/* XgmDevQuery::route: the shape of the query on the device */
#define XGM_ROUTE_AND 0u /* required lists (then excluded and optional ones): the AND kernels */
#define XGM_ROUTE_OR 1u  /* OrPostList tree over the leaves: the OR kernels */

/* XgmDevQuery::or_fast: which kernels produce an OR's union */
#define XGM_OR_FAST_GENERAL 0u /* xgm_or_kernel: a leaf without bitmap, more than five leaves, or filter / AND_NOT terms */
#define XGM_OR_FAST_OR3 1u     /* xgm_or3_kernel<0>: at most five leaves, all with bitmaps */
#define XGM_OR_FAST_TILE 2u    /* as OR3 in relevance order with results and no value range: xgm_or_tile_kernel for
                                  the documents with two or more leaves, then xgm_or3_kernel<1> for the rest */

struct XgmDevQuery {
    uint32_t op, nterms, topk, check_at_least;
    double len_factor, k1, b, one_minus_b, min_normlen;
    uint32_t filter, filter_slot;
    uint64_t range_lo, range_hi;
    uint32_t sort_by, sort_slot, sort_reverse, sort_use_max;
    uint32_t prog_len;
    int8_t prog[2 * XGM_DEV_MAX_TERMS]; /* OR: postfix program over leaves (>=0) and '+' (-1) */
    uint32_t route;                     /* XGM_ROUTE_AND or XGM_ROUTE_OR */
    uint32_t nnot;                      /* AND: terms[nterms .. nterms+nnot) must be absent (OP_AND_NOT right side) */
    uint32_t nweighted;                 /* required leaves that carry a weight (OP_FILTER's boolean terms do not) */
    uint32_t nmaybe;                    /* AND: terms[nterms+nnot ..) are the optional leaves of an OP_AND_MAYBE; prog[] is
                                           the OrPostList tree over them */
    double bucket_scale;                /* XGM_NBINS / max_possible (or / (max sort key + 1)) */
    uint64_t sort_missing;              /* sort key of a document without a value in sort_slot */
    uint64_t bucket_key_min;            /* value sorts: smallest key of the slot (bucket = (key - min) * scale) */
    double src_weight;                  /* weighted value-range source: factor * 1.0 added to every match ... */
    uint32_t src_pos;                   /* ... before the weight of required list src_pos (MultiAndPostList order);
                                           nterms = after all; XGM_NO_SRC = the source only filters */
    uint32_t or_fast;                   /* OR: the kernels that produce its union, XGM_OR_FAST_* */
    uint32_t or_nreq;                   /* OR under OP_FILTER: terms[nterms .. nterms+or_nreq) must hold the document, then nnot excluded ones */
    uint32_t log_raises;                /* record the matches that attain the running maximum weight (XGM_RAISE_LOG) */
    uint32_t probe_coarse;              /* bitmap AND: test terms[1]'s coarse bit before its fine bit (sparse terms[1]) */
    uint32_t unweighted;                /* AND: bit j set = required list j has no Weight (an OP_FILTER boolean term or a
                                           factor-0 leaf) and adds nothing, as LeafPostList::get_weight returns 0 without
                                           one: its BM25 sumpart is not computed (at wdf 0 it would be 0 * (0 / 0)) */
    XgmDevTerm terms[XGM_DEV_MAX_TERMS]; /* AND: ascending termfreq (MultiAndPostList order) */
};

struct XgmWorkItem {
    uint32_t query;
    uint32_t b0, b1;   /* sparse kernel: driver-block range; dense kernel: docid tile range */
    uint32_t pad;
};

/* Range-major bitmap AND list: at most this many queries with the same driver list share one work item (a run),
 * which decodes the driver's blocks once for all of them.  Longer runs decode less but make fewer, longer items per
 * docid range, so more ranges are in flight at once and their bitmap slices outgrow L2 (DESIGN.md §6).  The AND
 * kernel tags a queued candidate with its query's slot in the run in 4 bits: at most 16. */
#define XGM_BM_RUN 6

/* per-query running state of a batch (zeroed before every launch) */
struct XgmQState {
    uint32_t total;            /* documents matching the boolean structure */
    uint32_t stored;           /* matches appended to the query's buffer (not yet prunable when seen) */
    uint32_t bstar;            /* pruning bucket: matches below it cannot reach the top-k any more */
    uint32_t rerun;            /* set by the top-k kernel: buffer overflowed, second pass with exact b* */
    unsigned long long maxw;   /* bit pattern of the best weight over all matches */
    uint32_t pool_off;         /* second pass: this query's slice of the overflow pool (entries) */
    uint32_t pool_cap;         /* exact number of matches at or above b* (from the completed histogram) */
    uint32_t skipped;          /* OR: whole work items were skipped by MaxScore (match count is a lower bound) */
    uint32_t nraise;           /* entries appended to the query's raise log (see XGM_RAISE_LOG) */
};

/* ProtoMSet::update_max_weight (matcher/protomset.h:174-183) remembers how many subqueries matched the
 * best-weighted document — the numerator of percent_scale_factor.  When that number varies per document (OR,
 * AND_MAYBE) and the MSet is NOT ordered by weight, the best-weighted document need not be among the results,
 * so queries that ask for it (XgmDevQuery::log_raises) log every match that attains the
 * running maximum: {weight bits, docid, matching subqueries}.  The running maximum only rises, so with distinct
 * weights the log holds about ln(matches) entries; but every match that ties the running maximum is logged too,
 * so a tie of more than XGM_RAISE_LOG matches at the best weight (or at a running maximum reached before it)
 * overflows it, and a query whose log overflows is declined. */
#define XGM_RAISE_LOG 64u
struct XgmRaise { unsigned long long wbits; uint32_t docid, subqs; };

#endif
