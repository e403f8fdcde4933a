/* oracle/xgm_oracle.h — TEST INFRASTRUCTURE, not product code.
 *
 * CPU restatement (plain C, sequential, deliberately simple) of the reference's
 * Enquire → Matcher → PostList tree → BM25 → ProtoMSet path over flat posting arrays.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may load it.
 * Parity status: PINNED — checked against the compiled reference itself (oracle/_ref, built from
 * /root/reference/src/xapian by oracle/build_ref.sh) by tests/golden/make_golden.py; the resulting
 * fixtures are committed under tests/golden/ and re-checked by tests/test_oracle_golden.py: docids,
 * f64 weights, the three bounds, max_possible, max_attained and every item's percentage, for
 * term / AND / OR, two-phase shards, value range + sort (all three sort modes), FILTER / AND_NOT /
 * AND_MAYBE groups, OP_SCALE_WEIGHT factors, wqf, non-default BM25 parameters and the check_at_least /
 * first regimes.  Not pinned by the reference: Xapiand's MultipleValueRange predicate (its sources need
 * Xapiand's serialisers; restated from src/multivalue/range.cc:351-368), and term groups around an OR
 * base agree with the reference except for its AndMaybePostList decay quirk (DESIGN.md §3.1).
 */
#ifndef XGM_ORACLE_H
#define XGM_ORACLE_H
#include <stdint.h>
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct orc_index {
    uint32_t doccount;       /* number of documents */
    uint32_t lastdocid;      /* highest docid in use */
    uint64_t total_length;   /* sum of document lengths */
    uint32_t doclen_lb, doclen_ub;
    uint32_t* doclen;        /* [lastdocid+1], index = docid, 0 = unused docid */
    uint32_t nterms;
    uint64_t* off;           /* [nterms+1] offsets into docids/wdfs */
    uint32_t* docids;
    uint32_t* wdfs;
    uint64_t* collfreq;      /* [nterms] */
    uint32_t* wdf_ub;        /* [nterms] reference get_wdf_upper_bound(term) */
    char** names;            /* [nterms] term bytes, NUL-terminated (synthetic: "T%06u") */
    /* value slots (BASELINE config C5): per doc up to 3 integer values in slot 0 (sorted
     * ascending), one integer in slot 1; nvals0[d]==0 → doc has no values */
    uint8_t* nvals0;         /* [lastdocid+1] or NULL */
    uint64_t* vals0;         /* [3*(lastdocid+1)] */
    uint64_t* val1;          /* [lastdocid+1] */
    uint8_t* has1;           /* [lastdocid+1] slot-1 value present, or NULL = every document has one */
} orc_index;

/* collection statistics used by Weight::init_ (global over all shards in Xapiand's two-phase
 * scheme, src/xapian/api/enquire.cc:385-394; NULL = this index's own) */
typedef struct orc_stats {
    uint32_t collection_size;
    uint64_t total_length;
    const uint32_t* termfreq; /* per query term, global */
    const uint32_t* maybe_termfreq; /* per AND_MAYBE term, global (NULL = this index's own) */
} orc_stats;

enum { ORC_OP_AND = 0, ORC_OP_OR = 1 };
enum { ORC_SORT_REL = 0, ORC_SORT_VAL_REL = 1, ORC_SORT_VAL = 2, ORC_SORT_REL_VAL = 3 };
enum { ORC_FILTER_NONE = 0, ORC_FILTER_VALUE_RANGE_MIN = 1, ORC_FILTER_MULTI_RANGE = 2 };

typedef struct orc_query {
    int op;
    uint32_t nterms;
    const uint32_t* terms;    /* term ids */
    const uint32_t* wqf;      /* NULL = all 1 */
    const double* factors;    /* NULL = all 1.0; per term OP_SCALE_WEIGHT factor (api/queryinternal.cc:1075-1080);
                                 0 makes the leaf unweighted (no Weight object, not a counted subquery) */
    uint32_t first, maxitems, check_at_least;
    const orc_stats* stats;   /* NULL = local */
    /* BM25 parameters (src/xapian/weight.h:665-667 defaults k1=1 k2=0 k3=1 b=0.5 min_normlen=0.5) */
    double k1, k3, b, min_normlen;
    int filter;               /* ORC_FILTER_* */
    uint64_t range_lo, range_hi;
    int sort_by;              /* ORC_SORT_* */
    int sort_slot;            /* 0: smallest slot-0 value, 1: slot 1, 2: largest slot-0 value */
    int sort_reverse;         /* set_sort_by_value_then_relevance(slot, reverse) */
    /* SURVEY.md §8(f)-1 shapes around an AND, single-term or OR base (the device path covers AND / single-term
     * bases; OR bases are restated here for the next round), innermost first:
     *   OP_FILTER(base, AND of boolean terms)      QueryFilter::postlist   api/queryinternal.cc:2270-2283
     *   OP_AND_NOT(…, OR of terms)                 QueryAndNot::postlist   api/queryinternal.cc:2208-2225
     *   OP_AND_MAYBE(…, OR of weighted terms)      QueryAndMaybe::postlist api/queryinternal.cc:2247-2268 */
    uint32_t nfilter;
    const uint32_t* filter_terms;
    uint32_t nnot;
    const uint32_t* not_terms;
    uint32_t nmaybe;
    const uint32_t* maybe_terms;
    /* Xapiand's range source as a child of the AND (ORC_FILTER_MULTI_RANGE on an AND / single-term base, no
     * term groups): MultipleValueRange is a ValuePostingSource with termfreq (min, est, max) = (0, value_freq,
     * value_freq) (src/multivalue/range.cc:457-464, api/postingsource.cc:201-214), sorted into the
     * MultiAndPostList by that estimate.  filter_weighted: OP_AND(base, source) instead of OP_FILTER — every
     * match gets filter_factor * 1.0 (range.cc:410-414) at the source's place, max_possible includes
     * filter_factor * DBL_MAX, and the source is one more of the total subqueries. */
    int filter_weighted;
    double filter_factor;
    /* Xapiand's sorter (Multi_MultiValueKeyMaker with one SerialiseKey): key of a document without a value,
     * on the oracle's numeric scale where a value v sorts as v + 1: 0 = below everything ("\0", reverse),
     * UINT64_MAX = above everything ("\xff", forward).  sort_keymaker != 0 selects this scale. */
    int sort_keymaker;
    uint64_t sort_missing;
} orc_query;

typedef struct orc_mset {
    uint32_t n;
    uint32_t* docids;
    double* weights;
    uint64_t* sortvals;       /* numeric sort value per item (when sort_by != REL) */
    uint32_t matches_lower_bound, matches_estimated, matches_upper_bound;
    uint32_t known_matching_docs;
    uint32_t exact_matches;   /* docs matching the boolean structure (all of them) */
    double max_possible, max_attained, percent_scale_factor;
} orc_mset;

orc_index* orc_index_synthetic(uint32_t N, uint32_t V, uint64_t seed, uint32_t nshards, uint32_t shard,
                               int with_values);
orc_index* orc_index_load_flat(const char* path);
void orc_index_free(orc_index*);
/* Drop slot-0 values of documents whose smallest value is a multiple of mod0 and slot-1 values that are
 * multiples of mod1 (0 = keep all) — the rule of `ref_runner build --mvalues-sparse`. */
void orc_index_make_sparse(orc_index*, uint32_t mod0, uint32_t mod1);
/* Give slot 0 the values of a hand-made corpus (an XGMFLAT1 file carries none): nvals[lastdocid + 1] values per
 * document (0..3), vals[3 * (lastdocid + 1)] ascending per document.  Both are copied. */
void orc_index_set_slot0(orc_index*, const uint8_t* nvals, const uint64_t* vals);
int orc_term_lookup(const orc_index*, const char* name, uint32_t* id);

void orc_query_defaults(orc_query* q);
void orc_bm25_init(uint32_t collection_size, uint64_t total_length, uint32_t termfreq, uint32_t wqf,
                   double factor, double k1, double k3, double b, double* termweight, double* len_factor);
double orc_bm25_sumpart(double termweight, double len_factor, double k1, double b, double min_normlen,
                        uint32_t wdf, uint32_t len);
double orc_bm25_maxpart(double termweight, double len_factor, double k1, double b, double min_normlen,
                        uint32_t wdf_ub, uint32_t doclen_lb);

/* Run one query; result arrays are malloc'd, free with orc_mset_free. Returns 0 on success. */
int orc_match(const orc_index*, const orc_query*, orc_mset* out);
/* Matcher::merge_mset over per-shard msets whose docids are already unsharded. */
int orc_merge(const orc_mset* parts, uint32_t nparts, uint32_t first, uint32_t maxitems, int sort_by,
              int sort_reverse, orc_mset* out);
void orc_mset_free(orc_mset*);
uint32_t orc_round_estimate(uint32_t lb, uint32_t ub, uint32_t est);

/* AND evaluation order (ascending termfreq, libstdc++ partial_sort_copy tie behaviour) and OR tree
 * (postfix program: value >= 0 → leaf index into the query's term array, -1 → add the two
 * operands below), exported for the host-side planner's own tests. */
void orc_and_order(const uint32_t* termfreq, uint32_t n, uint32_t* order);
uint32_t orc_or_program(const uint32_t* termfreq, uint32_t n, int32_t* prog /* [2n-1] */);

#ifdef __cplusplus
}
#endif
#endif
