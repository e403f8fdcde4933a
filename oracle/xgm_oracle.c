/* oracle/xgm_oracle.c — TEST INFRASTRUCTURE, not product code (see xgm_oracle.h).
 *
 * Sequential restatement of the reference hot path over flat posting arrays.  Every function
 * cites the reference file:line (paths relative to /root/reference/src/xapian unless noted) whose
 * behaviour it restates.  Compile with -O2 -ffp-contract=off: the reference is built without FMA
 * contraction (CMakeLists.txt:99-104, plain x86-64), and the weights below must be bit-identical.
 */
#include "xgm_oracle.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../xapiand_b200/csrc/xgm_corpus.h"

/* ------------------------------------------------------------------ index construction */

static void* xcalloc(size_t n, size_t sz) {
    void* p = calloc(n ? n : 1, sz);
    if (!p) { fprintf(stderr, "oracle: out of memory\n"); abort(); }
    return p;
}

/* reference GlassPostListTable::get_freqs wdf upper bound, backends/glass/glass_postlist.cc:175-190
 * combined with GlassDatabase::get_wdf_upper_bound, backends/glass/glass_database.cc:822-829:
 *   min( cf==0||tf==1 ? cf : max(cf - first_wdf, first_wdf), db_wdf_ubound )
 * where db_wdf_ubound is the largest wdf ever added (GlassVersion::check_wdf,
 * backends/glass/glass_version.h:269-271). */
static uint32_t wdf_upper_bound(uint32_t tf, uint64_t cf, uint32_t first_wdf, uint32_t db_wdf_ub) {
    uint64_t ub;
    if (cf == 0 || tf == 1) ub = cf;
    else ub = (cf - first_wdf > first_wdf) ? cf - first_wdf : first_wdf;
    if (ub > db_wdf_ub) ub = db_wdf_ub;
    return (uint32_t)ub;
}

orc_index* orc_index_synthetic(uint32_t N, uint32_t V, uint64_t seed, uint32_t nshards, uint32_t shard,
                               int with_values) {
    xgm_zipf z;
    if (xgm_zipf_init(&z, V)) return NULL;
    orc_index* ix = (orc_index*)xcalloc(1, sizeof(*ix));
    uint32_t nlocal = 0;
    for (uint32_t d = shard + 1; d <= N; d += nshards) ++nlocal;
    ix->doccount = ix->lastdocid = nlocal;
    ix->nterms = V;
    ix->doclen = (uint32_t*)xcalloc((size_t)nlocal + 1, 4);
    ix->off = (uint64_t*)xcalloc((size_t)V + 1, 8);
    ix->collfreq = (uint64_t*)xcalloc(V, 8);
    ix->wdf_ub = (uint32_t*)xcalloc(V, 4);
    ix->names = (char**)xcalloc(V, sizeof(char*));
    if (with_values) {
        ix->nvals0 = (uint8_t*)xcalloc((size_t)nlocal + 1, 1);
        ix->vals0 = (uint64_t*)xcalloc(3 * ((size_t)nlocal + 1), 8);
        ix->val1 = (uint64_t*)xcalloc((size_t)nlocal + 1, 8);
    }
    uint32_t ranks[XGM_CORPUS_MAX_LEN], wdf[XGM_CORPUS_MAX_LEN];
    /* pass 1: count postings per term */
    uint32_t local = 0;
    ix->doclen_lb = 0xffffffffu;
    for (uint32_t d = shard + 1; d <= N; d += nshards) {
        ++local;
        uint32_t len = xgm_corpus_doc(&z, seed, d, ranks);
        uint32_t n = xgm_corpus_collapse(ranks, len, wdf);
        for (uint32_t i = 0; i < n; ++i) ix->off[ranks[i] + 1]++;
        ix->doclen[local] = len;
        ix->total_length += len;
        if (len < ix->doclen_lb) ix->doclen_lb = len;
        if (len > ix->doclen_ub) ix->doclen_ub = len;
    }
    if (nlocal == 0) ix->doclen_lb = 0;
    for (uint32_t t = 0; t < V; ++t) ix->off[t + 1] += ix->off[t];
    uint64_t total = ix->off[V];
    ix->docids = (uint32_t*)xcalloc(total, 4);
    ix->wdfs = (uint32_t*)xcalloc(total, 4);
    uint64_t* cur = (uint64_t*)xcalloc(V, 8);
    memcpy(cur, ix->off, (size_t)V * 8);
    local = 0;
    for (uint32_t d = shard + 1; d <= N; d += nshards) {
        ++local;
        uint32_t len = xgm_corpus_doc(&z, seed, d, ranks);
        uint32_t n = xgm_corpus_collapse(ranks, len, wdf);
        for (uint32_t i = 0; i < n; ++i) {
            uint64_t p = cur[ranks[i]]++;
            ix->docids[p] = local;
            ix->wdfs[p] = wdf[i];
            ix->collfreq[ranks[i]] += wdf[i];
        }
        if (with_values) {
            uint64_t v0[3], v1;
            uint32_t n0 = xgm_corpus_values(seed, d, v0, &v1);
            ix->nvals0[local] = (uint8_t)n0;
            for (uint32_t i = 0; i < n0; ++i) ix->vals0[3 * (size_t)local + i] = v0[i];
            ix->val1[local] = v1;
        }
    }
    free(cur);
    uint32_t db_wdf_ub = 0;
    for (uint64_t p = 0; p < total; ++p) if (ix->wdfs[p] > db_wdf_ub) db_wdf_ub = ix->wdfs[p];
    for (uint32_t t = 0; t < V; ++t) {
        char b[16];
        int k = xgm_corpus_term(t, b);
        ix->names[t] = (char*)xcalloc((size_t)k + 1, 1);
        memcpy(ix->names[t], b, (size_t)k);
        uint32_t tf = (uint32_t)(ix->off[t + 1] - ix->off[t]);
        ix->wdf_ub[t] = tf ? wdf_upper_bound(tf, ix->collfreq[t], ix->wdfs[ix->off[t]], db_wdf_ub) : 0;
    }
    xgm_zipf_free(&z);
    return ix;
}

static int rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n ? 0 : -1; }

/* XGMFLAT1 as written by oracle/ref_runner.cc `export` (public Xapian iterators over a glass DB) */
orc_index* orc_index_load_flat(const char* path) {
    FILE* f = fopen(path, "rb");
    if (!f) return NULL;
    char magic[8];
    orc_index* ix = (orc_index*)xcalloc(1, sizeof(*ix));
    uint32_t nslots;
    if (rd(f, magic, 8) || memcmp(magic, "XGMFLAT1", 8)) goto bad;
    if (rd(f, &ix->doccount, 4) || rd(f, &ix->lastdocid, 4) || rd(f, &ix->total_length, 8) ||
        rd(f, &ix->nterms, 4) || rd(f, &nslots, 4) || rd(f, &ix->doclen_lb, 4) || rd(f, &ix->doclen_ub, 4))
        goto bad;
    ix->doclen = (uint32_t*)xcalloc((size_t)ix->lastdocid + 1, 4);
    if (rd(f, ix->doclen, ((size_t)ix->lastdocid + 1) * 4)) goto bad;
    ix->off = (uint64_t*)xcalloc((size_t)ix->nterms + 1, 8);
    ix->collfreq = (uint64_t*)xcalloc(ix->nterms, 8);
    ix->wdf_ub = (uint32_t*)xcalloc(ix->nterms, 4);
    ix->names = (char**)xcalloc(ix->nterms, sizeof(char*));
    size_t cap = 1024, used = 0;
    ix->docids = (uint32_t*)malloc(cap * 4);
    ix->wdfs = (uint32_t*)malloc(cap * 4);
    for (uint32_t t = 0; t < ix->nterms; ++t) {
        uint32_t nl, tf, wub, n;
        uint64_t cf;
        if (rd(f, &nl, 4)) goto bad;
        ix->names[t] = (char*)xcalloc((size_t)nl + 1, 1);
        if (rd(f, ix->names[t], nl) || rd(f, &tf, 4) || rd(f, &cf, 8) || rd(f, &wub, 4) || rd(f, &n, 4)) goto bad;
        if (used + n > cap) {
            while (used + n > cap) cap *= 2;
            ix->docids = (uint32_t*)realloc(ix->docids, cap * 4);
            ix->wdfs = (uint32_t*)realloc(ix->wdfs, cap * 4);
        }
        if (rd(f, ix->docids + used, (size_t)n * 4) || rd(f, ix->wdfs + used, (size_t)n * 4)) goto bad;
        ix->off[t] = used;
        used += n;
        ix->collfreq[t] = cf;
        ix->wdf_ub[t] = wub;
        (void)tf;
    }
    ix->off[ix->nterms] = used;
    /* value slots are decoded by the python side when needed (sortable_serialise strings) */
    fclose(f);
    return ix;
bad:
    fclose(f);
    orc_index_free(ix);
    return NULL;
}

void orc_index_free(orc_index* ix) {
    if (ix) free(ix->has1);
    if (!ix) return;
    if (ix->names) for (uint32_t t = 0; t < ix->nterms; ++t) free(ix->names[t]);
    free(ix->names); free(ix->doclen); free(ix->off); free(ix->docids); free(ix->wdfs);
    free(ix->collfreq); free(ix->wdf_ub); free(ix->nvals0); free(ix->vals0); free(ix->val1);
    free(ix);
}

int orc_term_lookup(const orc_index* ix, const char* name, uint32_t* id) {
    for (uint32_t t = 0; t < ix->nterms; ++t)
        if (strcmp(ix->names[t], name) == 0) { *id = t; return 0; }
    return -1;
}

/* ------------------------------------------------------------------ BM25 (a4, a5, a6) */

void orc_query_defaults(orc_query* q) {
    memset(q, 0, sizeof(*q));
    /* weight.h:665-667 */
    q->k1 = 1.0; q->k3 = 1.0; q->b = 0.5; q->min_normlen = 0.5;
    q->maxitems = 10;
}

/* Weight::init_ weight/weight.cc:59-83 + BM25Weight::init weight/bm25weight.cc:46-130 (no RSet) */
void orc_bm25_init(uint32_t collection_size, uint64_t total_length, uint32_t termfreq, uint32_t wqf,
                   double factor, double k1, double k3, double b, double* termweight, double* len_factor) {
    double tw = ((double)(collection_size - termfreq) + 0.5) / ((double)termfreq + 0.5);
    if (tw < 2) tw = tw * 0.5 + 1;
    double w = log(tw) * factor;
    if (k3 != 0) {
        double wqf_double = wqf;
        w *= (k3 + 1) * wqf_double / (k3 + wqf_double);
    }
    w *= (k1 + 1);
    *termweight = w;
    /* k2 == 0 here (Xapiand never changes the default, SURVEY.md §2) */
    if (b == 0 || k1 == 0) {
        *len_factor = 0;
    } else {
        /* Weight::Internal::get_average_length weight/weightinternal.h:235-240 */
        double avg = collection_size == 0 ? 0.0 : (double)total_length / collection_size;
        *len_factor = avg != 0 ? 1 / avg : 0;
    }
}

/* BM25Weight::get_sumpart weight/bm25weight.cc:170-181 — this exact operation order */
double orc_bm25_sumpart(double termweight, double len_factor, double k1, double b, double min_normlen,
                        uint32_t wdf, uint32_t len) {
    double normlen = len * len_factor;
    if (normlen < min_normlen) normlen = min_normlen;
    double wdf_double = wdf;
    double denom = k1 * (normlen * b + (1 - b)) + wdf_double;
    return termweight * (wdf_double / denom);
}

/* BM25Weight::get_maxpart weight/bm25weight.cc:183-207 */
double orc_bm25_maxpart(double termweight, double len_factor, double k1, double b, double min_normlen,
                        uint32_t wdf_ub, uint32_t doclen_lb) {
    double denom = k1;
    if (k1 != 0.0 && b != 0.0) {
        uint32_t m = wdf_ub > doclen_lb ? wdf_ub : doclen_lb;
        double normlen_lb = m * len_factor;
        if (normlen_lb < min_normlen) normlen_lb = min_normlen;
        denom *= (normlen_lb * b + (1 - b));
    }
    double wdf_max = wdf_ub;
    denom += wdf_max;
    return termweight * (wdf_max / denom);
}

/* ------------------------------------------------------------------ evaluation order */

/* MultiAndPostList ctor, matcher/multiandpostlist.h:118-131: std::partial_sort_copy of all children
 * by ascending termfreq estimate.  With equal range sizes libstdc++ copies, make_heap()s and
 * sort_heap()s (bits/stl_algo.h __partial_sort_copy, bits/stl_heap.h); equal keys therefore land
 * in heapsort order, restated here so ties match the reference build (g++ 13). */
typedef struct { uint32_t tf, idx; } tf_ent;

static void gnu_push_heap(tf_ent* a, long hole, long top, tf_ent v) {
    long parent = (hole - 1) / 2;
    while (hole > top && a[parent].tf < v.tf) {
        a[hole] = a[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    a[hole] = v;
}

static void gnu_adjust_heap(tf_ent* a, long hole, long len, tf_ent v) {
    const long top = hole;
    long child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (a[child].tf < a[child - 1].tf) --child;
        a[hole] = a[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        a[hole] = a[child - 1];
        hole = child - 1;
    }
    gnu_push_heap(a, hole, top, v);
}

void orc_and_order(const uint32_t* termfreq, uint32_t n, uint32_t* order) {
    tf_ent* a = (tf_ent*)xcalloc(n, sizeof(tf_ent));
    for (uint32_t i = 0; i < n; ++i) { a[i].tf = termfreq[i]; a[i].idx = i; }
    if (n > 1) {
        /* make_heap */
        long len = n;
        for (long parent = (len - 2) / 2;; --parent) {
            tf_ent v = a[parent];
            gnu_adjust_heap(a, parent, len, v);
            if (parent == 0) break;
        }
        /* sort_heap */
        for (long last = len; last > 1; --last) {
            tf_ent v = a[last - 1];
            a[last - 1] = a[0];
            gnu_adjust_heap(a, 0, last - 1, v);
        }
    }
    for (uint32_t i = 0; i < n; ++i) order[i] = a[i].idx;
    free(a);
}

/* OrContext::postlist api/queryinternal.cc:440-489 with the reference's own heap, common/heap.h
 * (libc++-style make/pop/replace; comparator a.tf > b.tf, queryinternal.cc:142-147), replayed on
 * (node, termfreq) pairs. Output: postfix program. */
typedef struct { uint32_t tf; int32_t node; } or_ent;

static int or_cmp(const or_ent* a, const or_ent* b) { return a->tf > b->tf; }

static void or_sift_down(or_ent* first, long len, long start) {
    long child = start;
    if (len < 2 || (len - 2) / 2 < child) return;
    child = 2 * child + 1;
    if (child + 1 < len && or_cmp(&first[child], &first[child + 1])) ++child;
    if (or_cmp(&first[child], &first[start])) return;
    or_ent top = first[start];
    do {
        first[start] = first[child];
        start = child;
        if ((len - 2) / 2 < child) break;
        child = 2 * child + 1;
        if (child + 1 < len && or_cmp(&first[child], &first[child + 1])) ++child;
    } while (!or_cmp(&first[child], &top));
    first[start] = top;
}

uint32_t orc_or_program(const uint32_t* termfreq, uint32_t n, int32_t* prog) {
    /* nodes: 0..n-1 leaves; internal nodes appended; children recorded then emitted postfix */
    if (n == 0) return 0;
    if (n == 1) { prog[0] = 0; return 1; }
    or_ent* h = (or_ent*)xcalloc(n, sizeof(or_ent));
    int32_t* lch = (int32_t*)xcalloc(2 * n, 4);
    int32_t* rch = (int32_t*)xcalloc(2 * n, 4);
    for (uint32_t i = 0; i < n; ++i) { h[i].tf = termfreq[i]; h[i].node = (int32_t)i; }
    long len = n;
    for (long s = (len - 2) / 2; s >= 0; --s) or_sift_down(h, len, s); /* Heap::make */
    int32_t next = (int32_t)n, root = -1;
    for (;;) {
        int32_t r = h[0].node;
        uint32_t tf = h[0].tf;
        /* Heap::pop: swap first/last, sift down over len-1 */
        or_ent t = h[0]; h[0] = h[len - 1]; h[len - 1] = t;
        or_sift_down(h, len - 1, 0);
        --len;
        int32_t node = next++;
        lch[node] = h[0].node;
        rch[node] = r;
        if (len == 1) { root = node; break; }
        h[0].node = node;
        h[0].tf += tf;
        or_sift_down(h, len, 0); /* Heap::replace */
    }
    /* emit postfix: iterative */
    uint32_t np = 0;
    int32_t* stack = (int32_t*)xcalloc(4 * n, 4);
    long sp = 0;
    stack[sp++] = root;
    /* post-order via two-stack trick: produce reverse of (node, right, left) */
    int32_t* outrev = (int32_t*)xcalloc(2 * n, 4);
    uint32_t nr = 0;
    while (sp) {
        int32_t x = stack[--sp];
        outrev[nr++] = x;
        if (x >= (int32_t)n) { stack[sp++] = lch[x]; stack[sp++] = rch[x]; }
    }
    for (uint32_t i = nr; i-- > 0;) prog[np++] = outrev[i] < (int32_t)n ? outrev[i] : -1;
    free(h); free(lch); free(rch); free(stack); free(outrev);
    return np;
}

/* ------------------------------------------------------------------ matching */

typedef struct {
    double w;
    uint32_t did;
    uint64_t key;
} res_t;

typedef struct {
    int sort_by, reverse;
} cmp_t;

/* msetcmp.cc:54-61 (relevance), :64-72 (value), :75-85 (value then relevance), :88-98; docid order
 * ascending (sort_forward). The numeric key stands for the sortable_serialise byte string, which
 * is order-preserving (api/sortable-serialise.cc). Returns 1 when a ranks before b. */
static int mcmp(const cmp_t* c, const res_t* a, const res_t* b) {
    if (c->sort_by == ORC_SORT_VAL_REL || c->sort_by == ORC_SORT_VAL) {
        if (a->key > b->key) return c->reverse;
        if (a->key < b->key) return !c->reverse;
        if (c->sort_by == ORC_SORT_VAL) return a->did < b->did;
    }
    if (a->w > b->w) return 1;
    if (a->w < b->w) return 0;
    if (c->sort_by == ORC_SORT_REL_VAL) {
        if (a->key > b->key) return c->reverse;
        if (a->key < b->key) return !c->reverse;
    }
    return a->did < b->did;
}

static const cmp_t* g_cmp;
static int qsort_mcmp(const void* a, const void* b) {
    const res_t* x = (const res_t*)a; const res_t* y = (const res_t*)b;
    if (mcmp(g_cmp, x, y)) return -1;
    if (mcmp(g_cmp, y, x)) return 1;
    return 0;
}

/* ProtoMSet (matcher/protomset.h) without collapsing / percent cutoff / decider. The reference
 * keeps a lazily built min-heap of indices; because mcmp is a strict total order on distinct
 * docids the observable behaviour only depends on "which element is currently worst", which a
 * linear scan reproduces. */
typedef struct {
    res_t* results;
    uint32_t size, max_size, check_at_least;
    int heap_built;
    uint32_t worst;
    double min_weight, max_weight;
    uint32_t max_weight_subqs;
    uint32_t known_matching_docs;
    cmp_t cmp;
} proto_t;

static void proto_find_worst(proto_t* p) {
    uint32_t w = 0;
    for (uint32_t i = 1; i < p->size; ++i)
        if (mcmp(&p->cmp, &p->results[w], &p->results[i])) w = i;
    p->worst = w;
}

/* protomset.h:174-183 */
static void proto_update_max_weight(proto_t* p, double w, uint32_t subqs) {
    if (w <= p->max_weight) return;
    p->max_weight = w;
    p->max_weight_subqs = subqs;
}

/* protomset.h:185-194 (no time limit) */
static int proto_checked_enough(const proto_t* p) { return p->known_matching_docs >= p->check_at_least; }

/* protomset.h:340-400 */
static void proto_add(proto_t* p, const res_t* item, uint32_t subqs) {
    ++p->known_matching_docs;
    if (item->w < p->min_weight) return;
    if (item->w > p->max_weight) proto_update_max_weight(p, item->w, subqs);
    if (p->size < p->max_size) { p->results[p->size++] = *item; return; }
    int weight_first = (p->cmp.sort_by == ORC_SORT_REL || p->cmp.sort_by == ORC_SORT_REL_VAL);
    if (!p->heap_built) {
        if (p->size == 0) return;
        p->heap_built = 1;
        proto_find_worst(p);
        if (weight_first && proto_checked_enough(p)) p->min_weight = p->results[p->worst].w;
    }
    if (!mcmp(&p->cmp, item, &p->results[p->worst])) return;
    p->results[p->worst] = *item;
    proto_find_worst(p);
    if (weight_first && proto_checked_enough(p)) p->min_weight = p->results[p->worst].w;
}

/* protomset.h:248-288 (no collapser, no spies) */
static int proto_early_reject(proto_t* p, const res_t* item, uint32_t subqs) {
    if (!p->heap_built) return 0;
    if (mcmp(&p->cmp, item, &p->results[p->worst])) return 0;
    ++p->known_matching_docs;
    proto_update_max_weight(p, item->w, subqs);
    return 1;
}

static int pass_filter(const orc_index* ix, const orc_query* q, uint32_t did) {
    if (q->filter == ORC_FILTER_NONE) return 1;
    if (!ix->nvals0 || ix->nvals0[did] == 0) return 0;
    const uint64_t* v = ix->vals0 + 3 * (size_t)did;
    uint32_t n = ix->nvals0[did];
    if (q->filter == ORC_FILTER_VALUE_RANGE_MIN) {
        /* stock OP_VALUE_RANGE on the single-valued slot holding the smallest value:
         * ValueRangePostList::next matcher/valuerangepostlist.cc:132-151: begin <= v && v <= end */
        return v[0] >= q->range_lo && v[0] <= q->range_hi;
    }
    /* Xapiand MultipleValueRange::insideRange, /root/reference/src/multivalue/range.cc:351-368:
     * values are stored sorted; the doc matches iff the first value >= start is <= end */
    for (uint32_t i = 0; i < n; ++i)
        if (v[i] >= q->range_lo) return v[i] <= q->range_hi;
    return 0;
}

static uint64_t sort_value(const orc_index* ix, const orc_query* q, uint32_t did) {
    if (!ix->nvals0) return 0;
    if (q->sort_keymaker) {
        /* SerialiseKey::findSmallest / findBiggest, src/multivalue/keymaker.cc:67-92: first / last value of the
         * slot's StringList, MAX_STR_CMPVALUE / MIN_STR_CMPVALUE when the document has none */
        switch (q->sort_slot) {
            case 0: return ix->nvals0[did] ? ix->vals0[3 * (size_t)did] + 1 : q->sort_missing;
            case 2: return ix->nvals0[did] ? ix->vals0[3 * (size_t)did + ix->nvals0[did] - 1] + 1 : q->sort_missing;
            default: return (!ix->has1 || ix->has1[did]) ? ix->val1[did] + 1 : q->sort_missing;
        }
    }
    switch (q->sort_slot) {
        case 0: return ix->vals0[3 * (size_t)did];
        case 2: return ix->vals0[3 * (size_t)did + (ix->nvals0[did] ? ix->nvals0[did] - 1 : 0)];
        default: return ix->val1[did];
    }
}

void orc_index_make_sparse(orc_index* ix, uint32_t mod0, uint32_t mod1) {
    if (!ix || !ix->nvals0) return;
    if (!ix->has1) {
        ix->has1 = (uint8_t*)xcalloc((size_t)ix->lastdocid + 1, 1);
        memset(ix->has1, 1, (size_t)ix->lastdocid + 1);
    }
    for (uint32_t d = 1; d <= ix->lastdocid; ++d) {
        if (mod0 && ix->nvals0[d] && ix->vals0[3 * (size_t)d] % mod0 == 0) ix->nvals0[d] = 0;
        if (mod1 && ix->val1[d] % mod1 == 0) ix->has1[d] = 0;
    }
}

void orc_index_set_slot0(orc_index* ix, const uint8_t* nvals, const uint64_t* vals) {
    if (!ix) return;
    const size_t n = (size_t)ix->lastdocid + 1;
    if (!ix->nvals0) {
        ix->nvals0 = (uint8_t*)xcalloc(n, 1);
        ix->vals0 = (uint64_t*)xcalloc(3 * n, 8);
        ix->val1 = (uint64_t*)xcalloc(n, 8);
    }
    memcpy(ix->nvals0, nvals, n);
    memcpy(ix->vals0, vals, 3 * n * 8);
}

/* (termfreq min, max, est, max weight) of a subtree, as the reference's PostList classes report them */
typedef struct { uint32_t mn, mx, est; double maxw; } node_t;

/* OrContext::postlist (api/queryinternal.cc:440-489) over leaves with termfreqs tf[] and max weights mw[]
 * (NULL = unweighted): OrPostList::get_termfreq_min/max/est (matcher/orpostlist.cc:80-83,353-384) and
 * recalc_maxweight (l_max + r_max) folded over the Huffman-shaped tree.  prog (size 2n) receives the
 * postfix program. */
static node_t or_tree_node(const uint32_t* tf, const double* mw, uint32_t n, uint32_t doccount, int32_t* prog,
                           uint32_t* nprog_out) {
    node_t r;
    uint32_t nprog = orc_or_program(tf, n, prog);
    if (nprog_out) *nprog_out = nprog;
    double dbsize = doccount;
    node_t* st = (node_t*)xcalloc(2 * n + 2, sizeof(node_t));
    uint32_t sp = 0;
    for (uint32_t i = 0; i < nprog; ++i) {
        if (prog[i] >= 0) {
            st[sp].mn = st[sp].mx = st[sp].est = tf[prog[i]];
            st[sp].maxw = mw ? mw[prog[i]] : 0.0;
            ++sp;
        } else {
            --sp;
            node_t* l = &st[sp - 1];
            const node_t* rr = &st[sp];
            l->maxw = l->maxw + rr->maxw;
            l->mn = l->mn > rr->mn ? l->mn : rr->mn;
            uint32_t t = l->mx + rr->mx;
            if (t > doccount || t < l->mx) t = doccount;
            l->mx = t;
            double a = (double)l->est, b2 = (double)rr->est;
            l->est = dbsize == 0.0 ? 0 : (uint32_t)(a + b2 - (a * b2 / dbsize) + 0.5);
        }
    }
    r = st[0];
    free(st);
    return r;
}

/* MultiAndPostList over two subtrees (QueryFilter::postlist): get_termfreq_min/max/est
 * matcher/multiandpostlist.cc:55-105 with the children in ascending-estimate order; the maximum weight is
 * the sum of the children's (one of them is 0 here, so the order of the sum is immaterial). */
static node_t and_pair_node(node_t a, node_t b, uint32_t doccount) {
    node_t c0 = a, c1 = b, r;
    if (b.est < a.est) { c0 = b; c1 = a; }
    uint32_t sum = c0.mn;
    if (sum) {
        uint32_t old = sum;
        sum += c1.mn;
        if (sum >= old && sum <= doccount) sum = 0;
        else sum -= doccount;
    }
    r.mn = sum;
    r.mx = c0.mx < c1.mx ? c0.mx : c1.mx;
    double e = doccount ? ((double)c0.est * (double)c1.est) / (double)doccount : 0.0;
    r.est = doccount ? (uint32_t)(e + 0.5) : 0;
    r.maxw = c0.maxw + c1.maxw;
    return r;
}

/* The range of OP_FILTER(base, range) as a MultiAndPostList child.  A MultipleValueRange source has termfreqs
 * (min, est, max) = (0, vf, vf) (range.cc:457-464, api/postingsource.cc:201-214).  A stock OP_VALUE_RANGE has
 * max = vf and min = vf when [lo, hi] covers every value in the slot, 0 otherwise (valuerangepostlist.cc:40-54,
 * 145-148); its string-fraction estimate (valuerangepostlist.cc:70-130) is not restated and vf stands in for it. */
static node_t range_child_node(const orc_index* ix, const orc_query* q) {
    uint32_t vf = 0;
    uint64_t lo = ~0ull, hi = 0;
    if (ix->nvals0)
        for (uint32_t d = 1; d <= ix->lastdocid; ++d) {
            if (!ix->nvals0[d]) continue;
            const uint64_t v = ix->vals0[3 * (size_t)d];
            ++vf;
            if (v < lo) lo = v;
            if (v > hi) hi = v;
        }
    node_t r;
    r.mn = q->filter == ORC_FILTER_VALUE_RANGE_MIN && vf && q->range_lo <= lo && hi <= q->range_hi ? vf : 0;
    r.mx = r.est = vf;
    r.maxw = 0.0;
    return r;
}

static int list_contains(const uint32_t* d, uint32_t n, uint32_t did, uint32_t* where) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { uint32_t m = (lo + hi) / 2; if (d[m] < did) lo = m + 1; else hi = m; }
    if (where) *where = lo;
    return lo < n && d[lo] == did;
}

int orc_match(const orc_index* ix, const orc_query* qin, orc_mset* out) {
    memset(out, 0, sizeof(*out));
    /* BM25Weight's constructor, weight.h:639-646: k1, k3 < 0 become 0, b is clamped to [0, 1] */
    orc_query qc = *qin;
    if (qc.k1 < 0) qc.k1 = 0;
    if (qc.k3 < 0) qc.k3 = 0;
    if (qc.b < 0) qc.b = 0; else if (qc.b > 1) qc.b = 1;
    const orc_query* q = &qc;
    uint32_t n = q->nterms;
    if (n == 0 || n > 64) return -1;
    /* Enquire::Internal::get_mset clamping, api/enquire.cc:420-426 */
    uint32_t docs = ix->doccount;
    uint32_t first = q->first < docs ? q->first : docs;
    uint32_t maxitems = q->maxitems < docs - first ? q->maxitems : docs - first;
    uint32_t check_at_least = q->check_at_least < docs ? q->check_at_least : docs;
    if (check_at_least < first + maxitems) check_at_least = first + maxitems;

    const uint32_t** dl = (const uint32_t**)xcalloc(n, sizeof(void*));
    const uint32_t** wl = (const uint32_t**)xcalloc(n, sizeof(void*));
    uint32_t* len = (uint32_t*)xcalloc(n, 4);
    double* tw = (double*)xcalloc(n, 8);
    double len_factor = 0;
    double max_possible_leafsum = 0;
    double* maxpart = (double*)xcalloc(n, 8);
    uint32_t coll = q->stats ? q->stats->collection_size : ix->doccount;
    uint64_t tlen = q->stats ? q->stats->total_length : ix->total_length;
    for (uint32_t j = 0; j < n; ++j) {
        uint32_t t = q->terms[j];
        dl[j] = ix->docids + ix->off[t];
        wl[j] = ix->wdfs + ix->off[t];
        len[j] = (uint32_t)(ix->off[t + 1] - ix->off[t]);
        uint32_t gtf = q->stats ? q->stats->termfreq[j] : len[j];
        /* LocalSubMatch::open_post_list matcher/localsubmatch.cc:295-299: the leaf's factor is the product of
         * the OP_SCALE_WEIGHT factors above it (1.0 without any); factor 0 → no Weight object at all */
        const double factor = q->factors ? q->factors[j] : 1.0;
        orc_bm25_init(coll, tlen, gtf, q->wqf ? q->wqf[j] : 1, factor, q->k1, q->k3, q->b, &tw[j], &len_factor);
        maxpart[j] = orc_bm25_maxpart(tw[j], len_factor, q->k1, q->b, q->min_normlen, ix->wdf_ub[t], ix->doclen_lb);
        if (factor == 0.0) { tw[j] = 0.0; maxpart[j] = 0.0; }
        (void)max_possible_leafsum;
    }

    uint32_t* order = (uint32_t*)xcalloc(n, 4);
    int32_t* prog = (int32_t*)xcalloc(2 * n, 4);
    uint32_t nprog = 0;
    double max_possible = 0;
    uint32_t tf_min = 0, tf_est = 0, tf_max = 0;
    double dbsize = ix->doccount;
    uint32_t src_pos = 0xffffffffu; /* place of a weighted range source among the AND's children */
    double src_w = 0.0;
    if (q->op == ORC_OP_AND) {
        orc_and_order(len, n, order);
        if (q->filter != ORC_FILTER_NONE && !(q->nfilter || q->nnot || q->nmaybe)) {
            /* the range is one more child, sorted in by its termfreq estimate = value_freq */
            const node_t src = range_child_node(ix, q);
            const uint32_t vf = src.mx;
            uint32_t* cl = (uint32_t*)xcalloc(n + 1, 4);
            uint32_t* co = (uint32_t*)xcalloc(n + 1, 4);
            memcpy(cl, len, n * 4);
            cl[n] = vf;
            orc_and_order(cl, n + 1, co);
            src_w = q->filter_weighted ? (q->filter_factor != 0.0 ? q->filter_factor : 1.0) * 1.0 : 0.0;
            uint32_t k = 0;
            for (uint32_t i = 0; i <= n; ++i) { if (co[i] == n) src_pos = k; else order[k++] = co[i]; }
            for (uint32_t i = 0; i <= n; ++i)
                max_possible += co[i] == n ? (q->filter_weighted ? src_w * 1.7976931348623157e308 : 0.0) : maxpart[co[i]];
            #define CH_MIN(i) (co[i] == n ? src.mn : cl[co[i]])
            uint32_t sum = CH_MIN(0);
            if (sum) {
                for (uint32_t i = 1; i <= n; ++i) {
                    uint32_t old = sum;
                    sum += CH_MIN(i);
                    if (sum >= old && sum <= ix->doccount) { sum = 0; break; }
                    sum -= ix->doccount;
                }
            }
            #undef CH_MIN
            tf_min = sum;
            tf_max = cl[co[0]];
            for (uint32_t i = 1; i <= n; ++i) if (cl[co[i]] < tf_max) tf_max = cl[co[i]];
            double r = cl[co[0]];
            for (uint32_t i = 1; i <= n; ++i) r = (r * cl[co[i]]) / dbsize;
            tf_est = ix->doccount ? (uint32_t)(r + 0.5) : 0;
            free(cl); free(co);
        } else {
        /* MultiAndPostList::recalc_maxweight matcher/multiandpostlist.cc:161-171: sum in plist order */
        for (uint32_t i = 0; i < n; ++i) max_possible += maxpart[order[i]];
        /* get_termfreq_min/max/est multiandpostlist.cc:55-105 */
        uint32_t sum = len[order[0]];
        if (sum) {
            for (uint32_t i = 1; i < n; ++i) {
                uint32_t old = sum;
                sum += len[order[i]];
                if (sum >= old && sum <= ix->doccount) { sum = 0; break; }
                sum -= ix->doccount;
            }
        }
        tf_min = sum;
        tf_max = len[order[0]];
        for (uint32_t i = 1; i < n; ++i) if (len[order[i]] < tf_max) tf_max = len[order[i]];
        double r = len[order[0]];
        for (uint32_t i = 1; i < n; ++i) r = (r * len[order[i]]) / dbsize;
        tf_est = ix->doccount ? (uint32_t)(r + 0.5) : 0;
        }
    } else {
        nprog = orc_or_program(len, n, prog);
        /* OrPostList::recalc_maxweight orpostlist.cc:105-111 (l_max + r_max per node) and
         * get_termfreq_min/max/est orpostlist.cc:80-83,353-384, folded over the same tree */
        double* sm = (double*)xcalloc(2 * n, 8);
        double* se = (double*)xcalloc(2 * n, 8);
        uint32_t* smin = (uint32_t*)xcalloc(2 * n, 4);
        uint32_t* smax = (uint32_t*)xcalloc(2 * n, 4);
        uint32_t sp = 0;
        for (uint32_t i = 0; i < nprog; ++i) {
            if (prog[i] >= 0) {
                sm[sp] = maxpart[prog[i]];
                se[sp] = smin[sp] = smax[sp] = len[prog[i]];
                ++sp;
            } else {
                --sp; /* right operand at sp, left at sp-1 */
                sm[sp - 1] = sm[sp - 1] + sm[sp];
                smin[sp - 1] = smin[sp - 1] > smin[sp] ? smin[sp - 1] : smin[sp];
                uint32_t lm = smax[sp - 1], t = lm + smax[sp];
                if (t > ix->doccount || t < lm) t = ix->doccount;
                smax[sp - 1] = t;
                double a = (double)(uint32_t)se[sp - 1], b2 = (double)(uint32_t)se[sp];
                uint32_t e = dbsize == 0.0 ? 0 : (uint32_t)(a + b2 - (a * b2 / dbsize) + 0.5);
                se[sp - 1] = e;
            }
        }
        max_possible = sm[0]; tf_min = smin[0]; tf_max = smax[0]; tf_est = (uint32_t)se[0];
        free(sm); free(se); free(smin); free(smax);
        if (q->filter != ORC_FILTER_NONE) {
            /* QueryFilter::postlist: MultiAndPostList of [OrPostList tree, range] (api/queryinternal.cc:2271-2283);
             * the range weighs nothing, so max_possible stays the tree's */
            node_t cur; cur.mn = tf_min; cur.mx = tf_max; cur.est = tf_est; cur.maxw = max_possible;
            cur = and_pair_node(cur, range_child_node(ix, q), ix->doccount);
            tf_min = cur.mn; tf_max = cur.mx; tf_est = cur.est;
        }
    }

    /* §8(f)-1 groups around an AND base */
    const uint32_t nf = q->nfilter, nx = q->nnot, nm = q->nmaybe;
    if ((nf || nx || nm) && q->filter != ORC_FILTER_NONE) return -1;
    uint32_t* mlen = NULL; double* mtw = NULL; double* mmax = NULL; int32_t* mprog = NULL; uint32_t mnprog = 0;
    if (nf || nx || nm) {
        node_t cur; cur.mn = tf_min; cur.mx = tf_max; cur.est = tf_est; cur.maxw = max_possible;
        if (nf) {
            node_t f;
            uint32_t* fl = (uint32_t*)xcalloc(nf, 4);
            for (uint32_t i = 0; i < nf; ++i) fl[i] = (uint32_t)(ix->off[q->filter_terms[i] + 1] - ix->off[q->filter_terms[i]]);
            if (nf == 1) { f.mn = f.mx = f.est = fl[0]; }
            else {
                /* Query(OP_AND, boolean terms): a MultiAndPostList of unweighted leaves */
                uint32_t* fo = (uint32_t*)xcalloc(nf, 4);
                orc_and_order(fl, nf, fo);
                uint32_t sum = fl[fo[0]];
                if (sum) for (uint32_t i = 1; i < nf; ++i) {
                    uint32_t old = sum; sum += fl[fo[i]];
                    if (sum >= old && sum <= ix->doccount) { sum = 0; break; }
                    sum -= ix->doccount;
                }
                f.mn = sum;
                f.mx = fl[fo[0]];
                for (uint32_t i = 1; i < nf; ++i) if (fl[fo[i]] < f.mx) f.mx = fl[fo[i]];
                double r = fl[fo[0]];
                for (uint32_t i = 1; i < nf; ++i) r = (r * fl[fo[i]]) / dbsize;
                f.est = ix->doccount ? (uint32_t)(r + 0.5) : 0;
                free(fo);
            }
            f.maxw = 0.0;
            cur = and_pair_node(cur, f, ix->doccount);
            free(fl);
        }
        if (nx) {
            /* AndNotPostList::get_termfreq_min/max/est matcher/andnotpostlist.cc:30-62; the weight is the left's */
            uint32_t* xl = (uint32_t*)xcalloc(nx, 4);
            int32_t* xp = (int32_t*)xcalloc(2 * nx + 2, 4);
            for (uint32_t i = 0; i < nx; ++i) xl[i] = (uint32_t)(ix->off[q->not_terms[i] + 1] - ix->off[q->not_terms[i]]);
            node_t r;
            if (nx == 1) { r.mn = r.mx = r.est = xl[0]; r.maxw = 0; }
            else r = or_tree_node(xl, NULL, nx, ix->doccount, xp, NULL);
            node_t a = cur;
            cur.mn = a.mn <= r.mx ? 0 : a.mn - r.mx;
            cur.mx = ix->doccount - r.mn < a.mx ? ix->doccount - r.mn : a.mx;
            if (ix->doccount == 0) cur.est = 0;
            else {
                double e = a.est;
                e = (e * (double)(ix->doccount - r.est)) / (double)ix->doccount;
                cur.est = (uint32_t)(e + 0.5);
            }
            free(xl); free(xp);
        }
        if (nm) {
            /* AndMaybePostList: termfreqs are the left's (WrapperPostList), recalc_maxweight = pl_max + r_max
             * matcher/andmaybepostlist.cc:69-75 */
            mlen = (uint32_t*)xcalloc(nm, 4); mtw = (double*)xcalloc(nm, 8); mmax = (double*)xcalloc(nm, 8);
            mprog = (int32_t*)xcalloc(2 * nm + 2, 4);
            for (uint32_t i = 0; i < nm; ++i) {
                uint32_t t = q->maybe_terms[i];
                mlen[i] = (uint32_t)(ix->off[t + 1] - ix->off[t]);
                uint32_t gtf = (q->stats && q->stats->maybe_termfreq) ? q->stats->maybe_termfreq[i] : mlen[i];
                double lf;
                orc_bm25_init(coll, tlen, gtf, 1, 1.0, q->k1, q->k3, q->b, &mtw[i], &lf);
                mmax[i] = orc_bm25_maxpart(mtw[i], lf, q->k1, q->b, q->min_normlen, ix->wdf_ub[t], ix->doclen_lb);
            }
            node_t r;
            if (nm == 1) { r.maxw = mmax[0]; mprog[0] = 0; mnprog = 1; }
            else r = or_tree_node(mlen, mmax, nm, ix->doccount, mprog, &mnprog);
            cur.maxw = cur.maxw + r.maxw;
        }
        tf_min = cur.mn; tf_max = cur.mx; tf_est = cur.est; max_possible = cur.maxw;
    }

    proto_t P;
    memset(&P, 0, sizeof(P));
    P.max_size = first + maxitems;
    P.check_at_least = check_at_least;
    P.results = (res_t*)xcalloc((size_t)P.max_size + 1, sizeof(res_t));
    P.cmp.sort_by = q->sort_by;
    P.cmp.reverse = q->sort_reverse;
    uint32_t nweighted = 0; /* leaves with a Weight object: QueryTerm::postlist counts them only when factor != 0 */
    for (uint32_t j = 0; j < n; ++j) nweighted += (!q->factors || q->factors[j] != 0.0) ? 1u : 0u;
    uint32_t total_subqs = nweighted + nm; /* api/queryinternal.cc:1053-1054 */
    if (q->filter_weighted && q->filter == ORC_FILTER_MULTI_RANGE) ++total_subqs; /* QueryPostingSource::postlist, factor != 0 */

    /* a stock range covering every value of a slot that every document has is the all-documents list
     * (QueryValueRange::postlist api/queryinternal.cc:1116-1124), whose LeafPostList has no Weight: it matches no
     * subquery (leafpostlist.cc:88-91) */
    int filter_subq = q->filter != ORC_FILTER_NONE;
    if (q->filter == ORC_FILTER_VALUE_RANGE_MIN) {
        const node_t r = range_child_node(ix, q);
        if (r.mn != 0 && r.mn == ix->doccount) filter_subq = 0;
    }

    uint64_t* pos = (uint64_t*)xcalloc(n, 8);
    double* stk = (double*)xcalloc(2 * (n + nm) + 2, 8);
    int* stkp = (int*)xcalloc(2 * (n + nm) + 2, sizeof(int));
    uint32_t exact = 0;

    if (check_at_least != 0) {
        uint32_t did = 0;
        for (;;) {
            double weight = 0;
            uint32_t subqs = 0, doclen = 0;
            if (q->op == ORC_OP_AND) {
                /* MultiAndPostList::find_next_match matcher/multiandpostlist.cc:179-206 */
                uint32_t d0 = order[0];
                while (pos[d0] < len[d0] && dl[d0][pos[d0]] <= did) ++pos[d0];
                if (pos[d0] >= len[d0]) break;
                uint32_t cand = dl[d0][pos[d0]];
                int ok = 1, ended = 0;
                for (uint32_t i = 1; i < n; ++i) {
                    uint32_t j = order[i];
                    /* skip_to(cand): binary search from the current position */
                    uint64_t lo = pos[j], hi = len[j];
                    while (lo < hi) { uint64_t m = (lo + hi) / 2; if (dl[j][m] < cand) lo = m + 1; else hi = m; }
                    pos[j] = lo;
                    if (lo >= len[j]) { ended = 1; break; }
                    if (dl[j][lo] != cand) { ok = 0; break; }
                }
                if (ended) break;
                did = cand;
                if (!ok) continue;
                if (!pass_filter(ix, q, did)) continue;
                /* MultiAndPostList::get_weight multiandpostlist.cc:149-159: result = 0; += in plist order */
                doclen = ix->doclen[did];
                for (uint32_t i = 0; i < n; ++i) {
                    uint32_t j = order[i];
                    if (q->filter_weighted && src_pos == i) weight += src_w; /* ExternalPostList::get_weight */
                    /* LeafPostList::get_weight api/leafpostlist.cc:57-63: 0 for a leaf without a Weight, which
                     * get_sumpart is never asked about (at wdf 0 it would be 0 * (0 / 0)) */
                    if (q->factors && q->factors[j] == 0.0) continue;
                    weight += orc_bm25_sumpart(tw[j], len_factor, q->k1, q->b, q->min_normlen, wl[j][pos[j]], doclen);
                }
                if (q->filter_weighted && src_pos == n) weight += src_w;
                subqs = nweighted;
            } else {
                /* union in docid order; OrPostList::get_weight matcher/orpostlist.cc:93-103 folds
                 * l, r or l+r per node of the Huffman-shaped tree */
                uint32_t best = 0xffffffffu;
                for (uint32_t j = 0; j < n; ++j) {
                    while (pos[j] < len[j] && dl[j][pos[j]] <= did) ++pos[j];
                    if (pos[j] < len[j] && dl[j][pos[j]] < best) best = dl[j][pos[j]];
                }
                if (best == 0xffffffffu) break;
                did = best;
                if (!pass_filter(ix, q, did)) continue;
                doclen = ix->doclen[did];
                uint32_t sp = 0;
                for (uint32_t i = 0; i < nprog; ++i) {
                    if (prog[i] >= 0) {
                        uint32_t j = (uint32_t)prog[i];
                        if (pos[j] < len[j] && dl[j][pos[j]] == did) {
                            const int weighted = !q->factors || q->factors[j] != 0.0;
                            /* LeafPostList::get_weight: 0 without a Weight */
                            stk[sp] = weighted ? orc_bm25_sumpart(tw[j], len_factor, q->k1, q->b, q->min_normlen,
                                                                  wl[j][pos[j]], doclen) : 0.0;
                            stkp[sp] = 1;
                            if (weighted) ++subqs;
                        } else { stk[sp] = 0; stkp[sp] = 0; }
                        ++sp;
                    } else {
                        --sp;
                        if (stkp[sp - 1] && stkp[sp]) stk[sp - 1] = stk[sp - 1] + stk[sp];
                        else if (stkp[sp]) { stk[sp - 1] = stk[sp]; stkp[sp - 1] = 1; }
                    }
                }
                weight = stk[0];
            }
            if (nf || nx || nm) {
                int keep = 1;
                for (uint32_t i = 0; i < nf && keep; ++i) {
                    uint32_t t = q->filter_terms[i];
                    keep = list_contains(ix->docids + ix->off[t], (uint32_t)(ix->off[t + 1] - ix->off[t]), did, NULL);
                }
                for (uint32_t i = 0; i < nx && keep; ++i) {
                    uint32_t t = q->not_terms[i];
                    keep = !list_contains(ix->docids + ix->off[t], (uint32_t)(ix->off[t + 1] - ix->off[t]), did, NULL);
                }
                if (!keep) continue;
                if (nm) {
                    /* AndMaybePostList::get_weight matcher/andmaybepostlist.cc:59-67: l + (r if it matches);
                     * r is the OrPostList tree over the optional leaves (l, r or l + r per node) */
                    uint32_t sp = 0, present = 0;
                    for (uint32_t i = 0; i < mnprog; ++i) {
                        if (mprog[i] >= 0) {
                            uint32_t j = (uint32_t)mprog[i], t = q->maybe_terms[j], where;
                            if (list_contains(ix->docids + ix->off[t], mlen[j], did, &where)) {
                                stk[sp] = orc_bm25_sumpart(mtw[j], len_factor, q->k1, q->b, q->min_normlen,
                                                           ix->wdfs[ix->off[t] + where], doclen);
                                stkp[sp] = 1;
                                ++present;
                            } else { stk[sp] = 0; stkp[sp] = 0; }
                            ++sp;
                        } else {
                            --sp;
                            if (stkp[sp - 1] && stkp[sp]) stk[sp - 1] = stk[sp - 1] + stk[sp];
                            else if (stkp[sp]) { stk[sp - 1] = stk[sp]; stkp[sp - 1] = 1; }
                        }
                    }
                    if (present) { weight = weight + stk[0]; subqs += present; }
                }
            }
            ++exact;
            /* a value-range / posting-source filter is a matching subquery of every document it lets through
             * (ValueRangePostList / ExternalPostList::count_matching_subqs return 1) although, being unweighted,
             * it is not one of the total_subqs (api/queryinternal.cc:1097-1098): percentages of filtered
             * queries are scaled by (n+1)/n */
            if (filter_subq) ++subqs;
            /* main loop, matcher/matcher.cc:482-536 */
            if (weight < P.min_weight) continue;
            res_t item;
            item.w = weight; item.did = did; item.key = 0;
            if (q->sort_by != ORC_SORT_REL) {
                item.key = sort_value(ix, q, did);
                if (proto_early_reject(&P, &item, subqs)) continue;
            }
            proto_update_max_weight(&P, item.w, subqs); /* ProtoMSet::process protomset.h:295-299 */
            proto_add(&P, &item, subqs);
        }
    }

    /* ProtoMSet::finalise protomset.h:484-683 (no collapser / decider / percent threshold) */
    double percent_scale = 0;
    if (P.size != 0 && P.max_weight != 0.0) {
        percent_scale = P.max_weight_subqs / (double)total_subqs;
        percent_scale /= P.max_weight;
    }
    uint32_t lb = tf_min, est = tf_est, ub = tf_max;
    if (check_at_least == 0) {
        /* matcher.cc:437-461: bounds only */
    } else if (P.size != P.max_size) {
        lb = est = ub = P.size;
    } else if (P.known_matching_docs < check_at_least) {
        lb = est = ub = P.known_matching_docs;
    } else {
        if (P.known_matching_docs > lb) lb = P.known_matching_docs;
        if (P.known_matching_docs > est) est = P.known_matching_docs;
    }
    g_cmp = &P.cmp;
    qsort(P.results, P.size, sizeof(res_t), qsort_mcmp);
    uint32_t nout = P.size > first ? P.size - first : 0;
    out->n = nout;
    out->docids = (uint32_t*)xcalloc(nout, 4);
    out->weights = (double*)xcalloc(nout, 8);
    out->sortvals = (uint64_t*)xcalloc(nout, 8);
    for (uint32_t i = 0; i < nout; ++i) {
        out->docids[i] = P.results[first + i].did;
        out->weights[i] = P.results[first + i].w;
        out->sortvals[i] = P.results[first + i].key;
    }
    out->matches_lower_bound = lb;
    out->matches_estimated = est;
    out->matches_upper_bound = ub;
    out->known_matching_docs = P.known_matching_docs;
    out->exact_matches = exact;
    out->max_possible = max_possible;
    out->max_attained = P.max_weight;
    out->percent_scale_factor = percent_scale * 100.0;

    free(mlen); free(mtw); free(mmax); free(mprog);
    free(P.results); free(pos); free(stk); free(stkp); free(order); free(prog);
    free(dl); free(wl); free(len); free(tw); free(maxpart);
    return 0;
}

/* Matcher::merge_mset matcher/matcher.cc:653-782 + MSet::Internal::merge_stats api/mset.cc:376-395.
 * The k-way heap merge under a strict total order equals sort-and-slice of the concatenation. */
int orc_merge(const orc_mset* parts, uint32_t nparts, uint32_t first, uint32_t maxitems, int sort_by,
              int sort_reverse, orc_mset* out) {
    memset(out, 0, sizeof(*out));
    size_t total = 0;
    for (uint32_t i = 0; i < nparts; ++i) total += parts[i].n;
    res_t* all = (res_t*)xcalloc(total, sizeof(res_t));
    size_t k = 0;
    for (uint32_t i = 0; i < nparts; ++i) {
        const orc_mset* p = &parts[i];
        out->matches_lower_bound += p->matches_lower_bound;
        out->matches_estimated += p->matches_estimated;
        out->matches_upper_bound += p->matches_upper_bound;
        out->known_matching_docs += p->known_matching_docs;
        out->exact_matches += p->exact_matches;
        if (p->max_possible > out->max_possible) out->max_possible = p->max_possible;
        if (p->max_attained > out->max_attained) {
            out->max_attained = p->max_attained;
            out->percent_scale_factor = p->percent_scale_factor;
        }
        for (uint32_t j = 0; j < p->n; ++j) {
            all[k].w = p->weights[j]; all[k].did = p->docids[j];
            all[k].key = p->sortvals ? p->sortvals[j] : 0;
            ++k;
        }
    }
    cmp_t c; c.sort_by = sort_by; c.reverse = sort_reverse;
    g_cmp = &c;
    qsort(all, total, sizeof(res_t), qsort_mcmp);
    size_t nout = total > first ? total - first : 0;
    if (nout > maxitems) nout = maxitems;
    out->n = (uint32_t)nout;
    out->docids = (uint32_t*)xcalloc(nout, 4);
    out->weights = (double*)xcalloc(nout, 8);
    out->sortvals = (uint64_t*)xcalloc(nout, 8);
    for (size_t i = 0; i < nout; ++i) {
        out->docids[i] = all[first + i].did;
        out->weights[i] = all[first + i].w;
        out->sortvals[i] = all[first + i].key;
    }
    free(all);
    return 0;
}

/* round_estimate api/roundestimate.h:35-64, applied by MSet::get_matches_estimated api/mset.cc:145-153
 * (T = Xapian::doccount, unsigned 32-bit arithmetic) */
uint32_t orc_round_estimate(uint32_t m, uint32_t M, uint32_t e) {
    uint32_t D = M - m;
    if (D == 0 || e == 0) return e;
    int k = (int)log10((double)D);
    double p = 1.0;
    for (int i = 0; i < k; ++i) p *= 10.0;
    uint32_t r = (uint32_t)(p + 0.5);
    while (r > e) r /= 10;
    uint32_t R = e / r * r;
    if (R < m) {
        R += r;
    } else if (R > M) {
        R -= r;
    } else if (R < e && r % 2 == 0 && e - R == r / 2) {
        if (e - m < M - e) R += r;
    }
    if (R < m || R > M) R = e;
    return R;
}

void orc_mset_free(orc_mset* m) {
    free(m->docids); free(m->weights); free(m->sortvals);
    memset(m, 0, sizeof(*m));
}
