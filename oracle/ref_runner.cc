/* oracle/ref_runner.cc — TEST INFRASTRUCTURE, not product code.
 *
 * Driver for the UNMODIFIED reference matcher: links oracle/_ref/libxapian_ref.so (the reference's
 * vendored Xapian compiled from /root/reference/src/xapian by oracle/build_ref.sh) and calls only
 * its public API.  It is the oracle the CUDA path is checked against and the CPU baseline arm of
 * bench.py.  The product never links or executes this.
 *
 *   ref_runner build  --out DIR --docs N --vocab V --seed S [--nshards n --shard s] [--values | --mvalues]
 *                     [--termlist] [--range-first a --range-last b] [--boolean-terms K]
 *                                                       write a glass DB through WritableDatabase
 *                                                       (--range-*: only global docids a..b, as local 1..)
 *                                                       --mvalues: value slots the way Xapiand writes them —
 *                                                       slot 0 a StringList (src/serialise_list.h:301-356) of 1..3
 *                                                       Serialise::positive() keys, slot 1 one such key
 *   ref_runner compact --db DIR [--db DIR ...] --out DIR   Database::compact (renumbering by offset, so
 *                                                       contiguous docid-range parts give back the corpus)
 *   ref_runner query  --db DIR [--db DIR ...] [--twophase] --queries FILE [--threads T]
 *                     [--repeat R] [--dump FILE]        Enquire::get_mset over the query list
 *   ref_runner export --db DIR --out FILE               dump postings/doclens/values through the
 *                                                       public iterators (flat XGMFLAT1 file)
 *
 * Reference call sites this exercises: Enquire::get_mset (src/xapian/api/enquire.cc:396-470) and,
 * with --twophase, the prepare_mset / add_prepared_mset / set_prepared_mset / get_mset /
 * unshard_docids / merge_mset sequence of Xapiand's DocMatcher
 * (src/database/handler.cc:1250-1371, 1532-1551).
 */
#include <xapian.h>

/* Xapiand's own multivalue classes live in oracle/_ref/libxapiand_mv_ref.so (oracle/build_ref.sh); the factory
 * functions are oracle/ref_mv_glue.cc */
namespace xgmref {
std::string serialise_number(long double v);
std::string serialise_slot(const std::vector<std::string>& sorted_unique_values);
Xapian::PostingSource* make_multiple_value_range(unsigned slot, const std::string& start, const std::string& end);
Xapian::KeyMaker* make_key_maker(const std::vector<std::pair<unsigned, bool>>& slots);
}

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <fstream>
#include <mutex>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#include "../xapiand_b200/csrc/xgm_corpus.h"

#ifdef XGM_SHIM_RUNNER
/* linked against oracle/_ref/libxapian_ref_xgm.so: the same reference library with the xgm shim at the
 * Matcher::get_mset seam (xapiand_b200/shim/xgm_shim.h).  The dump records who answered each query. */
extern "C" int xgm_shim_last_served(void);
extern "C" unsigned xgm_shim_last_flags(void);
extern "C" const char* xgm_shim_last_reason(void);
#endif

using Clock = std::chrono::steady_clock;

static double now_s() {
    return std::chrono::duration<double>(Clock::now().time_since_epoch()).count();
}

[[noreturn]] static void die(const std::string& m) {
    fprintf(stderr, "ref_runner: %s\n", m.c_str());
    exit(2);
}

struct Args {
    std::vector<std::string> v;
    bool flag(const char* name) const {
        for (auto& s : v) if (s == name) return true;
        return false;
    }
    std::string get(const char* name, const char* def = nullptr) const {
        for (size_t i = 0; i + 1 < v.size(); ++i) if (v[i] == name) return v[i + 1];
        if (def) return def;
        die(std::string("missing ") + name);
    }
    std::vector<std::string> all(const char* name) const {
        std::vector<std::string> r;
        for (size_t i = 0; i + 1 < v.size(); ++i) if (v[i] == name) r.push_back(v[i + 1]);
        return r;
    }
};

/* ---------------------------------------------------------------- build */

static int cmd_build(const Args& a) {
    std::string out = a.get("--out");
    uint32_t N = (uint32_t)strtoul(a.get("--docs").c_str(), nullptr, 10);
    uint32_t V = (uint32_t)strtoul(a.get("--vocab").c_str(), nullptr, 10);
    uint64_t seed = strtoull(a.get("--seed", "12345").c_str(), nullptr, 10);
    uint32_t nshards = (uint32_t)strtoul(a.get("--nshards", "1").c_str(), nullptr, 10);
    uint32_t shard = (uint32_t)strtoul(a.get("--shard", "0").c_str(), nullptr, 10);
    bool values = a.flag("--values");
    bool mvalues = a.flag("--mvalues");
    const uint32_t nbool = (uint32_t)strtoul(a.get("--boolean-terms", "0").c_str(), nullptr, 10);
    /* --mvalues-sparse m0 m1: no slot-0 value where the smallest value is a multiple of m0, no slot-1 value
     * where it is a multiple of m1 (documents without a value: SerialiseKey's MAX/MIN_STR_CMPVALUE path) */
    uint32_t sp0 = 0, sp1 = 0;
    {
        for (size_t i = 0; i + 2 < a.v.size(); ++i)
            if (a.v[i] == "--mvalues-sparse") { sp0 = (uint32_t)strtoul(a.v[i + 1].c_str(), nullptr, 10); sp1 = (uint32_t)strtoul(a.v[i + 2].c_str(), nullptr, 10); }
    }
    uint32_t rfirst = (uint32_t)strtoul(a.get("--range-first", "1").c_str(), nullptr, 10);
    uint32_t rlast = (uint32_t)strtoul(a.get("--range-last", "0").c_str(), nullptr, 10);
    if (rlast == 0 || rlast > N) rlast = N;
    if (rfirst < 1) rfirst = 1;
    int flags = Xapian::DB_CREATE_OR_OVERWRITE | Xapian::DB_BACKEND_GLASS;
    if (!a.flag("--termlist")) flags |= Xapian::DB_NO_TERMLIST;

    xgm_zipf z;
    if (xgm_zipf_init(&z, V)) die("zipf alloc");
    std::vector<std::string> names(V);
    for (uint32_t r = 0; r < V; ++r) { char b[16]; int n = xgm_corpus_term(r, b); names[r].assign(b, n); }

    double t0 = now_s();
    Xapian::WritableDatabase db(out, flags);
    uint32_t ranks[XGM_CORPUS_MAX_LEN], wdf[XGM_CORPUS_MAX_LEN];
    uint32_t local = 0;
    uint32_t dstart = shard + 1;
    while (dstart < rfirst) dstart += nshards;
    for (uint32_t d = dstart; d <= rlast; d += nshards) {
        uint32_t len = xgm_corpus_doc(&z, seed, d, ranks);
        uint32_t n = xgm_corpus_collapse(ranks, len, wdf);
        Xapian::Document doc;
        /* --boolean-terms K: Document::add_boolean_term (wdf 0, no length), the way Xapiand stores boolean fields:
         * XBj on the docids that are multiples of j + 2; the multiples of 50 hold nothing else (length 0) */
        for (uint32_t j = 0; j < nbool; ++j)
            if (d % (j + 2) == 0) doc.add_boolean_term("XB" + std::to_string(j));
        if (nbool && d % 50 == 0) n = 0;
        for (uint32_t i = 0; i < n; ++i) doc.add_term(names[ranks[i]], wdf[i]);
        if (values) {
            uint64_t v0[3], v1;
            uint32_t n0 = xgm_corpus_values(seed, d, v0, &v1);
            /* slot 0: smallest of the 1..3 values (single-valued stock slot; the multi-valued
             * StringList encoding is Xapiand's, restated in oracle/xgm_oracle.c), slot 1: sort value,
             * slot 2: largest value */
            doc.add_value(0, Xapian::sortable_serialise((double)v0[0]));
            doc.add_value(1, Xapian::sortable_serialise((double)v1));
            doc.add_value(2, Xapian::sortable_serialise((double)v0[n0 - 1]));
        }
        if (mvalues) {
            uint64_t v0[3], v1;
            uint32_t n0 = xgm_corpus_values(seed, d, v0, &v1);
            std::vector<std::string> ser;
            for (uint32_t i = 0; i < n0; ++i) ser.push_back(xgmref::serialise_number((long double)v0[i]));
            /* Xapiand keeps the values of a slot in a std::set of serialised strings and writes
             * StringList::serialise of it (src/database/schema.cc:2958-2959, 5346): sorted, unique */
            ser.erase(std::unique(ser.begin(), ser.end()), ser.end());
            if (!(sp0 && v0[0] % sp0 == 0)) doc.add_value(0, xgmref::serialise_slot(ser));
            if (!(sp1 && v1 % sp1 == 0)) doc.add_value(1, xgmref::serialise_number((long double)v1));
        }
        Xapian::docid got = db.add_document(doc).did;
        if (got != ++local) die("unexpected docid");
    }
    db.commit();
    db.close();
    xgm_zipf_free(&z);
    printf("{\"cmd\":\"build\",\"out\":\"%s\",\"docs\":%u,\"shard\":%u,\"nshards\":%u,\"seconds\":%.3f}\n",
           out.c_str(), local, shard, nshards, now_s() - t0);
    return 0;
}

static int cmd_compact(const Args& a) {
    std::vector<std::string> dbs = a.all("--db");
    if (dbs.empty()) die("need --db");
    double t0 = now_s();
    Xapian::Database db;
    for (auto& p : dbs) db.add_database(Xapian::Database(p));
    db.compact(a.get("--out"), 0, 0);
    printf("{\"cmd\":\"compact\",\"parts\":%zu,\"seconds\":%.3f}\n", dbs.size(), now_s() - t0);
    return 0;
}

/* ---------------------------------------------------------------- query */

struct QSpec {
    std::string op;           /* AND | OR | TERM */
    uint32_t first = 0, maxitems = 10, check_at_least = 0;
    std::vector<std::string> terms;
    bool has_range = false;   /* VR slot lo hi → OP_FILTER(q, OP_VALUE_RANGE) */
    uint32_t r_slot = 0; double r_lo = 0, r_hi = 0;
    /* FT n t.. → OP_FILTER(q, AND of boolean terms); NOT n t.. → OP_AND_NOT(q, OR of terms);
     * MAYBE n t.. → OP_AND_MAYBE(q, OR of terms); applied in that order (innermost first) */
    std::vector<std::string> filter_terms, not_terms, maybe_terms;
    bool has_sort = false;    /* SORT slot reverse → set_sort_by_value_then_relevance */
    uint32_t s_slot = 0; bool s_rev = false;
    int s_mode = 0;           /* 0 value then relevance, 1 value only, 2 relevance then value */
    /* MVR slot lo hi  → OP_FILTER(q, MultipleValueRange(slot, ser(lo), ser(hi)))   (unweighted right side)
     * MVRW slot lo hi → OP_AND(q, MultipleValueRange(...))  — the source on the weighted side, the shape
     *                   MultipleValueRange::getQuery + query_dsl produce (src/multivalue/range.cc:110-125)
     * KEYSORT slot reverse → Enquire::set_sort_by_key_then_relevance(Multi_MultiValueKeyMaker{SerialiseKey}, false)
     *                   exactly as DocMatcher does (src/database/handler.cc:1269-1271) */
    int mvr = 0;              /* 0 none, 1 filter, 2 weighted */
    uint32_t mvr_slot = 0; double mvr_lo = 0, mvr_hi = 0;
    bool has_keysort = false; uint32_t ks_slot = 0; bool ks_rev = false;
    bool has_params = false;  /* BM25 k1 k3 b min_normlen → set_weighting_scheme(BM25Weight(k1, 0, k3, b, min_normlen)) */
    double k1 = 1, k3 = 1, b = 0.5, mnl = 0.5;
};

static std::vector<QSpec> load_queries(const std::string& path) {
    std::ifstream f(path);
    if (!f) die("cannot open " + path);
    std::vector<QSpec> qs;
    std::string line;
    while (std::getline(f, line)) {
        if (line.empty() || line[0] == '#') continue;
        std::istringstream is(line);
        QSpec q;
        uint32_t n;
        is >> q.op >> q.first >> q.maxitems >> q.check_at_least >> n;
        for (uint32_t i = 0; i < n; ++i) { std::string t; is >> t; q.terms.push_back(t); }
        std::string tok;
        while (is >> tok) {
            if (tok == "VR") { q.has_range = true; is >> q.r_slot >> q.r_lo >> q.r_hi; }
            else if (tok == "SORT") { q.has_sort = true; int r; is >> q.s_slot >> r; q.s_rev = r != 0; }
            else if (tok == "SORTMODE") { is >> q.s_mode; }
            else if (tok == "MVR" || tok == "MVRW") { q.mvr = tok == "MVR" ? 1 : 2; is >> q.mvr_slot >> q.mvr_lo >> q.mvr_hi; }
            else if (tok == "KEYSORT") { q.has_keysort = true; int r; is >> q.ks_slot >> r; q.ks_rev = r != 0; }
            else if (tok == "BM25") { q.has_params = true; is >> q.k1 >> q.k3 >> q.b >> q.mnl; }
            else if (tok == "FT" || tok == "NOT" || tok == "MAYBE") {
                uint32_t m; is >> m;
                std::vector<std::string>& dst = tok == "FT" ? q.filter_terms : tok == "NOT" ? q.not_terms : q.maybe_terms;
                for (uint32_t i = 0; i < m; ++i) { std::string t; is >> t; dst.push_back(t); }
            }
            else die("bad token " + tok);
        }
        if (!is.eof() && is.fail()) die("bad query line: " + line);
        qs.push_back(q);
    }
    return qs;
}

static Xapian::Query make_query(const QSpec& q) {
    /* "term^factor" → OP_SCALE_WEIGHT(term, factor) (Xapiand's _boost, QueryScaleWeight::postlist
     * api/queryinternal.cc:1075-1080) */
    /* "term#wqf" → Query(term, wqf) (within-query frequency, QueryTerm::get_wqf) */
    auto leaf = [](const std::string& t0) {
        std::string t = t0;
        const size_t c = t.find('^');
        double factor = 1.0;
        bool scaled = false;
        if (c != std::string::npos) { factor = atof(t.c_str() + c + 1); t = t.substr(0, c); scaled = true; }
        const size_t h = t.find('#');
        Xapian::termcount wqf = 1;
        if (h != std::string::npos) { wqf = (Xapian::termcount)atoi(t.c_str() + h + 1); t = t.substr(0, h); }
        Xapian::Query q(t, wqf);
        return scaled ? Xapian::Query(Xapian::Query::OP_SCALE_WEIGHT, q, factor) : q;
    };
    std::vector<Xapian::Query> leaves;
    for (const auto& t : q.terms) leaves.push_back(leaf(t));
    Xapian::Query base;
    if (q.op == "TERM") base = leaves.at(0);
    else if (q.op == "AND") base = Xapian::Query(Xapian::Query::OP_AND, leaves.begin(), leaves.end());
    else if (q.op == "OR") base = Xapian::Query(Xapian::Query::OP_OR, leaves.begin(), leaves.end());
    else die("bad op " + q.op);
    if (q.has_range) {
        Xapian::Query r(Xapian::Query::OP_VALUE_RANGE, q.r_slot,
                        Xapian::sortable_serialise(q.r_lo), Xapian::sortable_serialise(q.r_hi));
        base = Xapian::Query(Xapian::Query::OP_FILTER, base, r);
    }
    if (q.mvr) {
        Xapian::PostingSource* src = xgmref::make_multiple_value_range(
            q.mvr_slot, xgmref::serialise_number((long double)q.mvr_lo), xgmref::serialise_number((long double)q.mvr_hi));
        Xapian::Query r(src->release());
        base = Xapian::Query(q.mvr == 1 ? Xapian::Query::OP_FILTER : Xapian::Query::OP_AND, base, r);
    }
    auto group = [](Xapian::Query::op op, const std::vector<std::string>& ts) {
        return ts.size() == 1 ? Xapian::Query(ts[0]) : Xapian::Query(op, ts.begin(), ts.end());
    };
    if (!q.filter_terms.empty())
        base = Xapian::Query(Xapian::Query::OP_FILTER, base, group(Xapian::Query::OP_AND, q.filter_terms));
    if (!q.not_terms.empty())
        base = Xapian::Query(Xapian::Query::OP_AND_NOT, base, group(Xapian::Query::OP_OR, q.not_terms));
    if (!q.maybe_terms.empty())
        base = Xapian::Query(Xapian::Query::OP_AND_MAYBE, base, group(Xapian::Query::OP_OR, q.maybe_terms));
    return base;
}

struct QResult {
    std::vector<std::pair<uint32_t, double>> items;
    std::vector<std::string> sort_keys;
    std::vector<int> percents;   /* MSetIterator::get_percent */
    uint32_t lb = 0, est = 0, ub = 0;
    double max_possible = 0, max_attained = 0;
    double seconds = 0;
    int served = -1;          /* shim runner: 1 = libxgm answered, 0 = the reference matcher did */
    unsigned flags = 0;
    std::string reason;
};

static void setup_enquire(Xapian::Enquire& enq, const QSpec& q) {
    enq.set_query(make_query(q));
    if (q.has_keysort) {
        if (q.has_params) enq.set_weighting_scheme(Xapian::BM25Weight(q.k1, 0.0, q.k3, q.b, q.mnl));
        enq.set_sort_by_key_then_relevance(xgmref::make_key_maker({{q.ks_slot, q.ks_rev}})->release(), false);
        return;
    }
    if (q.has_params) enq.set_weighting_scheme(Xapian::BM25Weight(q.k1, 0.0, q.k3, q.b, q.mnl));
    if (q.has_sort && q.s_mode == 1) enq.set_sort_by_value(q.s_slot, q.s_rev);
    else if (q.has_sort && q.s_mode == 2) enq.set_sort_by_relevance_then_value(q.s_slot, q.s_rev);
    else if (q.has_sort) enq.set_sort_by_value_then_relevance(q.s_slot, q.s_rev);
    else enq.set_sort_by_relevance();
}

static void collect(const Xapian::MSet& m, QResult& r, bool want_keys) {
    r.items.clear(); r.sort_keys.clear(); r.percents.clear();
    for (auto it = m.begin(); it != m.end(); ++it) {
        r.items.emplace_back(*it, it.get_weight());
        r.percents.push_back(it.get_percent());
        if (want_keys) r.sort_keys.push_back(it.get_sort_key());
    }
    r.lb = m.get_matches_lower_bound();
    r.est = m.get_matches_estimated();
    r.ub = m.get_matches_upper_bound();
    r.max_possible = m.get_max_possible();
    r.max_attained = m.get_max_attained();
#ifdef XGM_SHIM_RUNNER
    r.served = xgm_shim_last_served();
    r.flags = xgm_shim_last_flags();
    r.reason = xgm_shim_last_reason();
#endif
}

static int cmd_query(const Args& a) {
    std::vector<std::string> dbs = a.all("--db");
    if (dbs.empty()) die("need --db");
    bool twophase = a.flag("--twophase");
    std::vector<QSpec> qs = load_queries(a.get("--queries"));
    int T = atoi(a.get("--threads", "1").c_str());
    int repeat = atoi(a.get("--repeat", "1").c_str());
    int warm = atoi(a.get("--warmup", "0").c_str());
    std::string dump = a.get("--dump", "");
    std::vector<QResult> res(qs.size());

    /* One worker per thread for the whole run: each opens its own Xapian::Database (+ Enquire) ONCE, outside
     * every timed wall, then takes part in the passes (warm-up and timed) released by the main thread.  A
     * pass's wall clock therefore covers Enquire::set_query + get_mset (+ MSet read-out) only — not thread
     * creation or the B-tree opens. */
    struct Gate {
        std::mutex mu; std::condition_variable cv;
        int pass = 0, done = 0, ready = 0; bool timed = false, quit = false;
    } gate;
    std::vector<std::thread> th;
    for (int t = 0; t < T; ++t) {
        th.emplace_back([&, t]() {
            try {
                Xapian::Database db;
                std::vector<Xapian::Database> sh;
                if (!twophase) { for (auto& p : dbs) db.add_database(Xapian::Database(p)); }
                else { for (auto& p : dbs) sh.emplace_back(p); }
                Xapian::Enquire enq(twophase ? Xapian::Database() : db);
                size_t n = sh.size();
                int seen = 0;
                { std::lock_guard<std::mutex> lk(gate.mu); ++gate.ready; }
                gate.cv.notify_all();
                for (;;) {
                    bool timed;
                    {
                        std::unique_lock<std::mutex> lk(gate.mu);
                        gate.cv.wait(lk, [&] { return gate.quit || gate.pass != seen; });
                        if (gate.quit) return;
                        seen = gate.pass;
                        timed = gate.timed;
                    }
                    for (size_t i = t; i < qs.size(); i += T) {
                        const QSpec& q = qs[i];
                        if (!twophase) {
                            setup_enquire(enq, q);
                            double t0 = now_s();
                            Xapian::MSet m = enq.get_mset(q.first, q.maxitems, q.check_at_least);
                            double dt = now_s() - t0;
                            if (timed) res[i].seconds = dt;
                            collect(m, res[i], q.has_sort || q.has_keysort);
                        } else {
                            /* Xapiand's DocMatcher scheme, src/database/handler.cc:1485-1551 */
                            double t0 = now_s();
                            Xapian::Enquire merger{Xapian::Database()};
                            std::vector<Xapian::Enquire> enqs;
                            std::vector<Xapian::MSet> msets(n);
                            Xapian::doccount doccount = 0;
                            for (size_t s = 0; s < n; ++s) {
                                enqs.emplace_back(sh[s]);
                                setup_enquire(enqs[s], q);
                                Xapian::MSet pm = enqs[s].prepare_mset("q", false, nullptr, nullptr);
                                merger.add_prepared_mset(pm);
                                doccount += sh[s].get_doccount();
                            }
                            for (size_t s = 0; s < n; ++s) {
                                enqs[s].set_prepared_mset(merger.get_prepared_mset());
                                msets[s] = enqs[s].get_mset(0, q.first + q.maxitems, q.check_at_least);
                                msets[s].unshard_docids(s, n);
                            }
                            setup_enquire(merger, q);
                            Xapian::MSet m = merger.merge_mset(msets, doccount, q.first, q.maxitems);
                            double dt = now_s() - t0;
                            if (timed) res[i].seconds = dt;
                            collect(m, res[i], q.has_sort || q.has_keysort);
                        }
                    }
                    { std::lock_guard<std::mutex> lk(gate.mu); ++gate.done; }
                    gate.cv.notify_all();
                }
            } catch (const Xapian::Error& e) {
                die("xapian: " + e.get_description());
            }
        });
    }
    {
        std::unique_lock<std::mutex> lk(gate.mu);
        gate.cv.wait(lk, [&] { return gate.ready == T; });
    }
    auto run_pass = [&](bool timed) {
        {
            std::lock_guard<std::mutex> lk(gate.mu);
            gate.timed = timed; gate.done = 0; ++gate.pass;
        }
        gate.cv.notify_all();
        std::unique_lock<std::mutex> lk(gate.mu);
        gate.cv.wait(lk, [&] { return gate.done == T; });
    };

    for (int w = 0; w < warm; ++w) run_pass(false);
    double best_wall = 1e300, total_wall = 0;
    std::vector<double> lat;
    for (int r = 0; r < repeat; ++r) {
        double t0 = now_s();
        run_pass(true);
        double w = now_s() - t0;
        total_wall += w;
        best_wall = std::min(best_wall, w);
        for (auto& x : res) lat.push_back(x.seconds);
    }
    {
        std::lock_guard<std::mutex> lk(gate.mu);
        gate.quit = true;
    }
    gate.cv.notify_all();
    for (auto& x : th) x.join();
    std::sort(lat.begin(), lat.end());
    auto pct = [&](double p) { return lat.empty() ? 0.0 : lat[std::min(lat.size() - 1, (size_t)(p * lat.size()))]; };
    if (!dump.empty()) {
        FILE* f = fopen(dump.c_str(), "w");
        if (!f) die("cannot write " + dump);
        for (size_t i = 0; i < res.size(); ++i) {
            const QResult& r = res[i];
            fprintf(f, "Q %zu %zu %u %u %u %.17g %.17g", i, r.items.size(), r.lb, r.est, r.ub,
                    r.max_possible, r.max_attained);
            if (r.served >= 0) {
                std::string why = r.reason;
                for (auto& c : why) if (c == ' ') c = '_';
                fprintf(f, " S%d F%u %s", r.served, r.flags, why.empty() ? "-" : why.c_str());
            }
            fputc('\n', f);
            for (size_t k = 0; k < r.items.size(); ++k) {
                fprintf(f, "%u %.17g", r.items[k].first, r.items[k].second);
                if (k < r.sort_keys.size()) {
                    fputc(' ', f);
                    for (unsigned char c : r.sort_keys[k]) fprintf(f, "%02x", c);
                    if (r.sort_keys[k].empty()) fputc('-', f);
                }
                if (k < r.percents.size()) fprintf(f, " p%d", r.percents[k]);
                fputc('\n', f);
            }
        }
        fclose(f);
    }
    double qps = (double)qs.size() * repeat / total_wall;
    printf("{\"cmd\":\"query\",\"queries\":%zu,\"threads\":%d,\"repeat\":%d,\"wall_s\":%.6f,\"qps\":%.3f,"
           "\"p50_ms\":%.6f,\"p99_ms\":%.6f,\"mode\":\"%s\",\"shards\":%zu}\n",
           qs.size(), T, repeat, total_wall, qps, pct(0.50) * 1e3, pct(0.99) * 1e3,
           twophase ? "twophase" : "multi", dbs.size());
    return 0;
}

/* ---------------------------------------------------------------- export */

static void w32(FILE* f, uint32_t v) { fwrite(&v, 4, 1, f); }
static void w64(FILE* f, uint64_t v) { fwrite(&v, 8, 1, f); }

static int cmd_export(const Args& a) {
    Xapian::Database db(a.get("--db"));
    std::string out = a.get("--out");
    FILE* f = fopen(out.c_str(), "wb");
    if (!f) die("cannot write " + out);
    uint32_t doccount = db.get_doccount(), lastdocid = db.get_lastdocid();
    uint64_t total_length = db.get_total_length();
    std::vector<std::string> terms;
    for (auto t = db.allterms_begin(); t != db.allterms_end(); ++t) terms.push_back(*t);
    std::vector<uint32_t> slots;
    for (uint32_t s = 0; s < 8; ++s) if (db.get_value_freq(s) > 0) slots.push_back(s);
    fwrite("XGMFLAT1", 8, 1, f);
    w32(f, doccount); w32(f, lastdocid); w64(f, total_length);
    w32(f, (uint32_t)terms.size()); w32(f, (uint32_t)slots.size());
    w32(f, db.get_doclength_lower_bound()); w32(f, db.get_doclength_upper_bound());
    std::vector<uint32_t> dl(lastdocid + 1, 0);
    for (auto p = db.postlist_begin(""); p != db.postlist_end(""); ++p) dl[*p] = db.get_doclength(*p);
    fwrite(dl.data(), 4, dl.size(), f);
    std::vector<uint32_t> dids, wdfs;
    for (auto& t : terms) {
        dids.clear(); wdfs.clear();
        for (auto p = db.postlist_begin(t); p != db.postlist_end(t); ++p) { dids.push_back(*p); wdfs.push_back(p.get_wdf()); }
        w32(f, (uint32_t)t.size()); fwrite(t.data(), 1, t.size(), f);
        w32(f, db.get_termfreq(t)); w64(f, db.get_collection_freq(t)); w32(f, db.get_wdf_upper_bound(t));
        w32(f, (uint32_t)dids.size());
        fwrite(dids.data(), 4, dids.size(), f);
        fwrite(wdfs.data(), 4, wdfs.size(), f);
    }
    for (uint32_t s : slots) {
        w32(f, s); w32(f, db.get_value_freq(s));
        for (auto v = db.valuestream_begin(s); v != db.valuestream_end(s); ++v) {
            std::string val = *v;
            w32(f, v.get_docid()); w32(f, (uint32_t)val.size()); fwrite(val.data(), 1, val.size(), f);
        }
    }
    fclose(f);
    printf("{\"cmd\":\"export\",\"doccount\":%u,\"terms\":%zu,\"slots\":%zu}\n", doccount, terms.size(), slots.size());
    return 0;
}

/* ref_runner slots --db DIR: "slot docid hex" of every stored value (Database::valuestream_begin) */
static int cmd_slots(const Args& a) {
    Xapian::Database db(a.get("--db"));
    for (uint32_t s = 0; s < 8; ++s) {
        if (db.get_value_freq(s) == 0) continue;
        for (auto v = db.valuestream_begin(s); v != db.valuestream_end(s); ++v) {
            std::string val = *v;
            printf("%u %u ", s, v.get_docid());
            for (unsigned char c : val) printf("%02x", c);
            printf("\n");
        }
    }
    return 0;
}

/* ref_runner serialise N...: hex of Xapiand's sortable_serialise (= Serialise::integer / positive / floating) */
static int cmd_serialise(int argc, char** argv) {
    for (int i = 2; i < argc; ++i) {
        std::string s = xgmref::serialise_number(strtold(argv[i], nullptr));
        for (unsigned char c : s) printf("%02x", c);
        printf("\n");
    }
    return 0;
}

int main(int argc, char** argv) {
    if (argc < 2) die("usage: ref_runner build|query|export ...");
    Args a;
    for (int i = 2; i < argc; ++i) a.v.push_back(argv[i]);
    std::string cmd = argv[1];
    try {
        if (cmd == "build") return cmd_build(a);
        if (cmd == "query") return cmd_query(a);
        if (cmd == "export") return cmd_export(a);
        if (cmd == "compact") return cmd_compact(a);
        if (cmd == "serialise") return cmd_serialise(argc, argv);
        if (cmd == "slots") return cmd_slots(a);
    } catch (const Xapian::Error& e) {
        die("xapian: " + e.get_description());
    }
    die("unknown command " + cmd);
}
