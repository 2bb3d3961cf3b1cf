// Batched keyword search: Search::execute for a batch of queries against the HBM-resident index.
//
// Control stays on the host (query graphs have tens of nodes), data stays on the device.  One host<->device round
// trip ("step") per ranking-rule *activation*: the step resolves every edge condition of the rule for the
// activation's universe into a bit-matrix and evaluates the whole cost-ordered path table with first-match
// semantics, which yields all buckets of that activation at once (DESIGN.md §3).  The reference interleaves the
// same work lazily (graph_based_ranking_rule.rs:220-368); the buckets are identical because a rule's universe only
// ever shrinks by the buckets it has already returned (bucket_sort.rs:298).
//
// Restated from: search/mod.rs:280-467, search/new/mod.rs:273-320,510-649,812-916, bucket_sort.rs:23-460,
// graph_based_ranking_rule.rs:136-368, ranking_rule_graph/{build.rs,cheapest_paths.rs,words,typo,proximity,fid,position,
// exactness}, exact_attribute.rs:96-301, query_graph.rs:96-187,254-301,346-406,453-543, query_term/parse_query.rs:28-300,
// query_term/compute_derivations.rs:170-253,363-383, resolve_query_graph.rs:33-130.
#include <atomic>
#include <chrono>
#include <cstring>
#include <functional>
#include <set>
#include <thread>

#include "engine.h"
#include "kernels.h"

namespace b200 {

#define CU(call, what)                                     \
    do {                                                   \
        cudaError_t e_ = (call);                           \
        if (e_ != cudaSuccess) return cuda_fail(e_, what); \
    } while (0)

namespace {

enum RuleKind { RK_WORDS = 0, RK_TYPO, RK_PROXIMITY, RK_FID, RK_POSITION, RK_EXACTNESS, RK_EXACT_ATTRIBUTE, RK_RESOLVE, RK_FREQ };

struct UnsupportedQuery {
    std::string why;
};
struct TooComplex {
    std::string why;
};

// ------------------------------------------------------------------------------------------------ terms
struct WordRef {
    uint32_t rank;
    bool derived;
};

// the terms of a query; QCtx binds them to the index they come from
struct QTerms {
    std::vector<ETerm> terms;
    std::vector<EPhrase> phrases;
    std::map<std::vector<int32_t>, uint32_t> phrase_ids;
    std::vector<uint32_t> neg_words;    // dictionary ranks of `-word` tokens (absent words exclude nothing)
    std::vector<uint32_t> neg_phrases;  // phrase ids of `-"..."`
    std::vector<uint16_t> freq_weight;  // TermsMatchingStrategy::Frequency: removal weight per term id (query_graph.rs:303-344)
};
struct QCtx : QTerms {
    const HostIndex &ix;
    explicit QCtx(const HostIndex &i) : ix(i) {}
    uint32_t intern_phrase(const EPhrase &p) {
        auto it = phrase_ids.find(p.words);
        if (it != phrase_ids.end()) return it->second;
        phrases.push_back(p);
        phrase_ids.emplace(p.words, (uint32_t)phrases.size() - 1);
        return (uint32_t)phrases.size() - 1;
    }
    int32_t word_rank_or_absent(const std::string &w) const {
        int64_t r = ix.find_word(w);
        return r >= 0 ? (int32_t)r : -2;
    }
    static int32_t first_word(const EPhrase &p) {
        for (auto w : p.words)
            if (w != -1) return w;
        return -1;
    }
};

uint8_t number_of_typos_allowed(const HostIndex &ix, const std::string &w) {  // parse_query.rs:204-225 (ASCII)
    const Settings &s = ix.settings;
    if (!s.authorize_typos || w.size() < s.one_typo || s.exact_words.count(w)) return 0;
    return w.size() < s.two_typos ? 1 : 2;
}

// compute_derivations.rs:170-253 (zero-typo part)
ETerm term_from_word(QCtx &c, const std::string &word, uint8_t max_typo, bool is_prefix, bool is_ngram) {
    const HostIndex &ix = c.ix;
    ETerm t;
    t.original = word;
    if (word.size() > 250) {
        t.empty_term = true;
        return t;
    }
    int32_t pid = ix.find_prefix(word);
    bool use_pdb = is_prefix && pid >= 0 && (ix.pd_list[pid] != NO_LIST || (!is_ngram && ix.epd_list[pid] != NO_LIST));
    if (use_pdb) t.prefix_db = pid;
    t.exact = (int32_t)ix.find_word(word);
    if (is_prefix && !use_pdb) {
        uint64_t lo, hi;
        ix.prefix_range(word, lo, hi);
        for (uint64_t i = lo; i < hi; i++) {
            if ((int64_t)i == t.exact) continue;
            t.prefix_of.push_back((uint32_t)i);
            if (t.prefix_of.size() >= 1000) break;
        }
    }
    auto it = ix.settings.synonyms.find(std::vector<std::string>{word});
    if (it != ix.settings.synonyms.end()) {
        size_t synonym_word_count = 0, taken = 0;
        for (auto &syn : it->second) {
            if (taken++ >= 50) break;                             // MAX_SYNONYM_PHRASE_COUNT
            if (synonym_word_count + syn.size() > 100) continue;  // MAX_SYNONYM_WORD_COUNT
            synonym_word_count += syn.size();
            EPhrase p;
            for (auto &w : syn) p.words.push_back(c.word_rank_or_absent(w));
            t.synonyms.push_back(c.intern_phrase(p));
        }
        std::sort(t.synonyms.begin(), t.synonyms.end());
        t.synonyms.erase(std::unique(t.synonyms.begin(), t.synonyms.end()), t.synonyms.end());
    }
    t.max_lev = max_typo;
    t.is_prefix = is_prefix;
    t.is_ngram = is_ngram;
    return t;
}

// compute_derivations.rs:363-383 + 255-317
void find_split_words(QCtx &c, ETerm &t) {
    const HostIndex &ix = c.ix;
    const std::string &o = t.original;
    uint32_t best = 0, bl = 0, br = 0;
    bool have = false;
    t.split = -1;
    if (!t.allows_split_words()) return;
    for (size_t i = 1; i < o.size(); i++) {
        int64_t l = ix.find_word((const uint8_t *)o.data(), i), r = ix.find_word((const uint8_t *)o.data() + i, o.size() - i);
        if (l < 0 || r < 0) continue;
        uint32_t list = ix.find_pair(1, (uint32_t)l, (uint32_t)r);
        if (list == NO_LIST) continue;
        uint32_t freq = ix.lists[list].card;
        if (!have || freq > best) {
            have = true;
            best = freq;
            bl = (uint32_t)l;
            br = (uint32_t)r;
        }
    }
    if (!have) return;
    if (t.is_ngram && t.max_lev <= 1) {
        // only in the <=1 typo initialisation (compute_derivations.rs:297-311): drop the split equal to the ngram's own words
        if (t.ngram_words.size() == 2 && ix.word(bl) == t.ngram_words[0] && ix.word(br) == t.ngram_words[1]) return;
    }
    EPhrase p;
    p.words = {(int32_t)bl, (int32_t)br};
    t.split = (int32_t)c.intern_phrase(p);
}

struct ExactTermRef {
    int kind = 0;  // 0 none, 1 word, 2 phrase
    uint32_t id = 0;
};
ExactTermRef exact_term(const QCtx &c, const ETermSubset &s) {  // query_term/mod.rs:131-143
    const ETerm &t = c.terms[s.term];
    ExactTermRef e;
    if (t.is_ngram) return e;
    if (t.phrase >= 0) {
        if (s.zero.contains_phrase((uint32_t)t.phrase)) e = {2, (uint32_t)t.phrase};
    } else if (t.exact >= 0) {
        if (s.zero.contains_word((uint32_t)t.exact)) e = {1, (uint32_t)t.exact};
    }
    return e;
}
bool use_prefix_db(const QCtx &c, const ETermSubset &s, uint32_t &pid, bool &derived) {  // :177-198
    const ETerm &t = c.terms[s.term];
    if (t.prefix_db < 0) return false;
    bool ok = s.zero.kind == N_ALL || (s.zero.kind == N_SUBSET && t.exact >= 0 && s.zero.contains_word((uint32_t)t.exact));
    if (!ok) return false;
    pid = (uint32_t)t.prefix_db;
    derived = t.is_ngram;
    return true;
}
std::vector<WordRef> all_single_words(const QCtx &c, const ETermSubset &s) {  // :199-292
    const ETerm &t = c.terms[s.term];
    std::vector<WordRef> r;
    if (s.zero.kind != N_NOTHING) {
        if (t.exact >= 0 && s.zero.contains_word((uint32_t)t.exact)) r.push_back({(uint32_t)t.exact, t.is_ngram});
        for (auto w : t.prefix_of)
            if (s.zero.contains_word(w)) r.push_back({w, t.is_ngram});
    }
    if (s.one.kind != N_NOTHING)
        for (auto w : t.one_typo)
            if (s.one.contains_word(w)) r.push_back({w, true});
    if (s.two.kind != N_NOTHING)
        for (auto w : t.two_typo)
            if (s.two.contains_word(w)) r.push_back({w, true});
    return r;
}
// all_phrases (:293-329): the zero-typo phrase and the synonyms are returned whatever zero_typo_subset says
std::vector<uint32_t> all_phrases(const QCtx &c, const ETermSubset &s) {
    const ETerm &t = c.terms[s.term];
    std::vector<uint32_t> r;
    if (t.phrase >= 0) r.push_back((uint32_t)t.phrase);
    for (auto p : t.synonyms) r.push_back(p);
    if (t.split >= 0 && (s.one.kind == N_ALL || (s.one.kind == N_SUBSET && s.one.contains_phrase((uint32_t)t.split)))) r.push_back((uint32_t)t.split);
    std::sort(r.begin(), r.end());
    r.erase(std::unique(r.begin(), r.end()), r.end());
    return r;
}
bool original_phrase(const QCtx &c, const ETermSubset &s, uint32_t &p) {  // :331-339
    const ETerm &t = c.terms[s.term];
    if (t.phrase >= 0 && s.zero.contains_phrase((uint32_t)t.phrase)) {
        p = (uint32_t)t.phrase;
        return true;
    }
    return false;
}
uint8_t max_typo_cost(const QCtx &c, const ETermSubset &s) {  // :340-370
    const ETerm &t = c.terms[s.term];
    switch (t.max_lev) {
        case 0: return t.allows_split_words() ? 1 : 0;
        case 1: return s.one.is_empty() ? 0 : 1;
        default: return s.two.is_empty() ? (s.one.is_empty() ? 0 : 1) : 2;
    }
}

// ------------------------------------------------------------------------------------------------ graph
void build_initial_edges(EGraph &g) {  // query_graph.rs:254-301
    for (auto &n : g.nodes) {
        n.pred.clear();
        n.succ.clear();
    }
    uint16_t n = (uint16_t)g.nodes.size();
    for (uint16_t id = 0; id < n; id++) {
        int end_prev;
        if (g.nodes[id].kind == ND_TERM)
            end_prev = g.nodes[id].term.t1;
        else if (g.nodes[id].kind == ND_START)
            end_prev = -1;
        else
            continue;
        int mn = 32767;
        std::vector<uint16_t> succ;
        for (uint16_t j = 0; j < n; j++) {
            int start_next;
            if (g.nodes[j].kind == ND_TERM)
                start_next = g.nodes[j].term.t0;
            else if (g.nodes[j].kind == ND_END)
                start_next = 32767;
            else
                continue;
            if (start_next <= end_prev) continue;
            if (start_next < mn) {
                mn = start_next;
                succ.clear();
                succ.push_back(j);
            } else if (start_next == mn)
                succ.push_back(j);
        }
        g.nodes[id].succ = succ;
        for (auto s : succ) sorted_insert(g.nodes[s].pred, id);
    }
}

void remove_nodes_keep_edges(EGraph &g, const std::vector<uint16_t> &nodes) {  // :190-210
    for (auto id : nodes) {
        auto pred = g.nodes[id].pred, succ = g.nodes[id].succ;
        for (auto p : pred) {
            sorted_remove(g.nodes[p].succ, id);
            for (auto s : succ) sorted_insert(g.nodes[p].succ, s);
        }
        for (auto s : succ) {
            sorted_remove(g.nodes[s].pred, id);
            for (auto p : pred) sorted_insert(g.nodes[s].pred, p);
        }
        g.nodes[id].kind = ND_DELETED;
        g.nodes[id].pred.clear();
        g.nodes[id].succ.clear();
    }
}

// removal_order_for_terms_matching_strategy (query_graph.rs:379-406): groups of nodes, cheapest removal first.
// Last: weight(term) = 1 + last - term (:346-377); Frequency: weight from the term frequencies (:303-344, QCtx::freq_weight).
std::vector<std::vector<uint16_t>> removal_order(const QCtx &c, const EGraph &g, int tms) {
    int first = 255, last = 0;
    for (auto &n : g.nodes)
        if (n.kind == ND_TERM) {
            last = std::max<int>(last, n.term.t1);
            first = std::min<int>(first, n.term.t0);
        }
    if (tms == B200_TMS_LAST && first >= last) return {};
    std::map<uint16_t, std::vector<uint16_t>> groups;
    bool mandatory = false;
    for (uint16_t id = 0; id < g.nodes.size(); id++) {
        const ENode &n = g.nodes[id];
        if (n.kind != ND_TERM) continue;
        uint32_t ph;
        if (original_phrase(c, n.term.ts, ph) || n.term.ts.mandatory) {
            mandatory = true;
            continue;
        }
        uint16_t cost = 0;
        for (int t = n.term.t0; t <= n.term.t1; t++) {
            uint16_t w = tms == B200_TMS_FREQUENCY ? ((size_t)t < c.freq_weight.size() ? c.freq_weight[t] : (uint16_t)1) : (uint16_t)(1 + last - t);
            cost = std::max<uint16_t>(cost, w);
        }
        groups[cost].push_back(id);
    }
    std::vector<std::vector<uint16_t>> res;
    for (auto &kv : groups) res.push_back(kv.second);
    if (!mandatory && !res.empty()) res.pop_back();
    return res;
}

// ------------------------------------------------------------------------------------------------ activations
struct ECond {
    int rule = 0;
    ELocated term;
    uint8_t nbr_typos = 0;
    bool prox_uninit = false;
    ELocated left;
    uint8_t cost = 0;
    bool has_fid = false;
    uint16_t fid = 0;
    std::vector<uint16_t> positions;
    bool exact_in_attribute = false;
    // what a surviving path hands to the next rule (ComputedCondition::{start,end}_term_subset)
    bool has_start = false;
    ELocated start_subset, end_subset;
    uint16_t col = 0;
};

struct EEdge {
    uint16_t src, dst;
    uint32_t cost;
    int32_t cond;
};

struct SEdge {  // edge of the state graph handed to the device
    uint16_t src, dst;  // state ids (topological)
    uint32_t cost;
    int32_t cond;       // condition id or -1
};
struct SurvPath {
    uint16_t cost_idx;
    std::vector<uint16_t> edges;  // state-graph edge ids, START..END
};

struct StepOut {  // per-activation device work, appended to the step blob by the driver
    std::vector<Job> jobs;            // act filled in by the driver
    std::vector<PairSet> pairsets;    // left_off/right_off relative to `words`
    std::vector<uint32_t> words;
    std::vector<ColOp> colprog;
    std::vector<DpState> dp_states;   // edge_begin relative to dp_edges
    std::vector<DpEdge> dp_edges;
    std::vector<uint16_t> cost_vals;
    std::vector<uint32_t> prog;       // DP program for eval_dp_kernel (device_types.h: EVAL_COL_*)
    uint32_t n_cols = 0, n_costs = 0, n_pairs = 0, want_paths = 0, all_conditional = 0;
    uint64_t posting_bytes = 0;
};

struct Level {
    int rule_idx = -1;  // index in the query's rule list; -1 = universe resolution
    int kind = RK_RESOLVE;
    EGraph graph;
    std::vector<ECond> conds;
    // state graph: states in topological order (0 = START, last = END); edges grouped by source in visiting order
    uint16_t n_states = 0;
    std::vector<SEdge> sedges;
    std::vector<uint32_t> state_edge_begin;            // n_states + 1
    std::vector<std::pair<uint16_t, uint16_t>> state_cost_range;  // (rmin, rcount) per state
    std::vector<uint32_t> cost_vals;
    bool want_paths = false;
    bool neg_only = false;  // RK_RESOLVE of a query made only of negative terms: the one condition is the ignored documents, the answer the rest
    std::vector<SurvPath> surv;
    uint64_t next_max_cost = 1;
    // device buffers (arena)
    uint32_t *uw = nullptr;
    unsigned long long *ub = nullptr, *out = nullptr;
    uint32_t ld = 0, rows = 0, res_off = 0;
    uint32_t walked_m = 0;               // last bucket whose surviving paths were computed (walk_kernel)
    bool below_done = false;             // a bucket of this level already fell below the ranking-score threshold
    size_t a_off = SIZE_MAX, a_len = 0;  // the level's block in its lane's arena (uw | ub | out)
    std::vector<uint32_t> counts;  // per cost idx, last = unmatched
    size_t cursor = 0;
    uint64_t universe_count = 0;
};

// Tree mode (no deadline): every needed bucket of a level is expanded as soon as the level's counts are known — the result window of
// each bucket follows from the counts of the buckets before it, so sibling subtrees are independent searches.  A Node is one rule
// level of one query: its Level, where it stands in the result order and the scores its documents carry on entry.
struct Node {
    Level L;
    Node *parent = nullptr;
    std::atomic<uint32_t> live_children{0};  // child nodes whose activation has not completed (it reads this level's buckets)
    bool self_done = false;       // this level's own bucket loop is done
    uint64_t off0 = 0;            // documents of the query that come before this level's universe in result order
    std::vector<EScore> scores;   // ranking-rule scores on entry (the path of buckets that led here)
};

// The universe of an activation (ActDesc::p_*): bucket column `col` of its parent level, or the query's universe for its first
// activation.  cap bounds the activation's rows.
struct ParentRef {
    const uint32_t *uw = nullptr;
    const unsigned long long *ub = nullptr, *out = nullptr;
    uint32_t rows = 0, ld = 0, col = 0, cap = 0;
    static ParentRef bucket(const Level &L, uint32_t ci, uint64_t cnt) {
        return ParentRef{L.uw, L.ub, L.out, L.rows, L.ld, ci, (uint32_t)std::min<uint64_t>(cnt, L.rows)};
    }
    static ParentRef universe(const unsigned long long *ub, uint32_t n_words64) { return ParentRef{nullptr, ub, nullptr, n_words64, n_words64, 0, n_words64}; }
};

// One requested activation: the level it evaluates, the device work description and where its parent universe is.
struct Pending {
    Level *L = nullptr;           // in QState::levels (sequential mode: stable until the activation completes) or in a Node
    Node *node = nullptr;         // tree mode
    StepOut o;
    ParentRef parent;
    uint32_t need = 1;            // documents bucket_sort can still use from this activation (ActDesc::need)
    uint32_t tab_shift = 0;       // path de-duplication table = 4096 << tab_shift slots
    size_t demand = 0;            // device bytes asked for (capacity diagnostics)
};

// What the completion of one activation adds to its query in tree mode.  Activations of the same query complete on different
// threads; each fills its own ActOut and the query folds them in afterwards (one thread per query).
struct ActOut {
    std::vector<EmitDesc> emits;
    std::vector<std::unique_ptr<Node>> nodes;
    std::vector<std::unique_ptr<Pending>> pendings;
    std::vector<std::pair<size_t, size_t>> freed;
    uint32_t n_results = 0;
    int status = 0;
    std::string error;
    bool retry = false, expanded = false;
};

struct QState {
    QCtx ctx;
    int status = 0;
    std::string error;
    bool done = false, placeholder = false, neg_only = false;
    EGraph graph;
    std::vector<int> rules;  // RuleKind per rule
    std::vector<Level> levels;
    std::vector<EScore> rr_scores;
    uint32_t n_results = 0;
    uint64_t cur_offset = 0;
    uint64_t n_candidates = 0;
    std::vector<std::vector<EScore>> scores;  // per hit
    // device work requested for the next steps (sequential mode: at most one)
    std::vector<std::unique_ptr<Pending>> pendings;
    std::vector<EmitDesc> emits;
    // tree mode
    bool tree = false;
    std::vector<std::unique_ptr<Node>> nodes;
    uint32_t outstanding = 0;  // activations requested and not yet expanded
    const unsigned long long *d_univ = nullptr;  // filtered_universe of the query on the device (nullptr = documents_ids)
    uint64_t univ_count = 0;
    bool degraded = false, used_negative = false;
    long polls = 0;                   // Deadline::exceeded() calls so far (stop_after hook)
    const unsigned long long *cand_src = nullptr;  // device bitmap to copy into b200_results::candidates at the lane's next step
    std::vector<uint64_t> term_freq;  // Frequency: documents per term id, filled one device step per term before anything else
    uint32_t n_term_ids = 0;
    // Sort rules of a placeholder search (search/new/mod.rs:351-416): fid and direction per rule; sort_lo/hi: the ranks of the
    // universe the result window holds, produced by sort_window_kernel after the step loop
    std::vector<SortRule> sort_rules;
    bool sort_pending = false;
    uint32_t sort_lo = 0, sort_hi = 0;
    std::vector<uint32_t> sort_ids;  // the result window's docids
    // a leading GeoSort rule (geo_windows): |universe AND geo| and the first rows of its order, with their haversine distance and
    // rtree key; the Dynamic strategy's rtree / iterative split (the rtree tuple of rank geo_m - 1)
    uint32_t geo_n = 0, geo_m = 0;
    bool geo_split_known = false;
    unsigned long long geo_split_key = 0;
    uint32_t geo_split_doc = 0;
    std::vector<uint32_t> geo_docs;
    std::vector<double> geo_dist;  // computed on the host (geo_distance_host), as the chain compares them
    // the iterative keys the device cannot decide, decided on the host: (docid << 32 | floor metres), ascending; listed once, the
    // first time a window of the query reaches its iterative part
    bool geo_patched = false;
    std::vector<unsigned long long> geo_patch;
    // arena blocks of levels bucket_sort has left; the lane's driver returns them to its allocator at the start of its next step
    // (the emissions queued by the same advance() still read them: they run first on the lane's stream, before any new owner writes)
    std::vector<std::pair<size_t, size_t>> freed;
    void release_level(Level &L) {
        if (L.a_off != SIZE_MAX) freed.emplace_back(L.a_off, L.a_len);
        L.a_off = SIZE_MAX;
    }
    void pop_level() {
        release_level(levels.back());
        levels.pop_back();
    }
    void drop_levels() {
        for (auto &L : levels) release_level(L);
        levels.clear();
    }
    explicit QState(const HostIndex &ix) : ctx(ix) {}
};

struct ActBuilder {
    const QCtx &c;
    StepOut &o;
    uint16_t next_col = 0;
    std::map<uint32_t, uint16_t> phrase_cols;  // phrase id -> column
    ActBuilder(const QCtx &ctx, StepOut &out) : c(ctx), o(out) {}
    uint16_t new_col() { return next_col++; }
    void add_list(uint16_t col, uint32_t list) {
        if (list == NO_LIST) return;
        const ListRef &lr = c.ix.lists[list];
        if (lr.card == 0) return;
        uint32_t units = lr.dense ? c.ix.n_words64 : lr.card;
        uint32_t nch = (units + JOB_CHUNK - 1) / JOB_CHUNK;
        for (uint32_t k = 0; k < nch; k++) o.jobs.push_back(Job{0, col, list, k});
        o.posting_bytes += lr.dense ? (uint64_t)c.ix.n_words64 * 8 : (uint64_t)lr.card * 4;
    }
    void op(uint16_t code, uint16_t dst, uint16_t a, uint16_t b) { o.colprog.push_back(ColOp{code, dst, a, b}); }
    // Word::Original -> exact_word_docids | word_docids ; Word::Derived -> word_docids   (db_cache.rs:183-205)
    void add_word_docids(uint16_t col, const WordRef &w) {
        add_list(col, c.ix.wd_list[w.rank]);
        if (!w.derived) add_list(col, c.ix.ewd_list[w.rank]);
    }
    // compute_phrase_docids (resolve_query_graph.rs:187-268) as a column: AND of the words' lists, then for every window of
    // up to three words the AND of the pair-proximity unions.  Universe-restricted like every column; every use of phrase
    // docids in the reference intersects with the universe anyway.
    uint16_t phrase_col(uint32_t pid) {
        auto it = phrase_cols.find(pid);
        if (it != phrase_cols.end()) return it->second;
        uint16_t col = new_col();
        phrase_cols.emplace(pid, col);
        const std::vector<int32_t> &words = c.phrases[pid].words;
        std::vector<uint32_t> real;
        for (auto w : words) {
            if (w == -2) return col;  // a word that is not in the dictionary: the phrase matches nothing
            if (w >= 0) real.push_back((uint32_t)w);
        }
        if (real.empty()) return col;
        if (words.size() == 2 && real.size() == 2) {  // docids of a 2-word phrase == its proximity-1 pair list
            add_list(col, c.ix.find_pair(1, real[0], real[1]));
            return col;
        }
        // plan first: any missing mandatory list makes the phrase empty
        struct Group {
            std::vector<uint32_t> lists;
        };
        std::vector<Group> groups;
        for (auto w : real) {
            Group g;
            if (c.ix.wd_list[w] != NO_LIST) g.lists.push_back(c.ix.wd_list[w]);
            if (c.ix.ewd_list[w] != NO_LIST) g.lists.push_back(c.ix.ewd_list[w]);
            if (g.lists.empty()) return col;
            groups.push_back(std::move(g));
        }
        size_t winsize = std::min<size_t>(words.size(), 3);
        for (size_t ws = 0; ws + winsize <= words.size(); ws++)
            for (size_t i = 0; i < winsize; i++) {
                if (words[ws + i] < 0) continue;
                for (size_t k = i + 1; k < winsize; k++) {
                    if (words[ws + k] < 0) continue;
                    size_t dist = k - i - 1;
                    Group g;
                    for (size_t d = 0; d <= dist; d++) {
                        uint32_t l = c.ix.find_pair((uint32_t)d + 1, (uint32_t)words[ws + i], (uint32_t)words[ws + k]);
                        if (dist == 0 && l == NO_LIST) return col;
                        if (l != NO_LIST) g.lists.push_back(l);
                    }
                    if (g.lists.empty()) return col;
                    groups.push_back(std::move(g));
                }
            }
        bool first = true;
        for (auto &g : groups) {
            uint16_t t = first ? col : new_col();
            for (auto l : g.lists) add_list(t, l);
            if (!first) op(0, col, col, t);
            first = false;
        }
        return col;
    }
    // compute_query_term_subset_docids (resolve_query_graph.rs:33-59) into `col`
    void term_docids(uint16_t col, const ETermSubset &s) {
        for (auto &w : all_single_words(c, s)) add_word_docids(col, w);
        for (auto p : all_phrases(c, s)) op(1, col, col, phrase_col(p));
        uint32_t pid;
        bool derived;
        if (use_prefix_db(c, s, pid, derived)) {
            add_list(col, c.ix.pd_list[pid]);
            if (!derived) add_list(col, c.ix.epd_list[pid]);
        }
    }
    uint32_t push_words(const std::vector<uint32_t> &w) {
        uint32_t off = (uint32_t)o.words.size();
        o.words.insert(o.words.end(), w.begin(), w.end());
        return off;
    }
    void add_pairset(uint16_t col, const std::vector<uint32_t> &left, const std::vector<uint32_t> &right, uint8_t fwd, uint8_t bwd, bool range) {
        uint32_t nr = range ? (uint32_t)right.size() / 2 : (uint32_t)right.size();
        if (left.empty() || nr == 0 || (fwd == 0 && bwd == 0)) return;
        PairSet ps{};
        ps.col = col;
        ps.left_off = push_words(left);
        ps.n_left = (uint32_t)left.size();
        ps.right_off = push_words(right);
        ps.n_right = nr;
        ps.fwd_prox = fwd;
        ps.bwd_prox = bwd;
        ps.right_is_range = range ? 1 : 0;
        o.pairsets.push_back(ps);
    }
};

// proximity/compute_docids.rs:15-108 as device work
void build_proximity_cond(ActBuilder &b, const ECond &cond) {
    const QCtx &c = b.c;
    if (!cond.prox_uninit) {
        b.term_docids(cond.col, cond.term.ts);
        return;
    }
    uint8_t right_len = (uint8_t)cond.term.n_term_ids();
    uint8_t fwd = (uint8_t)(1 + cond.cost - right_len), bwd = (uint8_t)(cond.cost - right_len);
    if (fwd > 3) fwd = 0;  // keys only exist for proximities 1..3
    if (bwd > 3) bwd = 0;
    // last_words_of_term_derivations (:213-231) / first_word_of_term_iter (:232-251)
    std::vector<uint32_t> left_words, right_words;
    for (auto &w : all_single_words(c, cond.left.ts)) left_words.push_back(w.rank);
    for (auto &w : all_single_words(c, cond.term.ts)) right_words.push_back(w.rank);
    for (auto *v : {&left_words, &right_words}) {
        std::sort(v->begin(), v->end());
        v->erase(std::unique(v->begin(), v->end()), v->end());
    }
    std::vector<std::pair<uint32_t, uint32_t>> left_phr, right_phr;  // (phrase id, boundary word)
    for (auto p : all_phrases(c, cond.left.ts)) {
        int32_t last = c.phrases[p].words.empty() ? -1 : c.phrases[p].words.back();
        if (last >= 0) left_phr.push_back({p, (uint32_t)last});
    }
    for (auto p : all_phrases(c, cond.term.ts)) {
        int32_t first = c.phrases[p].words.empty() ? -1 : c.phrases[p].words.front();
        if (first >= 0) right_phr.push_back({p, (uint32_t)first});
    }
    auto anded = [&](const std::vector<uint32_t> &l, const std::vector<uint32_t> &r, bool range, std::initializer_list<uint32_t> phrases) {
        uint16_t t = b.new_col();
        b.add_pairset(t, l, r, fwd, 0, range);  // no swapping when a phrase is involved (:149, :199)
        for (auto p : phrases) b.op(0, t, t, b.phrase_col(p));
        b.op(1, cond.col, cond.col, t);
    };
    // prefix-db part (compute_prefix_edges :110-170)
    uint32_t pid;
    bool pderived;
    if (use_prefix_db(c, cond.term.ts, pid, pderived)) {
        uint64_t lo, hi;
        c.ix.prefix_range(c.ix.prefixes[pid], lo, hi);
        std::vector<uint32_t> range{(uint32_t)lo, (uint32_t)hi};
        b.add_pairset(cond.col, left_words, range, fwd, 0, true);
        int64_t prefix_as_word = c.ix.find_word(c.ix.prefixes[pid]);
        if (prefix_as_word >= 0 && bwd) b.add_pairset(cond.col, left_words, {(uint32_t)prefix_as_word}, 0, bwd, false);
        for (auto &lp : left_phr) anded({lp.second}, range, true, {lp.first});
    }
    // non-prefix part (compute_non_prefix_edges :172-211)
    b.add_pairset(cond.col, left_words, right_words, fwd, bwd, false);
    for (auto &lp : left_phr) anded({lp.second}, right_words, false, {lp.first});
    for (auto &rp : right_phr) anded(left_words, {rp.second}, false, {rp.first});
    for (auto &lp : left_phr)
        for (auto &rp : right_phr) anded({lp.second}, {rp.second}, false, {lp.first, rp.first});
}

void build_cond(ActBuilder &b, const ECond &cond) {
    const QCtx &c = b.c;
    switch (cond.rule) {
        case RK_WORDS:
        case RK_TYPO:
        case RK_RESOLVE: b.term_docids(cond.col, cond.term.ts); break;
        case RK_PROXIMITY: build_proximity_cond(b, cond); break;
        case RK_FID: {  // resolve_query_graph.rs:61-93
            if (!cond.has_fid) break;
            for (auto &w : all_single_words(c, cond.term.ts)) b.add_list(cond.col, c.ix.word_fid_list(w.rank, cond.fid));
            for (auto p : all_phrases(c, cond.term.ts)) {
                int32_t fw = QCtx::first_word(c.phrases[p]);
                if (fw < 0) continue;
                uint32_t l = c.ix.word_fid_list((uint32_t)fw, cond.fid);
                if (l == NO_LIST) continue;
                uint16_t tf = b.new_col();
                b.add_list(tf, l);
                b.op(0, tf, tf, b.phrase_col(p));
                b.op(1, cond.col, cond.col, tf);
            }
            uint32_t pid;
            bool derived;
            if (use_prefix_db(c, cond.term.ts, pid, derived)) b.add_list(cond.col, c.ix.prefix_fid_list(pid, cond.fid));
            break;
        }
        case RK_POSITION: {  // position/mod.rs:24-47 + resolve_query_graph.rs:95-130
            auto words = all_single_words(c, cond.term.ts);
            auto phrases = all_phrases(c, cond.term.ts);
            uint32_t pid;
            bool derived;
            bool pdb = use_prefix_db(c, cond.term.ts, pid, derived);
            for (auto p : cond.positions) {
                for (auto &w : words) b.add_list(cond.col, c.ix.word_pos_list(w.rank, p));
                if (pdb) b.add_list(cond.col, c.ix.prefix_pos_list(pid, p));
            }
            for (auto ph : phrases) {  // phrase & (first word at any of the positions)
                int32_t fw = QCtx::first_word(c.phrases[ph]);
                if (fw < 0) continue;
                uint16_t tf = 0;
                bool have = false;
                for (auto p : cond.positions) {
                    uint32_t l = c.ix.word_pos_list((uint32_t)fw, p);
                    if (l == NO_LIST) continue;
                    if (!have) {
                        tf = b.new_col();
                        have = true;
                    }
                    b.add_list(tf, l);
                }
                if (have) {
                    b.op(0, tf, tf, b.phrase_col(ph));
                    b.op(1, cond.col, cond.col, tf);
                }
            }
            break;
        }
        case RK_EXACTNESS: {  // exactness/mod.rs:19-73
            if (cond.exact_in_attribute) {
                ExactTermRef e = exact_term(c, cond.term.ts);
                if (e.kind == 1)
                    b.add_word_docids(cond.col, WordRef{e.id, false});
                else if (e.kind == 2)
                    b.op(1, cond.col, cond.col, b.phrase_col(e.id));
            } else
                b.term_docids(cond.col, cond.term.ts);
            break;
        }
    }
}

uint32_t position_cost_from_distance(uint32_t d) {  // position/mod.rs:129-143
    if (d == 0) return 0;
    if (d == 1) return 1;
    if (d <= 4) return 2;
    if (d <= 7) return 3;
    if (d <= 11) return 4;
    if (d <= 16) return 5;
    if (d <= 24) return 6;
    if (d <= 64) return 7;
    if (d <= 256) return 8;
    if (d <= 1024) return 9;
    return 10;
}
uint16_t bucketed_position(uint16_t rel) {  // lib.rs:248-260
    if (rel < 16) return rel;
    if (rel < 24) return 24;
    uint32_t p = 1;
    while (p < rel) p <<= 1;
    return (uint16_t)p;
}

// Conditions of one rule graph.  The reference interns conditions (DedupInterner); here equal conditions can only arise from the
// same destination node (they are functions of `to`, plus `from` for proximity), so they are built once per destination and
// shared by id — no structural hashing on the hot path.
struct CondTable {
    std::vector<ECond> items;
    CondTable() { items.reserve(48); }
    uint32_t insert(ECond &&c) {
        items.push_back(std::move(c));
        return (uint32_t)items.size() - 1;
    }
};

// G::build_edges for the six graph rules
std::vector<std::pair<uint32_t, uint32_t>> build_edges(const QCtx &c, int rule, CondTable &ct, const ELocated *from, const ELocated &to,
                                                     int32_t *base_cache = nullptr) {
    std::vector<std::pair<uint32_t, uint32_t>> edges;
    auto base_id = [&]() -> uint32_t {
        if (base_cache && *base_cache >= 0) return (uint32_t)*base_cache;
        ECond x;
        x.rule = rule;
        x.term = to;
        x.end_subset = to;
        uint32_t id = ct.insert(std::move(x));
        if (base_cache) *base_cache = (int32_t)id;
        return id;
    };
    auto base = [&]() {
        ECond x;
        x.rule = rule;
        x.term = to;
        x.end_subset = to;
        return x;
    };
    switch (rule) {
        case RK_WORDS: edges.push_back({0, ct.insert(base())}); break;
        case RK_TYPO: {  // typo/mod.rs:42-77
            uint32_t bc = to.n_term_ids() == 1 ? 0 : to.n_term_ids();
            uint8_t mx = max_typo_cost(c, to.ts);
            for (uint8_t n = 0; n <= mx; n++) {
                ECond x = base();
                x.nbr_typos = n;
                if (n != 0) x.term.ts.zero = ESubset{};
                if (n != 1) x.term.ts.one = ESubset{};
                if (n != 2) x.term.ts.two = ESubset{};
                x.end_subset = x.term;
                edges.push_back({n + bc, ct.insert(std::move(x))});
            }
            break;
        }
        case RK_PROXIMITY: {  // proximity/build.rs:10-56
            uint32_t rmax = to.n_term_ids() - 1;
            if (!from || (uint16_t)(from->pe + 1) != to.ps) {
                edges.push_back({rmax, base_id()});
                break;
            }
            for (uint32_t cost = rmax; cost < 3 + rmax; cost++) {
                ECond x = base();
                x.prox_uninit = true;
                x.left = *from;
                x.cost = (uint8_t)(cost + 1);
                x.has_start = true;
                x.start_subset = *from;
                edges.push_back({cost, ct.insert(std::move(x))});
            }
            edges.push_back({3 + rmax, base_id()});
            break;
        }
        case RK_FID: {  // fid/mod.rs:49-121; edge order: ascending fid (the reference iterates an FxHashSet)
            std::set<uint16_t> fields;
            for (auto &w : all_single_words(c, to.ts))
                for (uint32_t i = c.ix.wf_off[w.rank]; i < c.ix.wf_off[w.rank + 1]; i++) fields.insert(c.ix.wf_fid[i]);
            for (auto p : all_phrases(c, to.ts))
                for (auto w : c.phrases[p].words)
                    if (w >= 0)
                        for (uint32_t i = c.ix.wf_off[w]; i < c.ix.wf_off[w + 1]; i++) fields.insert(c.ix.wf_fid[i]);
            uint32_t pid;
            bool derived;
            if (use_prefix_db(c, to.ts, pid, derived))
                for (uint32_t i = c.ix.pf_off[pid]; i < c.ix.pf_off[pid + 1]; i++) fields.insert(c.ix.pf_fid[i]);
            uint16_t cur_max = 0;
            for (auto fid : fields) {
                if (fid >= c.ix.settings.weights.size()) continue;
                uint16_t weight = c.ix.settings.weights[fid];
                cur_max = std::max(cur_max, weight);
                ECond x = base();
                x.has_fid = true;
                x.fid = fid;
                edges.push_back({(uint32_t)weight * to.n_term_ids(), ct.insert(std::move(x))});
            }
            uint16_t mw = c.ix.settings.max_weight();
            if (cur_max < mw) edges.push_back({(uint32_t)mw * to.n_term_ids(), ct.insert(base())});
            break;
        }
        case RK_POSITION: {  // position/mod.rs:50-126; edge order: ascending cost (FxHashMap in the reference)
            std::set<uint16_t> all_pos;
            for (auto &w : all_single_words(c, to.ts))
                for (uint32_t i = c.ix.wp_off[w.rank]; i < c.ix.wp_off[w.rank + 1]; i++) all_pos.insert(c.ix.wp_pos[i]);
            for (auto p : all_phrases(c, to.ts)) {
                int32_t w = QCtx::first_word(c.phrases[p]);
                if (w >= 0)
                    for (uint32_t i = c.ix.wp_off[w]; i < c.ix.wp_off[w + 1]; i++) all_pos.insert(c.ix.wp_pos[i]);
            }
            uint32_t pid;
            bool derived;
            if (use_prefix_db(c, to.ts, pid, derived))
                for (uint32_t i = c.ix.pp_off[pid]; i < c.ix.pp_off[pid + 1]; i++) all_pos.insert(c.ix.pp_pos[i]);
            std::map<uint32_t, std::vector<uint16_t>> by_cost;
            for (auto p : all_pos) {
                uint32_t dist = p > to.ps ? p - to.ps : to.ps - p, cost = 0;
                for (uint32_t i = 0; i < to.n_term_ids(); i++) cost += position_cost_from_distance(dist + i);
                by_cost[cost].push_back(p);
            }
            uint32_t max_cost = to.n_term_ids() * 10;
            for (auto &kv : by_cost) {
                ECond x = base();
                x.positions = kv.second;
                edges.push_back({kv.first, ct.insert(std::move(x))});
            }
            if (!by_cost.count(max_cost)) edges.push_back({max_cost, ct.insert(base())});
            break;
        }
        case RK_EXACTNESS: {  // exactness/mod.rs:45-91
            ECond e = base();
            e.exact_in_attribute = true;
            {  // end_term_subset: keep_only_exact_term + mandatory
                ExactTermRef et = exact_term(c, to.ts);
                if (et.kind) {
                    ESubset z;
                    z.kind = N_SUBSET;
                    (et.kind == 1 ? z.words : z.phrases).push_back(et.id);
                    e.end_subset.ts.zero = z;
                    e.end_subset.ts.one = ESubset{};
                    e.end_subset.ts.two = ESubset{};
                }
                e.end_subset.ts.mandatory = true;
            }
            uint32_t ei = ct.insert(std::move(e)), ai = ct.insert(base());
            edges.push_back({0, ei});
            edges.push_back({to.n_term_ids(), ai});
            break;
        }
    }
    return edges;
}

// Topologically order the states reachable from START that reach END, compute per-state feasible cost ranges, root costs.
template <class AE>
void finish_state_graph(Level &L, const std::vector<AE> &aedges, uint32_t root, uint32_t end, bool want_paths) {
    uint32_t max_id = std::max(root, end);
    for (auto &e : aedges) max_id = std::max(max_id, std::max(e.src, e.dst));
    const uint32_t NS = max_id + 1;
    // adjacency in insertion (= visiting) order
    std::vector<uint32_t> deg(NS + 1, 0);
    for (auto &e : aedges) deg[e.src + 1]++;
    for (uint32_t i = 0; i < NS; i++) deg[i + 1] += deg[i];
    std::vector<uint32_t> adj(aedges.size());
    {
        std::vector<uint32_t> cur(deg.begin(), deg.end() - 1);
        for (uint32_t i = 0; i < aedges.size(); i++) adj[cur[aedges[i].src]++] = i;
    }
    // feasible costs to END (memoised DFS; post-order gives a reverse topological order)
    std::vector<std::vector<uint32_t>> costs(NS);
    std::vector<uint8_t> seen(NS, 0);
    std::vector<uint32_t> post;
    std::vector<std::pair<uint32_t, uint32_t>> stack;  // (state, next adjacency index)
    stack.push_back({root, deg[root]});
    seen[root] = 1;
    while (!stack.empty()) {
        uint32_t sst = stack.back().first;
        uint32_t &k = stack.back().second;
        if (sst != end && k < deg[sst + 1]) {
            uint32_t dst = aedges[adj[k++]].dst;
            if (!seen[dst]) {
                seen[dst] = 1;
                stack.push_back({dst, deg[dst]});
            }
            continue;
        }
        if (sst == end)
            costs[sst] = {0};
        else {
            std::vector<uint32_t> &cs = costs[sst];
            for (uint32_t kk = deg[sst]; kk < deg[sst + 1]; kk++) {
                const AE &e = aedges[adj[kk]];
                for (auto c : costs[e.dst]) cs.push_back(e.cost + c);
            }
            std::sort(cs.begin(), cs.end());
            cs.erase(std::unique(cs.begin(), cs.end()), cs.end());
        }
        post.push_back(sst);
        stack.pop_back();
    }
    std::vector<uint32_t> order;
    for (auto it = post.rbegin(); it != post.rend(); ++it)
        if (*it != end && !costs[*it].empty()) order.push_back(*it);
    if (order.empty() || order[0] != root) order.insert(order.begin(), root);  // START with no way to END: no buckets
    order.push_back(end);
    std::vector<int32_t> idx(NS, -1);
    for (size_t i = 0; i < order.size(); i++) idx[order[i]] = (int32_t)i;
    L.n_states = (uint16_t)order.size();
    L.sedges.clear();
    L.state_edge_begin.assign(L.n_states + 1, 0);
    L.state_cost_range.assign(L.n_states, {0, 0});
    for (size_t i = 0; i < order.size(); i++) {
        L.state_edge_begin[i] = (uint32_t)L.sedges.size();
        uint32_t sst = order[i];
        if (!costs[sst].empty()) {
            uint32_t lo = costs[sst].front(), hi = costs[sst].back();
            if (hi >= 65535) throw TooComplex{"ranking-rule cost above 65534"};
            L.state_cost_range[i] = {(uint16_t)lo, (uint16_t)(hi - lo + 1)};
        }
        if (sst == end) continue;
        for (uint32_t kk = deg[sst]; kk < deg[sst + 1]; kk++) {
            const AE &e = aedges[adj[kk]];
            if (idx[e.dst] < 0) continue;
            if (e.dst != end && costs[e.dst].empty()) continue;
            L.sedges.push_back(SEdge{(uint16_t)i, (uint16_t)idx[e.dst], e.cost, e.cond});
        }
    }
    L.state_edge_begin[L.n_states] = (uint32_t)L.sedges.size();
    L.cost_vals.assign(costs[root].begin(), costs[root].end());
    if (L.cost_vals.size() > MAX_COSTS) throw TooComplex{"more than 128 distinct costs in one ranking rule"};
    if (L.sedges.size() > 60000) throw TooComplex{"ranking-rule graph too large"};
    L.want_paths = want_paths;
}

// Build graph + enumerate all START->END paths (cheapest_paths.rs semantics without the dead-end cache: every
// path is handed to the device, which finds the empty ones itself).
void prepare_graph_rule(const QCtx &c, int rule, bool has_tms, int tms, Level &L) {
    const EGraph &qg = L.graph;
    uint16_t n = (uint16_t)qg.nodes.size();
    // cost of ignoring a node (graph_based_ranking_rule.rs:149-193)
    std::vector<int> ignore_cost(n, -1);
    if (has_tms && (tms == B200_TMS_LAST || tms == B200_TMS_FREQUENCY))
        for (auto &grp : removal_order(c, qg, tms))
            for (auto nd : grp) ignore_cost[nd] = 1;
    CondTable ct;
    std::vector<EEdge> edges;
    std::vector<std::vector<uint32_t>> eon(n);
    // every (src, dst) pair is visited once, so edges are distinct by construction; conditions that depend on the destination only
    // are built once per destination and shared by all its predecessors
    std::vector<std::vector<std::pair<uint32_t, uint32_t>>> dst_edges(n);
    std::vector<uint8_t> dst_done(n, 0);
    std::vector<int32_t> base_cond(n, -1);
    for (uint16_t src = 0; src < n; src++) {
        const ENode &sn = qg.nodes[src];
        if (sn.kind != ND_TERM && sn.kind != ND_START) continue;
        for (auto dst : sn.succ) {
            const ENode &dn = qg.nodes[dst];
            if (dn.kind == ND_END) {
                edges.push_back(EEdge{src, dst, 0, -1});
                eon[src].push_back((uint32_t)edges.size() - 1);
                continue;
            }
            if (ignore_cost[dst] >= 0) {
                edges.push_back(EEdge{src, dst, (uint32_t)ignore_cost[dst] * dn.term.n_term_ids(), -1});
                eon[src].push_back((uint32_t)edges.size() - 1);
            }
            const std::vector<std::pair<uint32_t, uint32_t>> *es;
            std::vector<std::pair<uint32_t, uint32_t>> pair_edges;
            if (rule == RK_PROXIMITY) {
                pair_edges = build_edges(c, rule, ct, sn.kind == ND_TERM ? &sn.term : nullptr, dn.term, &base_cond[dst]);
                es = &pair_edges;
            } else {
                if (!dst_done[dst]) {
                    dst_edges[dst] = build_edges(c, rule, ct, nullptr, dn.term);
                    dst_done[dst] = 1;
                }
                es = &dst_edges[dst];
            }
            for (auto &e : *es) {
                edges.push_back(EEdge{src, dst, e.first, (int32_t)e.second});
                eon[src].push_back((uint32_t)edges.size() - 1);
            }
        }
    }
    L.conds = std::move(ct.items);
    // max cost over the graph ignoring skip constraints (the maximum of find_all_costs_to_end :285-310)
    uint64_t mx = 0;
    {
        std::vector<int64_t> best(n, -2);  // -2 unvisited, -1 END unreachable
        std::vector<std::pair<uint16_t, uint32_t>> stk{{qg.root, 0}};
        while (!stk.empty()) {
            uint16_t nd = stk.back().first;
            uint32_t &k = stk.back().second;
            if (nd == qg.end) {
                best[nd] = 0;
                stk.pop_back();
                continue;
            }
            if (k < eon[nd].size()) {
                uint16_t d2 = edges[eon[nd][k++]].dst;
                if (best[d2] == -2) {
                    best[d2] = -3;  // on the stack (the graph is a DAG)
                    stk.push_back({d2, 0});
                }
                continue;
            }
            int64_t m = -1;
            for (auto ei : eon[nd])
                if (best[edges[ei].dst] >= 0) m = std::max<int64_t>(m, (int64_t)edges[ei].cost + best[edges[ei].dst]);
            best[nd] = m;
            stk.pop_back();
        }
        mx = best[qg.root] > 0 ? (uint64_t)best[qg.root] : 0;
    }
    L.next_max_cost = 1 + mx;
    if (has_tms) {  // words matched inside phrases count too (graph_based_ranking_rule.rs:149-157)
        size_t wip = 0;
        for (auto &nd : qg.nodes) {
            uint32_t ph;
            if (nd.kind == ND_TERM && original_phrase(c, nd.term.ts, ph))
                for (auto w : c.phrases[ph].words)
                    if (w != -1) wip++;
        }
        L.next_max_cost += wip > 0 ? wip - 1 : 0;
    }
    // state graph for the device.  Without a matching strategy a state is a query-graph node.  With `Last`, skipping a node of
    // removal group k forbids matching any node of a cheaper group afterwards (the skip edge's `nodes_to_skip`,
    // cheapest_paths.rs:189-281 with the removal order of query_graph.rs:346-406); mandatory nodes (phrases) stay matchable.
    // The groups are nested, so a state is (node, m) = "nodes of groups < m are forbidden", canonicalised to the groups that
    // still occur among the node's descendants.
    struct AEdge {
        uint32_t src, dst, cost;
        int32_t cond;
    };
    std::vector<AEdge> aedges;
    std::vector<uint16_t> grp(n, 0);  // 1-based removal group, 0 = never removed
    if (has_tms && (tms == B200_TMS_LAST || tms == B200_TMS_FREQUENCY)) {
        uint16_t k = 1;
        for (auto &g : removal_order(c, qg, tms)) {
            for (auto nd : g) grp[nd] = k;
            k++;
        }
    }
    // descendants' groups: dgrp[nd] = sorted distinct groups (>0) among strict descendants of nd
    std::vector<std::vector<uint16_t>> dgrp(n);
    {
        std::vector<uint8_t> done(n, 0);
        std::function<void(uint16_t)> go = [&](uint16_t nd) {
            if (done[nd]) return;
            done[nd] = 1;
            std::vector<uint16_t> &d = dgrp[nd];
            for (auto s2 : qg.nodes[nd].succ) {
                go(s2);
                if (grp[s2]) d.push_back(grp[s2]);
                d.insert(d.end(), dgrp[s2].begin(), dgrp[s2].end());
            }
            std::sort(d.begin(), d.end());
            d.erase(std::unique(d.begin(), d.end()), d.end());
        };
        go(qg.root);
    }
    auto canon = [&](uint16_t nd, uint16_t m) -> uint16_t {  // 1 + largest descendant group below m, or 0
        const std::vector<uint16_t> &d = dgrp[nd];
        auto it = std::lower_bound(d.begin(), d.end(), m);
        return it == d.begin() ? 0 : (uint16_t)(*(it - 1) + 1);
    };
    std::map<std::pair<uint16_t, uint16_t>, uint32_t> sids;
    std::vector<std::pair<uint16_t, uint16_t>> work;
    auto sid = [&](uint16_t node, uint16_t m) {
        if (node == qg.end) m = 0;
        auto key = std::make_pair(node, m);
        auto it = sids.find(key);
        if (it != sids.end()) return it->second;
        uint32_t id = (uint32_t)sids.size();
        sids.emplace(key, id);
        work.push_back(key);
        return id;
    };
    uint32_t root_sid = sid(qg.root, 0), end_sid = sid(qg.end, 0);
    for (size_t wi = 0; wi < work.size(); wi++) {
        auto [nd, m] = work[wi];
        if (nd == qg.end) continue;
        uint32_t from = sids[work[wi]];
        for (auto ei : eon[nd]) {
            const EEdge &e = edges[ei];
            if (e.dst == qg.end) {
                aedges.push_back({from, end_sid, e.cost, -1});
            } else if (e.cond >= 0) {
                if (grp[e.dst] && grp[e.dst] < m) continue;  // nodes_to_skip.contains(dest)
                aedges.push_back({from, sid(e.dst, canon(e.dst, m)), e.cost, e.cond});
            } else {
                uint16_t m2 = std::max<uint16_t>(m, grp[e.dst]);
                aedges.push_back({from, sid(e.dst, canon(e.dst, m2)), e.cost, -1});  // skip edge
            }
        }
    }
    finish_state_graph(L, aedges, root_sid, end_sid, true);
}

// universe resolution (resolve_query_graph.rs:133-185 == union over START->END routes of the AND of the term docids)
void prepare_resolve(const QCtx &c, Level &L) {
    const EGraph &g = L.graph;
    L.conds.clear();
    std::vector<int> cond_of(g.nodes.size(), -1);
    for (uint16_t i = 0; i < g.nodes.size(); i++)
        if (g.nodes[i].kind == ND_TERM) {
            ECond x;
            x.rule = RK_RESOLVE;
            x.term = g.nodes[i].term;
            x.end_subset = x.term;
            cond_of[i] = (int)L.conds.size();
            L.conds.push_back(x);
        }
    struct AEdge {
        uint32_t src, dst, cost;
        int32_t cond;
    };
    std::vector<AEdge> ae;
    for (uint16_t u = 0; u < g.nodes.size(); u++) {
        if (g.nodes[u].kind != ND_TERM && g.nodes[u].kind != ND_START) continue;
        for (auto v : g.nodes[u].succ) ae.push_back({u, v, 0, v == g.end ? -1 : cond_of[v]});
    }
    finish_state_graph(L, ae, g.root, g.end, false);
    L.next_max_cost = 1;
    (void)c;
}

// exact_attribute.rs:96-240 as three first-match paths: [A]=ExactMatch, [B]=MatchesStart, []=NoExactMatch
void prepare_exact_attribute(const QCtx &c, Level &L, StepOut &o) {
    const EGraph &g = L.graph;
    ActBuilder b(c, o);
    uint16_t colA = b.new_col(), colB = b.new_col();
    L.conds.clear();
    for (int k = 0; k < 2; k++) {
        ECond x;
        x.rule = RK_EXACT_ATTRIBUTE;
        x.col = k == 0 ? colA : colB;
        L.conds.push_back(x);
    }
    {
        struct AEdge {
            uint32_t src, dst, cost;
            int32_t cond;
        };
        std::vector<AEdge> ae{{0, 1, 0, 0}, {0, 1, 1, 1}, {0, 1, 2, -1}, {1, 2, 0, -1}};
        finish_state_graph(L, ae, 0, 2, false);
    }
    L.next_max_cost = 3;
    struct Info {
        std::vector<int32_t> words;  // the exact term's words (a phrase may hold -1 holes / -2 unknown words)
        uint16_t start_position;
        uint8_t start_term_id;
        size_t position_count;
    };
    std::vector<Info> ets;
    for (auto &n : g.nodes) {
        if (n.kind != ND_TERM) continue;
        ExactTermRef e = exact_term(c, n.term.ts);
        if (!e.kind) continue;
        Info inf;
        if (e.kind == 1)
            inf.words = {(int32_t)e.id};
        else
            inf.words = c.phrases[e.id].words;
        inf.start_position = n.term.ps;
        inf.start_term_id = n.term.t0;
        inf.position_count = (size_t)n.term.pe - n.term.ps + 1;
        ets.push_back(std::move(inf));
    }
    std::stable_sort(ets.begin(), ets.end(), [](const Info &a, const Info &b2) { return a.start_term_id < b2.start_term_id; });
    {
        std::vector<Info> dd;
        for (auto &e : ets)
            if (dd.empty() || dd.back().start_term_id != e.start_term_id) dd.push_back(e);
        ets.swap(dd);
    }
    size_t count_all = 0;
    for (auto &e : ets) count_all += e.position_count;
    bool empty_state = ets.empty() || ets[0].start_term_id != 0;
    uint8_t prev = 0;
    for (auto &e : ets) {
        if (e.start_term_id < prev || e.start_term_id - prev > 1) empty_state = true;
        prev = e.start_term_id;
    }
    if (!empty_state) {
        // candidates = AND over every word of every exact term of word_position[w, bucketed(pos + offset)]  (:159-186)
        uint16_t cand = b.new_col();
        bool first = true;
        for (auto &e : ets)
            for (size_t off = 0; off < e.words.size(); off++) {
                int32_t w = e.words[off];
                if (w == -1) continue;  // stop-word hole
                uint16_t t = first ? cand : b.new_col();
                if (w >= 0) b.add_list(t, c.ix.word_pos_list((uint32_t)w, bucketed_position((uint16_t)(e.start_position + off))));
                if (!first) b.op(0, cand, cand, t);
                first = false;
            }
        for (uint16_t fid = 0; fid < c.ix.settings.n_fields; fid++) {
            uint16_t swe = b.new_col();
            b.op(3, swe, cand, 0);
            for (auto &e : ets)
                for (auto w : e.words) {
                    if (w == -1) continue;
                    uint16_t t = b.new_col();
                    if (w >= 0) b.add_list(t, c.ix.word_fid_list((uint32_t)w, fid));
                    b.op(0, swe, swe, t);
                }
            uint16_t cnt = b.new_col();
            if (count_all < 255) {
                auto it = c.ix.fwc_list.find(((uint32_t)fid << 8) | (uint32_t)count_all);
                if (it != c.ix.fwc_list.end()) b.add_list(cnt, it->second);
            }
            uint16_t t1 = b.new_col();
            b.op(0, t1, swe, cnt);
            b.op(1, colA, colA, t1);
            uint16_t t2 = b.new_col();
            b.op(2, t2, swe, cnt);
            b.op(1, colB, colB, t2);
        }
    }
    o.n_cols = b.next_col;
}

// query_graph.rs:453-543
EGraph build_from_paths(const std::vector<std::vector<const ECond *>> &paths) {
    std::vector<std::vector<ELocated>> single;
    for (auto &path : paths) {
        std::vector<ELocated> processed;
        bool have_prev = false;
        ELocated prev;
        for (auto *cd : path) {
            if (have_prev) {
                if (cd->has_start) {
                    ELocated start = cd->start_subset;
                    if (start.t0 == prev.t0 && start.t1 == prev.t1) {
                        start.ts.intersect(prev.ts);
                        processed.push_back(start);
                    } else {
                        processed.push_back(prev);
                        processed.push_back(start);
                    }
                } else
                    processed.push_back(prev);
            } else if (cd->has_start)
                processed.push_back(cd->start_subset);
            prev = cd->end_subset;
            have_prev = true;
        }
        if (have_prev) processed.push_back(prev);
        single.push_back(std::move(processed));
    }
    EGraph g;
    g.nodes.resize(2);
    g.nodes[0].kind = ND_START;
    g.nodes[1].kind = ND_END;
    std::map<std::string, uint16_t> ids;
    std::vector<std::vector<uint16_t>> pid;
    for (auto &path : single) {
        std::vector<std::string> suffix(path.size());
        std::string acc;
        for (size_t i = path.size(); i-- > 0;) {
            std::string k;
            k.reserve(64 + acc.size());
            path[i].key(k);
            k += acc;
            acc.swap(k);
            suffix[i] = acc;
        }
        std::vector<uint16_t> p;
        for (size_t i = 0; i < path.size(); i++) {
            auto it = ids.find(suffix[i]);
            if (it == ids.end()) {
                ENode nd;
                nd.kind = ND_TERM;
                nd.term = path[i];
                g.nodes.push_back(nd);
                it = ids.emplace(suffix[i], (uint16_t)(g.nodes.size() - 1)).first;
            }
            p.push_back(it->second);
        }
        pid.push_back(std::move(p));
    }
    for (auto &p : pid) {
        uint16_t prev = g.root;
        for (auto id : p) {
            sorted_insert(g.nodes[prev].succ, id);
            sorted_insert(g.nodes[id].pred, prev);
            prev = id;
        }
        sorted_insert(g.nodes[prev].succ, g.end);
        sorted_insert(g.nodes[g.end].pred, prev);
    }
    return g;
}

// conditions -> columns, scatter jobs, column program; state graph -> device form
void emit_activation_work(const QCtx &c, Level &L, StepOut &o) {
    if (L.kind == RK_RESOLVE && L.neg_only) {
        // the single condition of the level = documents of the negative words and phrases (search/new/mod.rs:719-731); the level's
        // "unmatched" column (universe minus every bucket) is then the universe the placeholder search returns
        ActBuilder b(c, o);
        uint16_t ign = b.new_col();
        L.conds[0].col = ign;
        for (auto w : c.neg_words) b.add_word_docids(ign, WordRef{w, false});
        for (auto ph : c.neg_phrases) b.op(1, ign, ign, b.phrase_col(ph));
        o.n_cols = b.next_col;
    } else if (L.kind != RK_EXACT_ATTRIBUTE) {
        ActBuilder b(c, o);
        for (auto &cd : L.conds) cd.col = b.new_col();
        for (auto &cd : L.conds) build_cond(b, cd);
        if (L.kind == RK_RESOLVE && (!c.neg_words.empty() || !c.neg_phrases.empty())) {
            // universe -= negative words / phrases (search/mod.rs:436-437,463): every node column loses the ignored documents
            uint16_t ign = b.new_col();
            for (auto w : c.neg_words) b.add_word_docids(ign, WordRef{w, false});
            for (auto ph : c.neg_phrases) b.op(1, ign, ign, b.phrase_col(ph));
            for (auto &cd : L.conds) b.op(2, cd.col, cd.col, ign);
        }
        o.n_cols = b.next_col;
    }
    o.n_costs = (uint32_t)L.cost_vals.size();
    o.want_paths = L.want_paths ? 1 : 0;
    // every START->END path carries at least one condition unless START reaches END through unconditional edges only
    {
        std::vector<uint8_t> free_reach(L.n_states, 0);
        if (L.n_states) free_reach[0] = 1;
        for (auto &e : L.sedges)
            if (free_reach[e.src] && e.cond < 0) free_reach[e.dst] = 1;  // states are topologically ordered, edges grouped by source
        o.all_conditional = (L.n_states && free_reach[L.n_states - 1]) ? 0 : 1;
    }
    uint32_t pair = 0;
    for (uint16_t st = 0; st < L.n_states; st++) {
        DpState ds{};
        ds.edge_begin = L.state_edge_begin[st];
        ds.n_edges = (uint16_t)(L.state_edge_begin[st + 1] - L.state_edge_begin[st]);
        ds.rmin = L.state_cost_range[st].first;
        ds.rcount = L.state_cost_range[st].second;
        if (st + 1 == L.n_states) {  // END: the single pair (cost 0)
            ds.rmin = 0;
            ds.rcount = 1;
        }
        ds.pair_off = pair;
        pair += ds.rcount;
        o.dp_states.push_back(ds);
    }
    o.n_pairs = std::max(1u, pair);
    for (auto &e : L.sedges) {
        if (e.cost > 65534) throw TooComplex{"edge cost too large"};
        o.dp_edges.push_back(DpEdge{e.dst, (uint16_t)e.cost, e.cond >= 0 ? L.conds[e.cond].col : (uint16_t)0xffff, 0});
    }
    for (auto cv : L.cost_vals) o.cost_vals.push_back((uint16_t)cv);
    // The DP as a straight-line program over the row's slots (condition columns first, then the (state, cost) pairs): pairs in
    // descending order = states in reverse topological order; one op per feasible edge, the last one of a pair flagged.
    const uint32_t n_cols = std::max(1u, o.n_cols), n_pairs = o.n_pairs;
    if (n_cols + n_pairs + EVAL_EXTRA_SLOTS > 0x7ffe) throw TooComplex{"ranking-rule step with more than 32764 columns"};
    const uint32_t zero_slot = n_cols + n_pairs, ones_slot = zero_slot + 1;
    o.prog.clear();
    for (int sidx = (int)o.dp_states.size() - 2; sidx >= 0; sidx--) {  // END (last state) is the seed, not computed
        const DpState &ss = o.dp_states[sidx];
        for (int k = (int)ss.rcount - 1; k >= 0; k--) {
            const int r = (int)ss.rmin + k;
            const size_t first = o.prog.size();
            for (uint32_t e = 0; e < ss.n_edges; e++) {
                const DpEdge &ee = o.dp_edges[ss.edge_begin + e];
                const DpState &ds = o.dp_states[ee.dst];
                const int rr = r - (int)ee.cost;
                if (rr < (int)ds.rmin || rr >= (int)ds.rmin + (int)ds.rcount) continue;
                o.prog.push_back((n_cols + ds.pair_off + (uint32_t)(rr - (int)ds.rmin)) | ((ee.col == 0xffff ? ones_slot : (uint32_t)ee.col) << 16));
            }
            if (o.prog.size() == first) o.prog.push_back(zero_slot | (zero_slot << 16));
            o.prog.back() |= 0x8000u;
        }
    }
    while (o.prog.size() % 4) o.prog.push_back(zero_slot | (zero_slot << 16));
}

// located_query_terms_from_tokens (parse_query.rs:28-202)
void parse_query(QState &q, const b200_query_batch *b, uint32_t qi) {
    QCtx &c = q.ctx;
    const HostIndex &ix = c.ix;
    struct Tok {
        int kind;
        std::string lemma;
    };
    std::vector<Tok> toks;
    for (uint32_t t = b->token_begin[qi]; t < b->token_begin[qi + 1]; t++)
        toks.push_back({b->token_kind[t], std::string(b->lemma_bytes + b->lemma_off[t], b->lemma_off[t + 1] - b->lemma_off[t])});
    if (toks.size() > 1000) toks.resize(1000);  // MAX_TOKEN_COUNT
    struct Located {
        uint32_t term;
        uint16_t ps, pe;
    };
    std::vector<Located> located;
    struct PhraseBuilder {
        std::vector<int32_t> words;
        uint16_t start = 0xffff, end = 0xffff;
        bool is_empty() const {
            for (auto w : words)
                if (w != -1) return false;
            return true;
        }
    };
    auto build_phrase = [&](PhraseBuilder &pb, Located &out) -> bool {
        if (pb.is_empty()) return false;
        EPhrase p;
        p.words = pb.words;
        ETerm t;
        t.phrase = (int32_t)c.intern_phrase(p);
        t.original = "\x01phrase";
        c.terms.push_back(std::move(t));
        out = Located{(uint32_t)c.terms.size() - 1, pb.start, pb.end};
        return true;
    };
    uint16_t position = 0xffff;
    bool encountered_whitespace = true, negative_next_token = false, negative_phrase = false, has_phrase = false;
    PhraseBuilder phrase;
    size_t words_limit = b->words_limit ? b->words_limit : 10;
    bool limit_hit = false;
    for (size_t ti = 0; ti < toks.size(); ti++) {
        const Tok &tk = toks[ti];
        if (tk.lemma.empty()) continue;
        if (located.size() >= words_limit) {
            limit_hit = true;
            break;
        }
        bool has_next = ti + 1 < toks.size();
        if (tk.kind == 0 || tk.kind == 1) {
            position = (uint16_t)(position + 1);
            if (has_phrase) {
                if (phrase.is_empty()) phrase.start = position;
                phrase.end = position;
                phrase.words.push_back(tk.kind == 1 ? -1 : c.word_rank_or_absent(tk.lemma));
            } else if (negative_next_token) {
                int64_t r = ix.find_word(tk.lemma);
                if (r >= 0) c.neg_words.push_back((uint32_t)r);
                negative_next_token = false;
            } else if (has_next) {
                if (tk.kind == 0) {
                    c.terms.push_back(term_from_word(c, tk.lemma, number_of_typos_allowed(ix, tk.lemma), false, false));
                    located.push_back({(uint32_t)c.terms.size() - 1, position, position});
                }
            } else {
                c.terms.push_back(term_from_word(c, tk.lemma, number_of_typos_allowed(ix, tk.lemma), ix.settings.prefix_search, false));
                located.push_back({(uint32_t)c.terms.size() - 1, position, position});
            }
        } else {
            bool hard = tk.kind == 3;
            if (hard) position = (uint16_t)(position + 7);
            bool had = has_phrase;
            PhraseBuilder cur = phrase;
            has_phrase = false;
            phrase = PhraseBuilder();
            if (hard && had) {  // a hard separator inside a phrase closes it and immediately opens a new one
                Located lt;
                if (build_phrase(cur, lt)) {
                    if (negative_phrase)
                        c.neg_phrases.push_back((uint32_t)c.terms[lt.term].phrase);
                    else
                        located.push_back(lt);
                }
                cur = PhraseBuilder();
            }
            size_t quotes = 0;
            for (char ch : tk.lemma)
                if (ch == '"') quotes++;
            if (quotes == 0) {
                has_phrase = had;
                phrase = cur;
            } else {
                if (had) {
                    quotes -= 1;
                    Located lt;
                    if (build_phrase(cur, lt)) {
                        if (negative_phrase) {
                            c.neg_phrases.push_back((uint32_t)c.terms[lt.term].phrase);
                            negative_phrase = false;
                        } else
                            located.push_back(lt);
                    }
                }
                if (quotes % 2 == 1) {
                    negative_phrase = negative_next_token;
                    has_phrase = true;
                    phrase = PhraseBuilder();
                }
            }
            negative_next_token = !has_phrase && tk.lemma == "-" && encountered_whitespace;
        }
        char last = tk.lemma.back();
        encountered_whitespace = (last == ' ' || last == '\t' || last == '\n');
    }
    if (!limit_hit && has_phrase) {  // a quote that is never closed: the rest of the query is the phrase
        Located lt;
        if (build_phrase(phrase, lt)) {
            if (negative_phrase)
                c.neg_phrases.push_back((uint32_t)c.terms[lt.term].phrase);
            else
                located.push_back(lt);
        }
    }
    // QueryGraph::from_query (query_graph.rs:96-187) + make_ngram (parse_query.rs:227-300)
    EGraph &g = q.graph;
    g.nodes.clear();
    g.nodes.resize(2);
    g.nodes[0].kind = ND_START;
    g.nodes[1].kind = ND_END;
    auto add_term_node = [&](uint32_t term, uint16_t ps, uint16_t pe, uint8_t t0, uint8_t t1) {
        ENode n;
        n.kind = ND_TERM;
        n.term.ts = ETermSubset::full(term);
        n.term.ps = ps;
        n.term.pe = pe;
        n.term.t0 = t0;
        n.term.t1 = t1;
        g.nodes.push_back(n);
    };
    auto make_ngram = [&](size_t from, size_t to) -> bool {
        for (size_t i = from; i <= to; i++)
            if (c.terms[located[i].term].phrase >= 0) return false;
        for (size_t i = from; i < to; i++)
            if (located[i].pe != (uint16_t)(located[i + 1].ps - 1)) return false;
        std::string s;
        std::vector<std::string> ws;
        for (size_t i = from; i <= to; i++) {
            ws.push_back(c.terms[located[i].term].original);
            s += ws.back();
        }
        if (s.size() > 250) return false;
        bool is_prefix = c.terms[located[to].term].is_prefix;
        uint8_t n = number_of_typos_allowed(ix, s), dec = (uint8_t)(to - from);
        ETerm t = term_from_word(c, s, n > dec ? (uint8_t)(n - dec) : 0, is_prefix, true);
        auto it = ix.settings.synonyms.find(ws);
        if (it != ix.settings.synonyms.end()) {
            for (auto &syn : it->second) {
                EPhrase p;
                for (auto &w : syn) p.words.push_back(c.word_rank_or_absent(w));
                t.synonyms.push_back(c.intern_phrase(p));
            }
            std::sort(t.synonyms.begin(), t.synonyms.end());
            t.synonyms.erase(std::unique(t.synonyms.begin(), t.synonyms.end()), t.synonyms.end());
        }
        t.ngram_words = ws;
        t.is_ngram = true;
        c.terms.push_back(std::move(t));
        add_term_node((uint32_t)c.terms.size() - 1, located[from].ps, located[to].pe, (uint8_t)from, (uint8_t)to);
        return true;
    };
    if (located.size() > 12) throw UnsupportedQuery{"more than 12 query terms"};
    for (size_t i = 0; i < located.size(); i++) {
        add_term_node(located[i].term, located[i].ps, located[i].pe, (uint8_t)i, (uint8_t)i);
        if (i >= 1) make_ngram(i - 1, i);
        if (i >= 2) make_ngram(i - 2, i);
    }
    build_initial_edges(g);
    q.used_negative = !c.neg_words.empty() || !c.neg_phrases.empty();
    // no positive term: a placeholder search (search/new/mod.rs:733-737) — over the universe minus the negative terms' documents
    // when there are any (:719-731), which needs one device step
    q.neg_only = located.empty() && q.used_negative;
    q.placeholder = located.empty() && !q.used_negative;
}

// get_ranking_rules_for_query_graph_search (search/new/mod.rs:510-649)
std::vector<int> rule_list(const Settings &s, int tms) {
    std::vector<int> rules;
    bool words = tms == B200_TMS_ALL, typo = false, prox = false, attr = false, attr_rank = false, wpos = false, exact = false;
    for (int rr : s.criteria) {
        if ((rr == B200_C_TYPO || rr == B200_C_ATTRIBUTE || rr == B200_C_ATTRIBUTE_RANK || rr == B200_C_WORD_POSITION || rr == B200_C_PROXIMITY ||
             rr == B200_C_EXACTNESS) &&
            !words) {
            rules.push_back(RK_WORDS);
            words = true;
        }
        switch (rr) {
            case B200_C_WORDS:
                if (!words) {
                    rules.push_back(RK_WORDS);
                    words = true;
                }
                break;
            case B200_C_TYPO:
                if (!typo) {
                    typo = true;
                    rules.push_back(RK_TYPO);
                }
                break;
            case B200_C_PROXIMITY:
                if (!prox) {
                    prox = true;
                    rules.push_back(RK_PROXIMITY);
                }
                break;
            case B200_C_ATTRIBUTE:
                if (!(attr || attr_rank || wpos)) {
                    attr = true;
                    rules.push_back(RK_FID);
                    rules.push_back(RK_POSITION);
                }
                break;
            case B200_C_ATTRIBUTE_RANK:
                if (!(attr || attr_rank)) {
                    attr_rank = true;
                    rules.push_back(RK_FID);
                }
                break;
            case B200_C_WORD_POSITION:
                if (!(attr || wpos)) {
                    wpos = true;
                    rules.push_back(RK_POSITION);
                }
                break;
            case B200_C_EXACTNESS:
                if (!exact) {
                    exact = true;
                    rules.push_back(RK_EXACT_ATTRIBUTE);
                    rules.push_back(RK_EXACTNESS);
                }
                break;
            default: break;  // sort: no sort criteria on this path
        }
    }
    return rules;
}

uint8_t score_kind_of(int rk) {
    switch (rk) {
        case RK_WORDS: return B200_S_WORDS;
        case RK_TYPO: return B200_S_TYPO;
        case RK_PROXIMITY: return B200_S_PROXIMITY;
        case RK_FID: return B200_S_FID;
        case RK_POSITION: return B200_S_POSITION;
        case RK_EXACT_ATTRIBUTE: return B200_S_EXACT_ATTRIBUTE;
        default: return B200_S_EXACT_WORDS;
    }
}

// ScoreDetails::global_score over rank-valued details (score_details.rs:133-154, Rank::merge :524-547); Skipped = Rank{0, 1}
double global_score_of(const std::vector<EScore> &sc) {
    uint64_t rk = 1, mx = 1;
    for (auto &x : sc) {
        if (x.kind == B200_S_VECTOR || x.kind == B200_S_SORT || x.kind == B200_S_GEO_SORT) continue;  // no Rank (score_details.rs:110-154)
        rk = rk > 0 ? rk - 1 : 0;
        rk = rk * x.max_rank + x.rank;
        mx *= x.max_rank;
    }
    return (double)rk / (double)mx;
}

}  // namespace

// S1: an opaque query graph (QueryGraph + the terms it refers to)
struct GraphObj {
    QCtx ctx;
    EGraph graph;
    GraphObj(const QCtx &c, const EGraph &g) : ctx(c), graph(g) {}
};
// S1: one bucket of the rule rule_start ran, in ascending cost order (empty buckets included)
struct RuleBucket {
    uint32_t rank, max_rank;
    uint64_t count;
    std::vector<uint64_t> bitmap;  // dense, n_words64 words
    GraphObj *child = nullptr;     // the query graph of the paths that produced the bucket (nullptr: no path information)
};

namespace {

// worker threads of the host phases (B200_HOST_THREADS; the calling thread counts as one)
unsigned host_threads() {
    unsigned hw = std::thread::hardware_concurrency();
    const char *env = getenv("B200_HOST_THREADS");
    return env ? (unsigned)atoi(env) : std::max(4u, std::min(32u, hw / 2));
}

// An activation waiting in a lane: its query and its request
struct Cand {
    uint32_t qi;
    Pending *pd;
};
// Where pass 1 placed one scheduled activation: its offsets in every section of the step blob, its device memory and its row table
struct Plan {
    uint32_t jobs, sets, words, colprog, states, edges, costs, tiles, probes, res_off, ctiles, n_seg, prog;
    uint32_t ld, cls, tab_size, rpt, rt_slot, rt_tag;
    uint8_t *pb;
    size_t coff, toff, soff_from_end;
    bool identity;
};
// One step of a lane: what joins it (pass 1), the totals that size its blob and where the blob's sections start (pass 2)
struct Step {
    std::vector<uint32_t> emit_q;
    std::vector<Cand> cand_q;
    std::vector<Plan> plan;
    std::vector<size_t> sched;  // indices in cand_q of the activations that join this step
    uint32_t n_jobs = 0, n_sets = 0, n_words = 0, n_colprog = 0, n_states = 0, n_edges = 0, n_costs_tot = 0, n_tiles = 0, n_probes = 0, res_words = 0, n_prog = 0;
    uint32_t n_ctiles = 0, n_tiles_cls[EVAL_CLASSES + 1] = {};
    bool want_paths_cls[EVAL_CLASSES + 1] = {};
    bool multi_segment = false;
    size_t z_used = 0, s_used = 0;
    uint64_t compact_bytes = 0, eval_bytes = 0, fill_bytes = 0;
    uint32_t tile_base[EVAL_CLASSES + 2] = {};
    uint32_t n_emits = 0;
    size_t o_acts = 0, o_sets = 0, o_words = 0, o_colprog = 0, o_states = 0, o_edges = 0, o_costs = 0, o_prog = 0, o_tiles = 0, o_ctiles = 0, o_emits = 0,
           o_jobs = 0, o_nstatic = 0, nbytes = 0;
};
// B200_WORK_HIST=1: where the steps' work comes from (developer statistics, see tools/)
struct WorkHist {
    std::mutex mu;
    uint64_t lists[4][33][2] = {};  // [universe class][log2 card | 32 = dense] -> {lists, stored bytes}
    uint64_t eval[10][4][4] = {};   // [rule kind][universe class] -> {activations, rows(ld), rows x program ops, rows x columns}
    uint64_t probes[4] = {};
};

// One keyword_batch call: the batch, its per-query state and the lanes that step it.  The phases are member functions; the lanes'
// driver threads run launch() / finish() concurrently, each on its own lanes and queries.
struct KeywordBatch {
    using clk = std::chrono::steady_clock;
    Engine &eng;
    const HostIndex &hix;
    const DeviceIndex &dix;
    b200_stats &stats;
    Lane *const lanes;
    const b200_query_batch *b;
    b200_results *r;
    const clk::time_point t_total = clk::now();
    const uint32_t NQ, from, length;
    const int tms;
    const bool skip_scoring;
    const bool has_thr;
    const double thr;
    const bool has_budget;
    const clk::time_point deadline_at;
    const long stop_after;
    std::vector<std::unique_ptr<QState>> qs;
    const std::vector<int> rules;
    // tree-parallel bucket sort unless the order of bucket requests is observable: a deadline polls once per request, and a bucket
    // dropped by the ranking-score threshold moves every later hit forward
    const bool use_tree;
    // rule_start: the buckets of its single activation are collected here instead of being sorted further
    std::vector<RuleBucket> *rule_buckets = nullptr;
    // facets (b200_query_batch::facet_*): computed from each query's candidates where schedule() hands them over
    bool facets = false, facet_outputs = false;  // facet_outputs: facet_fid and every facet_* output are there
    // facet search (b200_query_batch::facet_search_*): each query's candidates are copied on the device where schedule() hands them
    // over, into Engine::d_fs_qcand at slot Engine::fs_slot[query]; the facet search runs over them once the batch is done
    bool fsearch = false;
    Engine::FacetOut fout;
    unsigned n_drivers = 1, lanes_per_driver = 1, n_lanes = 1;
    std::vector<std::vector<std::unique_ptr<Pending>>> lane_acts;  // per lane: the activations of its step in flight
    bool use_rowtab = false;
    std::vector<uint32_t> slot_tag;
    const uint32_t rowtab_min_rows = getenv("B200_ROWTAB_MIN") ? (uint32_t)atoi(getenv("B200_ROWTAB_MIN")) : 64;
    const uint32_t eval_rpt_big = getenv("B200_EVAL_RPT") ? (uint32_t)std::max(1, std::min(8, atoi(getenv("B200_EVAL_RPT")))) : 4;
    static constexpr size_t PATH_CAP = (size_t)1 << 20;
    const std::unique_ptr<WorkHist> work_hist{getenv("B200_WORK_HIST") ? new WorkHist() : nullptr};
    // optional host profile (B200_PROFILE=1): summed thread time per section, printed per batch
    enum ProfSection { PROF_PATHS, PROF_GRAPH_RULE, PROF_REQUEST, PROF_ADVANCE, PROF_SECTIONS };
    const bool prof = getenv("B200_PROFILE") != nullptr;
    std::atomic<uint64_t> prof_ns[PROF_SECTIONS] = {};
    struct ProfScope {
        std::atomic<uint64_t> *slot;
        clk::time_point t0;
        explicit ProfScope(std::atomic<uint64_t> *s) : slot(s) {
            if (slot) t0 = clk::now();
        }
        ProfScope(const ProfScope &) = delete;
        ~ProfScope() {
            if (slot) *slot += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(clk::now() - t0).count();
        }
    };
    ProfScope profile(ProfSection s) { return ProfScope(prof ? &prof_ns[s] : nullptr); }

    KeywordBatch(Engine &e, const b200_query_batch *batch, b200_results *res, uint32_t offset, uint32_t limit, int scoring)
        : eng(e), hix(e.hix), dix(e.dix), stats(e.stats), lanes(e.lanes), b(batch), r(res), NQ(batch->n_queries), from(offset), length(limit),
          tms(batch->terms_matching_strategy), skip_scoring(scoring == 0), has_thr(batch->has_ranking_score_threshold != 0),
          thr(batch->ranking_score_threshold), has_budget(batch->time_budget_ns > 0), deadline_at(t_total + std::chrono::nanoseconds(batch->time_budget_ns)),
          stop_after((long)batch->stop_after), qs(batch->n_queries), rules(rule_list(e.hix.settings, batch->terms_matching_strategy)),
          use_tree(stop_after < 0 && !has_budget && !has_thr && !getenv("B200_NO_TREE")) {
        if (!eng.pool) eng.pool.reset(new WorkerPool(std::max(1u, host_threads()) - 1));  // the calling thread works too
        for (uint32_t i = 0; i < NQ; i++) qs[i].reset(new QState(hix));
    }
    int fail(int code, const std::string &msg) { return eng.fail(code, msg); }
    int cuda_fail(cudaError_t e, const char *what) { return eng.cuda_fail(e, what); }
    static double ms_since(clk::time_point t) { return std::chrono::duration<double, std::milli>(clk::now() - t).count(); }
    void pfor(size_t n, std::function<void(size_t)> f) { eng.pool->run(n, std::move(f)); }
    // filtered_universe of a query on the device
    const unsigned long long *universe_of(const QState &q) const { return q.d_univ ? q.d_univ : dix.base_ub; }
    // contiguous query ranges per lane, so that the first half of the drivers can start while the second half's terms are derived
    uint32_t lane_lo(unsigned l) const { return (uint32_t)((uint64_t)NQ * l / n_lanes); }

    // ---- phase 1: tokens -> terms -> query graph
    void parse() {
        auto t_ph = clk::now();
        pfor(NQ, [&](size_t i) {
            QState &q = *qs[i];
            try {
                parse_query(q, b, (uint32_t)i);
            } catch (const UnsupportedQuery &u) {
                q.status = B200_ERR_UNSUPPORTED;
                q.error = u.why;
                q.done = true;
            }
        });
        stats.host_ms[0] += ms_since(t_ph);
    }
    void resolve_sort_rules() {
        for (uint32_t i = 0; i < NQ; i++) {
            QState &q = *qs[i];
            if (q.done) continue;
            const char *why = nullptr;
            const int code = eng.sort_rules(b, i, false, q.placeholder, q.sort_rules, why);
            if (code != B200_OK) {
                q.status = code;
                q.error = why;
                q.done = true;
            }
        }
    }
    // ---- facets: the queries that cannot have them fail alone; the others' slots get device outputs, and every lane room for the
    // counts of its queries' slots (in chunks of at most 64 MB when they are many)
    void check_facets() {
        facets = b->facet_begin != nullptr;
        if (!facets) return;
        const bool outputs = facet_outputs = b->facet_fid && r->facet_n_num && r->facet_n_str && r->facet_key && r->facet_count && r->facet_docid && r->facet_has_stats &&
                             r->facet_min && r->facet_max;
        for (uint32_t i = 0; i < NQ; i++) {
            QState &q = *qs[i];
            const uint32_t k0 = b->facet_begin[i], k1 = b->facet_begin[i + 1];
            if (q.done || k1 <= k0) continue;
            const char *why = nullptr;
            int code = B200_ERR_UNSUPPORTED;
            if (b->mode != 0)
                why = "facets in a semantic or hybrid search (use b200_facet_distribution_batch over its candidates)";
            else if (has_thr)
                why = "facets together with a ranking-score threshold";
            else if (!outputs)
                code = B200_ERR_INVALID, why = "facet_begin without facet_fid or without the facet_* outputs";
            else
                for (uint32_t k = k0; k < k1 && b->facet_order && !why; k++)
                    if (b->facet_order[k] == 1)
                        why = "facet order by count (sortFacetValuesBy: count) is not built";
                    else if (b->facet_order[k] > 1)
                        code = B200_ERR_INVALID, why = "facet_order is not 0 (alpha) or 1 (count)";
            if (why) {
                q.status = code;
                q.error = why;
                q.done = true;
            }
        }
    }
    int setup_facet_search() {
        eng.fs_slot.assign(NQ, -1);
        fsearch = b->mode == 0 && b->facet_search_fid && !has_thr;
        if (!fsearch) return B200_OK;
        const size_t W = hix.n_words64;
        size_t n = 0;
        for (uint32_t i = 0; i < NQ; i++)
            if (b->facet_search_fid[i] != 0xFFFF) eng.fs_slot[i] = (int64_t)n++;
        if (eng.d_fs_qcand.reserve(std::max<size_t>(1, n * W)) != cudaSuccess) {
            cudaGetLastError();
            return fail(B200_ERR_CAPACITY, "facet search: the batch's candidate bitmaps (one per query with a facet search) do not fit in device memory");
        }
        // a query that never hands over candidates has none
        CU(cudaMemsetAsync(eng.d_fs_qcand.p, 0, std::max<size_t>(1, n * W) * 8, eng.stream), "zero facet search candidates");
        CU(cudaStreamSynchronize(eng.stream), "sync");
        return B200_OK;
    }
    int setup_facets() {
        if (!facets) return B200_OK;
        const uint32_t n_slots = b->facet_begin[NQ];
        int rc = eng.reserve_facet_out(n_slots, b->facet_cap, fout);
        if (rc != B200_OK) return rc;
        CU(cudaMemsetAsync(fout.sum, 0, (size_t)n_slots * 16, eng.stream), "zero facet outputs");
        for (unsigned l = 0; l < n_lanes; l++) {
            std::vector<uint16_t> fids;
            for (uint32_t i : lanes[l].members)
                if (!qs[i]->done)
                    for (uint32_t k = b->facet_begin[i]; k < b->facet_begin[i + 1]; k++) fids.push_back(b->facet_fid[k]);
            if ((rc = eng.reserve_facet_scratch(fids, (size_t)64 << 20, lanes[l].d_facet, lanes[l].d_facet_slots)) != B200_OK) return rc;
        }
        return B200_OK;
    }
    // ---- filtered universes (search/new/mod.rs:719): every distinct bitmap is intersected with documents_ids and uploaded once
    int stage_universes() {
        if (r->candidates && has_thr) return fail(B200_ERR_UNSUPPORTED, "candidates bitmap together with a ranking-score threshold");
        if (r->candidates && r->candidates_words < hix.n_words64) return fail(B200_ERR_INVALID, "candidates_words smaller than the document range");
        if (b->universes) {
            const uint64_t W = hix.n_words64;
            if (b->n_universe_words < W) return fail(B200_ERR_INVALID, "universe bitmaps shorter than the document range");
            std::map<const uint64_t *, uint32_t> slot_of;
            for (uint32_t i = 0; i < NQ; i++)
                if (b->universes[i] && !geo_universe(i)) slot_of.emplace(b->universes[i], 0);
            uint32_t ns = 0;
            for (auto &kv : slot_of) kv.second = ns++;
            CU(eng.d_universes.reserve((size_t)std::max(1u, ns) * W), "alloc universes");
            std::vector<uint64_t> counts(ns, 0), tmp(W);
            for (auto &kv : slot_of) {
                uint64_t c = 0;
                for (uint64_t w = 0; w < W; w++) {
                    tmp[w] = kv.first[w] & hix.base_ub[w];
                    c += (uint64_t)__builtin_popcountll(tmp[w]);
                }
                counts[kv.second] = c;
                CU(cudaMemcpy(eng.d_universes.p + (size_t)kv.second * W, tmp.data(), W * 8, cudaMemcpyHostToDevice), "H2D universe");
                stats.h2d_bytes += W * 8;
            }
            for (uint32_t i = 0; i < NQ; i++)
                if (b->universes[i] && !geo_universe(i)) {
                    uint32_t sl = slot_of[b->universes[i]];
                    qs[i]->d_univ = eng.d_universes.p + (size_t)sl * W;
                    qs[i]->univ_count = counts[sl];
                }
        }
        // geo filters (Engine::geo_filter_universes): the query's universe already holds its caller's bitmap and clauses
        if (const Engine::GeoFiltered *gf = eng.geo_filtered)
            for (uint32_t i = 0; i < NQ; i++) {
                QState &q = *qs[i];
                if (gf->status[i] && !q.done) {
                    q.status = gf->status[i];
                    q.error = gf->error[i];
                    q.done = true;
                } else if (gf->d_univ[i]) {
                    q.d_univ = gf->d_univ[i];
                    q.univ_count = gf->count[i];
                }
            }
        for (uint32_t i = 0; i < NQ; i++)
            if (!qs[i]->d_univ) qs[i]->univ_count = hix.n_documents;
        return B200_OK;
    }
    bool geo_universe(uint32_t i) const { return eng.geo_filtered && (eng.geo_filtered->d_univ[i] || eng.geo_filtered->status[i]); }
    // ---- phase 2 (per wave, see drive_waves): typo derivations for every term of queries [lo, hi) in one device sweep
    int derive_range(uint32_t lo, uint32_t hi) {
        auto t_ph = clk::now();
        std::vector<char> wbytes;
        std::vector<uint32_t> woff{0};
        std::vector<uint8_t> mt, ip;
        std::unordered_map<std::string, int32_t> slot_of;
        for (uint32_t qi = lo; qi < hi; qi++) {
            auto &qp = qs[qi];
            if (qp->done) continue;
            for (auto &t : qp->ctx.terms) {
                if (t.empty_term || t.max_lev == 0) continue;
                if (t.original.size() > LEV_MAX_Q) {
                    qp->status = B200_ERR_UNSUPPORTED;
                    qp->error = "typo-tolerant word longer than 64 bytes";
                    qp->done = true;
                    break;
                }
                // identical (word, budget, prefix) terms of different queries share one derivation slot
                std::string key = t.original;
                key.push_back((char)('0' + t.max_lev));
                key.push_back(t.is_prefix ? 'p' : 'w');
                auto it = slot_of.find(key);
                if (it != slot_of.end()) {
                    t.lev_slot = it->second;
                    continue;
                }
                t.lev_slot = (int32_t)mt.size();
                slot_of.emplace(std::move(key), t.lev_slot);
                wbytes.insert(wbytes.end(), t.original.begin(), t.original.end());
                woff.push_back((uint32_t)wbytes.size());
                mt.push_back(t.max_lev);
                ip.push_back(t.is_prefix ? 1 : 0);
            }
        }
        uint32_t n = (uint32_t)mt.size();
        std::vector<uint32_t> one((size_t)n * 150), n_one(n), two((size_t)n * 50), n_two(n);
        if (n) {
            int rc = eng.derive_batch(n, wbytes.data(), woff.data(), mt.data(), ip.data(), one.data(), n_one.data(), two.data(), n_two.data());
            if (rc != B200_OK) return rc;
        }
        stats.host_ms[1] += ms_since(t_ph);
        t_ph = clk::now();
        pfor(hi - lo, [&](size_t i) {
            QState &q = *qs[lo + i];
            if (q.done) return;
            for (auto &t : q.ctx.terms) {
                if (t.empty_term) continue;
                if (t.lev_slot >= 0) {
                    size_t s = (size_t)t.lev_slot;
                    t.one_typo.assign(one.begin() + s * 150, one.begin() + s * 150 + n_one[s]);
                    t.two_typo.assign(two.begin() + s * 50, two.begin() + s * 50 + n_two[s]);
                }
                find_split_words(q.ctx, t);
            }
        });
        stats.host_ms[2] += ms_since(t_ph);
        return B200_OK;
    }

    // ---- phase 3: initial requests (universe resolution) or placeholder emission
    Pending *make_pending(QState &q, Level &L, const ParentRef &parent, uint64_t off0, std::vector<std::unique_ptr<Pending>> &dst) {
        ProfScope ps = profile(PROF_REQUEST);
        std::unique_ptr<Pending> pd(new Pending());
        if (L.kind == RK_EXACT_ATTRIBUTE) prepare_exact_attribute(q.ctx, L, pd->o);
        emit_activation_work(q.ctx, L, pd->o);
        // what bucket_sort can still use from this activation: the hits it has to return plus the offset it has to skip, counted from
        // the first document of this level; the walk (pass 2) only looks at the cheapest buckets that together hold that many documents
        const uint64_t window_end = (uint64_t)from + length;
        pd->need = (uint32_t)std::min<uint64_t>(0xffffffffull, window_end > off0 ? window_end - off0 : 1);
        if (pd->need == 0) pd->need = 1;
        pd->parent = parent;
        dst.push_back(std::move(pd));
        return dst.back().get();
    }
    // sequential mode: the level goes on the query's stack
    Pending *request_activation(QState &q, Level &&L, const ParentRef &parent) {
        q.levels.push_back(std::move(L));
        // documents already returned or skipped: everything before this level in result order
        Pending *pd = make_pending(q, q.levels.back(), parent, q.cur_offset, q.pendings);
        pd->L = &q.levels.back();
        return pd;
    }
    // tree mode: the level becomes a node under `parent_node`
    Pending *request_node(QState &q, Node *parent_node, Level &&L, const ParentRef &parent, uint64_t off0, std::vector<EScore> scores, ActOut *out) {
        std::unique_ptr<Node> nd(new Node());
        nd->L = std::move(L);
        nd->parent = parent_node;
        nd->off0 = off0;
        nd->scores = std::move(scores);
        if (parent_node) parent_node->live_children++;
        Node *np = nd.get();
        if (out)
            out->nodes.push_back(std::move(nd));  // the query counts it when it folds `out` in
        else {
            q.outstanding++;
            q.nodes.push_back(std::move(nd));
        }
        Pending *pd = make_pending(q, np->L, parent, off0, out ? out->pendings : q.pendings);
        pd->L = &np->L;
        pd->node = np;
        return pd;
    }
    // The Level of ranking rule `kind` at position `rule_idx` over `graph`.  The matching strategy shapes the first rule when it is
    // Words; nothing descends from a `last` rule, so its buckets are emitted without computing their paths.
    Level rule_level(const QCtx &ctx, int rule_idx, int kind, EGraph graph, bool last) {
        Level C;
        C.rule_idx = rule_idx;
        C.kind = kind;
        C.graph = std::move(graph);
        if (C.kind != RK_EXACT_ATTRIBUTE) {
            ProfScope ps = profile(PROF_GRAPH_RULE);
            prepare_graph_rule(ctx, C.kind, rule_idx == 0 && C.kind == RK_WORDS, tms, C);
        }
        if (last) C.want_paths = false;
        return C;
    }
    // The query graph of the paths that put documents into bucket `ci` of L, in visiting order (= lexicographic in edge ids): what
    // the next rule iterates on.  ExactAttribute hands its own graph down.
    EGraph child_graph(const Level &L, size_t ci) {
        if (L.kind == RK_EXACT_ATTRIBUTE) return L.graph;
        ProfScope ps = profile(PROF_PATHS);
        std::vector<const SurvPath *> sp;
        for (auto &p : L.surv)
            if (p.cost_idx == ci) sp.push_back(&p);
        std::sort(sp.begin(), sp.end(), [](const SurvPath *x, const SurvPath *y) { return x->edges < y->edges; });
        std::vector<std::vector<const ECond *>> good;
        for (auto *p : sp) {
            std::vector<const ECond *> pc;
            for (auto e : p->edges)
                if (L.sedges[e].cond >= 0) pc.push_back(&L.conds[L.sedges[e].cond]);
            good.push_back(std::move(pc));
        }
        return build_from_paths(good);
    }
    // The documents [skip, skip + take) of bucket columns [col_lo, col_hi) of L — or, without a level, of the query's universe in docid
    // order — written to offset `at` of the query's result row (the driver turns the offset into a device pointer)
    EmitDesc emit_desc(const QState &q, const Level *L, uint32_t col_lo, uint32_t col_hi, uint64_t skip, uint64_t take, uint64_t at) const {
        EmitDesc d{};
        if (L) {
            d.uw = L->uw;
            d.ub = L->ub;
            d.out = L->out;
            d.rows = L->rows;
            d.ld = L->ld;
        } else {
            d.ub = universe_of(q);
            d.rows = d.ld = hix.n_words64;
        }
        d.col_lo = col_lo;
        d.col_hi = col_hi;
        d.skip = (uint32_t)skip;
        d.take = (uint32_t)take;
        d.dst = reinterpret_cast<uint32_t *>((uintptr_t)at);
        return d;
    }
    // resolve_maximally_reduced_query_graph (search/new/mod.rs:273-301)
    void start_resolve(QState &q) {
        Level L;
        L.kind = RK_RESOLVE;
        L.graph = q.graph;
        if (tms == B200_TMS_LAST || tms == B200_TMS_FREQUENCY) {
            std::vector<uint16_t> rm;
            for (auto &grp : removal_order(q.ctx, q.graph, tms))
                for (auto nd : grp) rm.push_back(nd);
            remove_nodes_keep_edges(L.graph, rm);
        }
        prepare_resolve(q.ctx, L);
        const ParentRef univ = ParentRef::universe(universe_of(q), hix.n_words64);
        if (q.tree)
            request_node(q, nullptr, std::move(L), univ, 0, {}, nullptr);
        else
            request_activation(q, std::move(L), univ);
    }
    // Frequency (query_graph.rs:303-344): documents of term id t = union of the docids of every node covering t, counted over the
    // whole index — one resolve-shaped activation START -> {covering nodes} -> END per term id
    void start_freq(QState &q, uint32_t t) {
        Level L;
        L.kind = RK_FREQ;
        L.rule_idx = (int)t;
        EGraph &g = L.graph;
        g.nodes.resize(2);
        g.root = 0;
        g.end = 1;
        g.nodes[0].kind = ND_START;
        g.nodes[1].kind = ND_END;
        for (auto &nd : q.graph.nodes)
            if (nd.kind == ND_TERM && nd.term.t0 <= t && t <= nd.term.t1) {
                ENode x;
                x.kind = ND_TERM;
                x.term = nd.term;
                uint16_t id = (uint16_t)g.nodes.size();
                x.pred = {0};
                x.succ = {1};
                g.nodes.push_back(std::move(x));
                sorted_insert(g.nodes[0].succ, id);
                sorted_insert(g.nodes[1].pred, id);
            }
        prepare_resolve(q.ctx, L);
        request_activation(q, std::move(L), ParentRef::universe(dix.base_ub, hix.n_words64));
    }
    void start_query(QState &q) {
        q.rules = rules;
        // tree mode unless a deadline is in force (its polls are defined on the sequential order of bucket requests)
        q.tree = use_tree;
        if (q.neg_only) {
            q.tree = false;
            Level L;
            L.kind = RK_RESOLVE;
            L.neg_only = true;
            ECond x;
            x.rule = RK_RESOLVE;
            L.conds.push_back(x);
            struct AEdge {
                uint32_t src, dst, cost;
                int32_t cond;
            };
            std::vector<AEdge> ae{{0, 1, 0, 0}};  // START -[ignored documents]-> END
            finish_state_graph(L, ae, 0, 1, false);
            L.next_max_cost = 1;
            request_activation(q, std::move(L), ParentRef::universe(universe_of(q), hix.n_words64));
            return;
        }
        if (q.placeholder && !q.sort_rules.empty()) {
            // placeholder search ordered by its sort rules: the window [offset, offset + limit) of the universe in (keys, docid) order,
            // one sort_window_kernel launch after the step loop.  Deadline::exceeded() is polled before the first bucket request
            // (bucket_sort.rs:206-264): when the budget is already spent the universe is returned as it is, Skipped and degraded.
            q.n_candidates = q.univ_count;
            q.cand_src = universe_of(q);
            uint64_t avail = q.univ_count > from ? q.univ_count - from : 0;
            uint32_t take = (uint32_t)std::min<uint64_t>(avail, length);
            if (has_budget && clk::now() >= deadline_at) {
                q.degraded = true;
                q.n_results = take;
                q.scores.assign(take, std::vector<EScore>{EScore{B200_S_SKIPPED, 0, 1, -1.f}});
                if (take) q.emits.push_back(emit_desc(q, nullptr, 0, 0, from, take, 0));
            } else {
                q.n_results = take;
                q.scores.assign(take, {});
                q.sort_pending = take > 0;
                q.sort_lo = from;
                q.sort_hi = from + take;
            }
            q.done = true;
            return;
        }
        if (q.placeholder) {
            // placeholder search: no text rules (search/new/mod.rs:353-416) -> universe in docid order (bucket_sort.rs:104-116)
            q.n_candidates = q.univ_count;
            q.cand_src = universe_of(q);
            uint64_t avail = q.univ_count > from ? q.univ_count - from : 0;
            const uint32_t take = (uint32_t)std::min<uint64_t>(avail, length);
            q.n_results = take;
            q.scores.assign(q.n_results, {});
            if (take) q.emits.push_back(emit_desc(q, nullptr, 0, 0, from, take, 0));
            q.done = true;
            return;
        }
        if (tms == B200_TMS_FREQUENCY) {
            q.n_term_ids = 0;
            for (auto &nd : q.graph.nodes)
                if (nd.kind == ND_TERM) q.n_term_ids = std::max<uint32_t>(q.n_term_ids, (uint32_t)nd.term.t1 + 1);
            q.term_freq.clear();
            if (q.n_term_ids > 0) {
                start_freq(q, 0);
                return;
            }
        }
        start_resolve(q);
    }
    void start_range(uint32_t lo, uint32_t hi) {
        auto t_ph = clk::now();
        pfor(hi - lo, [&](size_t i) {
            QState &q = *qs[lo + i];
            if (q.done) return;
            try {
                start_query(q);
            } catch (const TooComplex &t) {
                q.status = B200_ERR_CAPACITY;
                q.error = t.why;
                q.done = true;
            }
        });
        stats.host_ms[5] += ms_since(t_ph);
    }
    // S1: one ranking rule over the caller's universe and query graph (RankingRule::start_iteration); collect_rule_buckets() takes
    // its result
    void start_rule(QState &q, int kind) {
        auto t_ph = clk::now();
        try {
            Pending *pd = request_activation(q, rule_level(q.ctx, 0, kind, q.graph, false), ParentRef::universe(universe_of(q), hix.n_words64));
            pd->need = 0xffffffffu;  // every bucket may be asked for: walk them all
        } catch (const TooComplex &t) {
            q.status = B200_ERR_CAPACITY;
            q.error = t.why;
            q.done = true;
        }
        stats.host_ms[5] += ms_since(t_ph);
    }
    // S1: hand every bucket of the rule back (RankingRule::next_bucket serves them one by one): rank, documents, child graph
    void collect_rule_buckets(QState &q) {
        Level &L = q.levels.back();
        const uint64_t W = hix.n_words64;
        for (size_t ci = 0; ci < L.cost_vals.size(); ci++) {
            RuleBucket bk;
            bk.rank = (uint32_t)(L.next_max_cost - L.cost_vals[ci]);
            bk.max_rank = (uint32_t)L.next_max_cost;
            bk.count = L.counts[ci];
            bk.bitmap.assign(W, 0);
            if (bk.count) {
                // the activation ran on the dense universe (row j = word j): bucket column ci is a dense bitmap
                cudaMemcpy(bk.bitmap.data(), L.out + (size_t)ci * L.ld, W * 8, cudaMemcpyDeviceToHost);
                bk.child = new GraphObj(q.ctx, child_graph(L, ci));
            }
            rule_buckets->push_back(std::move(bk));
        }
        q.drop_levels();
        q.done = true;
    }
    // advance one query's bucket sort until it needs the device again (bucket_sort.rs:193-330)
    void emit_bucket(QState &q, Level &L, uint32_t col_lo, uint32_t col_hi, uint64_t count) {
        if (count == 0) return;
        uint64_t skip = 0;
        uint64_t take = 0;
        if (q.cur_offset < from) {
            if (q.cur_offset + count >= from) {
                skip = from - q.cur_offset;
                take = std::min<uint64_t>(count - skip, length - q.n_results);
            }
        } else
            take = std::min<uint64_t>(count, length - q.n_results);
        if (take) {
            q.emits.push_back(emit_desc(q, &L, col_lo, col_hi, skip, take, q.n_results));
            for (uint64_t k = 0; k < take; k++) q.scores.push_back(q.rr_scores);  // bucket_sort.rs:447-455 records them under either strategy
            q.n_results += (uint32_t)take;
        }
        q.cur_offset += count;
    }
    void advance(QState &q) {
        const size_t n_rules = q.rules.size();
        for (;;) {
            if (q.levels.empty()) break;
            // bucket_sort.rs:52-64,104-116: all_candidates is the universe even when no hit is asked for (limit 0)
            if (q.levels.back().kind == RK_RESOLVE && q.levels.back().cursor == 0)
                q.n_candidates = q.levels.back().neg_only ? q.levels.back().counts.back() : q.levels.back().counts[0];
            if (q.n_results >= length) break;
            size_t cur = q.levels.size() - 1;  // level index; rule index = cur - 1 (level 0 = resolve)
            Level &L = q.levels[cur];
            auto back = [&]() {
                q.pop_level();
                if (!q.levels.empty() && q.levels.size() - 1 >= 1) {
                    size_t rule_cur = q.levels.size() - 2;
                    if (q.rr_scores.size() > rule_cur) q.rr_scores.pop_back();
                } else if (q.levels.size() == 1)
                    q.rr_scores.clear();
            };
            if (L.kind == RK_FREQ) {
                const uint32_t t = (uint32_t)L.rule_idx;
                q.term_freq.push_back(L.counts.empty() ? 0 : L.counts[0]);
                q.drop_levels();
                if (t + 1 < q.n_term_ids) {
                    start_freq(q, t + 1);
                    return;
                }
                // weights: most frequent term first (ties share a weight); a term matching nothing counts as the most frequent
                std::vector<std::pair<uint8_t, uint64_t>> twf;
                for (uint32_t i = 0; i < q.n_term_ids; i++) twf.push_back({(uint8_t)i, q.term_freq[i] == 0 ? UINT64_MAX : q.term_freq[i]});
                std::stable_sort(twf.begin(), twf.end(), [](const auto &a, const auto &b2) { return a.second > b2.second; });
                q.ctx.freq_weight.assign(q.n_term_ids, 1);
                uint16_t weight = 1;
                for (size_t i = 0; i < twf.size(); i++) {
                    q.ctx.freq_weight[twf[i].first] = weight;
                    if (i + 1 < twf.size() && twf[i].second != twf[i + 1].second) weight++;
                }
                start_resolve(q);
                return;
            }
            if (L.kind == RK_RESOLVE) {
                // the resolve level is not a ranking rule: after it, start rule 0 on its bucket 0
                if (L.cursor > 0) {
                    q.drop_levels();
                    break;
                }
                L.cursor = 1;
                if (L.neg_only) {
                    // placeholder search over universe - ignored documents = the level's unmatched column (the one after its
                    // single bucket), in docid order (bucket_sort.rs:104-116)
                    const uint64_t rest = L.counts.back();
                    const uint32_t rest_col = (uint32_t)L.cost_vals.size();
                    q.n_candidates = rest;
                    q.cand_src = L.out + (size_t)rest_col * L.ld;
                    if (rest >= from) emit_bucket(q, L, rest_col, rest_col + 1, rest);
                    q.drop_levels();
                    break;
                }
                q.n_candidates = L.counts[0];
                q.cand_src = L.out;  // bucket 0 of the resolve level over the dense universe = SearchResult::candidates
                uint64_t cnt = L.counts[0];
                if (cnt < from) {  // bucket_sort.rs:52-64
                    q.drop_levels();
                    break;
                }
                if (n_rules == 0) {
                    emit_bucket(q, L, 0, 1, cnt);
                    q.drop_levels();
                    break;
                }
                request_activation(q, rule_level(q.ctx, 0, q.rules[0], q.graph, n_rules == 1), ParentRef::bucket(L, 0, cnt));
                return;
            }
            size_t rule_cur = (size_t)L.rule_idx;
            if (L.universe_count == 0 || (skip_scoring && L.universe_count == 1)) {
                if (L.universe_count == 1) emit_bucket(q, L, (uint32_t)L.cursor, (uint32_t)L.cost_vals.size() + 1, 1);
                back();
                continue;
            }
            // Deadline::exceeded() is polled once per bucket request (bucket_sort.rs:206); no graph rule can answer without blocking
            // (ranking_rules.rs:67-74), so on expiry every rule's remaining universe is returned as it is with a Skipped score,
            // from the current rule up to the first one, and the result is degraded (bucket_sort.rs:206-264)
            if (stop_after >= 0 ? q.polls++ >= stop_after : (has_budget && clk::now() > deadline_at)) {
                for (;;) {
                    Level &Lc = q.levels.back();
                    const uint64_t remaining = Lc.universe_count;
                    q.rr_scores.push_back(EScore{B200_S_SKIPPED, 0, 1, -1.f});
                    if (has_thr && global_score_of(q.rr_scores) < thr)
                        q.n_candidates -= std::min<uint64_t>(q.n_candidates, remaining);
                    else
                        emit_bucket(q, Lc, (uint32_t)Lc.cursor, (uint32_t)Lc.cost_vals.size() + 1, remaining);
                    q.rr_scores.pop_back();
                    if (Lc.rule_idx == 0) break;
                    back();
                }
                q.degraded = true;
                q.drop_levels();
                break;
            }
            // one bucket request = one cost of the rule, empty or not (graph_based_ranking_rule.rs:231-236 walks all_costs): an empty
            // bucket changes nothing but it does consume a deadline poll
            size_t ci = L.cursor;
            if (ci >= L.cost_vals.size()) {
                back();
                continue;
            }
            L.cursor = ci + 1;
            uint64_t cnt = L.counts[ci];
            if (cnt == 0) continue;
            EScore sc{score_kind_of(L.kind), (uint32_t)(L.next_max_cost - L.cost_vals[ci]), (uint32_t)L.next_max_cost, -1.f};
            q.rr_scores.push_back(sc);
            L.universe_count -= cnt;
            // bucket_sort.rs:293-296: a bucket whose score so far is below the threshold leaves the candidates together with
            // everything the rule has not returned yet (every later bucket of the rule scores lower still)
            const bool below = has_thr && global_score_of(q.rr_scores) < thr;
            if (rule_cur == n_rules - 1 || (skip_scoring && cnt <= 1) || q.cur_offset + cnt < from || below) {
                if (below) {
                    if (!L.below_done) q.n_candidates -= std::min<uint64_t>(q.n_candidates, cnt + L.universe_count);
                    L.below_done = true;
                } else
                    emit_bucket(q, L, (uint32_t)ci, (uint32_t)ci + 1, cnt);
                q.rr_scores.pop_back();
                continue;
            }
            // descend: the next rule iterates on this bucket with the query graph of the paths that produced it
            if (L.kind != RK_EXACT_ATTRIBUTE && ci > L.walked_m) {  // cannot happen: buckets 0..walked_m hold every document the query still needed
                q.status = B200_ERR_STATE;
                q.error = "internal: descent into a bucket whose surviving paths were not computed";
                q.drop_levels();
                q.done = true;
                return;
            }
            request_activation(q, rule_level(q.ctx, (int)rule_cur + 1, q.rules[rule_cur + 1], child_graph(L, ci), rule_cur + 2 == n_rules),
                               ParentRef::bucket(L, (uint32_t)ci, cnt));
            return;
        }
        q.drop_levels();
        q.done = true;
    }

    // tree mode: the documents of bucket [col_lo, col_hi) stand at [off, off + cnt) in the query's result order; write the part inside
    // the window [from, from + length) to its final place
    void emit_window(QState &q, Level &L, uint32_t col_lo, uint32_t col_hi, uint64_t cnt, uint64_t off, const std::vector<EScore> &sc, ActOut &out) {
        const uint64_t win_end = (uint64_t)from + length;
        const uint64_t skip = off < from ? from - off : 0;
        if (skip >= cnt) return;
        const uint64_t start = std::max<uint64_t>(off, from);
        if (start >= win_end) return;
        const uint64_t take = std::min<uint64_t>(cnt - skip, win_end - start);
        out.emits.push_back(emit_desc(q, &L, col_lo, col_hi, skip, take, start - from));
        const size_t at = (size_t)(start - from);  // q.scores was sized when the universe was resolved; windows of different buckets are disjoint
        for (uint64_t k = 0; k < take; k++) q.scores[at + k] = sc;
        out.n_results += (uint32_t)take;
    }
    static void release_node(Node *n, ActOut &out) {
        Level &L = n->L;
        if (L.a_off != SIZE_MAX) out.freed.emplace_back(L.a_off, L.a_len);
        L.a_off = SIZE_MAX;
        // the host side of the level is not needed any more either
        L.graph = EGraph();
        std::vector<ECond>().swap(L.conds);
        std::vector<SEdge>().swap(L.sedges);
        std::vector<SurvPath>().swap(L.surv);
    }
    // tree mode: the activation of node N is complete — place or descend into every bucket of it that reaches the result window
    // (the same decisions as advance(), bucket_sort.rs:193-330, taken for all buckets at once)
    void expand(QState &q, Node *N, ActOut &out) {
        Level &L = N->L;
        // the parent was expanded in an earlier step (self_done); the last of its children to complete gives its buckets back
        if (N->parent && N->parent->live_children.fetch_sub(1) == 1) release_node(N->parent, out);
        const size_t n_rules = q.rules.size();
        const uint64_t win_end = (uint64_t)from + length;
        uint64_t off = N->off0;
        if (L.kind == RK_RESOLVE) {
            const uint64_t cnt = L.counts[0];
            q.n_candidates = cnt;
            q.cand_src = L.out;
            if (length != 0 && cnt >= from) {  // bucket_sort.rs:52-64
                q.scores.resize((size_t)std::min<uint64_t>(length, cnt - from));
                if (n_rules == 0)
                    emit_window(q, L, 0, 1, cnt, 0, {}, out);
                else
                    request_node(q, N, rule_level(q.ctx, 0, q.rules[0], q.graph, n_rules == 1), ParentRef::bucket(L, 0, cnt), 0, {}, &out);
            }
        } else {
            const size_t rule_cur = (size_t)L.rule_idx;
            uint64_t remaining = L.universe_count;
            std::vector<EScore> sc = N->scores;
            for (size_t ci = 0; off < win_end; ci++) {
                if (remaining == 0 || (skip_scoring && remaining == 1)) {
                    if (remaining == 1) emit_window(q, L, (uint32_t)ci, (uint32_t)L.cost_vals.size() + 1, 1, off, N->scores, out);
                    break;
                }
                if (ci >= L.cost_vals.size()) break;
                const uint64_t cnt = L.counts[ci];
                if (cnt == 0) continue;
                remaining -= cnt;
                sc.push_back(EScore{score_kind_of(L.kind), (uint32_t)(L.next_max_cost - L.cost_vals[ci]), (uint32_t)L.next_max_cost, -1.f});
                if (rule_cur == n_rules - 1 || (skip_scoring && cnt <= 1) || off + cnt <= from)
                    emit_window(q, L, (uint32_t)ci, (uint32_t)ci + 1, cnt, off, sc, out);
                else {
                    if (L.kind != RK_EXACT_ATTRIBUTE && ci > L.walked_m) {  // cannot happen: buckets 0..walked_m hold every document this level still needed
                        out.status = B200_ERR_STATE;
                        out.error = "internal: descent into a bucket whose surviving paths were not computed";
                        return;
                    }
                    request_node(q, N, rule_level(q.ctx, (int)rule_cur + 1, q.rules[rule_cur + 1], child_graph(L, ci), rule_cur + 2 == n_rules),
                                 ParentRef::bucket(L, (uint32_t)ci, cnt), off, sc, &out);
                }
                sc.pop_back();
                off += cnt;
            }
        }
        N->self_done = true;
        if (N->live_children.load() == 0) release_node(N, out);  // no child: nothing will read these buckets after the emissions queued above
        out.expanded = true;
    }
    // a query that cannot go on: give everything it holds back
    static void abandon(QState &q) {
        q.pendings.clear();
        q.emits.clear();
        q.drop_levels();
        for (auto &n : q.nodes) q.release_level(n->L);
        q.nodes.clear();
        q.outstanding = 0;
        q.done = true;
    }

    // ---- phase 4: step loop.  The batch is split over lanes; every lane has its own stream, device buffers, arena slice, host
    // driver thread and worker sub-pool, so the host phases of one lane overlap both the kernels and the host phases of the others.
    // Drivers are host threads; each alternates between its lanes (software pipeline: while one lane's kernels run, the driver packs
    // and advances its other lane), and the drivers run concurrently.
    int setup_lanes() {
        CU(eng.d_docids_out.reserve((size_t)NQ * std::max(1u, length)), "alloc results");
        n_drivers = NQ >= 512 ? 4 : (NQ >= 64 ? 2 : 1);
        if (const char *env = getenv("B200_DRIVERS")) n_drivers = (unsigned)std::max(1, std::min((int)Engine::MAX_DRIVERS, atoi(env)));
        if (const char *env = getenv("B200_LANES_PER_DRIVER")) lanes_per_driver = (unsigned)std::max(1, atoi(env));
        if (getenv("B200_SINGLE_LANE")) n_drivers = lanes_per_driver = 1;
        // every lane that is given queries belongs to a driver: drive() and drive_waves() run lanes [0, n_drivers * lanes_per_driver)
        lanes_per_driver = std::min(lanes_per_driver, Engine::MAX_LANES / n_drivers);
        n_lanes = n_drivers * lanes_per_driver;
        if (NQ < n_lanes) n_lanes = n_drivers = lanes_per_driver = 1;
        {
            unsigned per_driver = std::max(1u, host_threads() / n_drivers);
            for (unsigned dr = 0; dr < n_drivers; dr++) {
                auto &dp = eng.driver_pools[dr];
                if (!dp || dp->threads.size() + 1 != per_driver) dp.reset(new WorkerPool(per_driver - 1));
                for (unsigned k = 0; k < lanes_per_driver; k++) lanes[dr * lanes_per_driver + k].pool = dp.get();
            }
        }
        for (unsigned l = 0; l < n_lanes; l++) {
            Lane &ln = lanes[l];
            if (!ln.stream) {
                CU(cudaStreamCreateWithFlags(&ln.stream, cudaStreamNonBlocking), "lane stream");
                CU(cudaEventCreate(&ln.e0), "lane event");
                CU(cudaEventCreate(&ln.e1), "lane event");
                CU(cudaEventCreateWithFlags(&ln.ev_fork, cudaEventDisableTiming), "lane event");
                for (uint32_t c = 1; c <= EVAL_CLASSES; c++) {
                    CU(cudaStreamCreateWithFlags(&ln.cls_stream[c], cudaStreamNonBlocking), "class stream");
                    CU(cudaEventCreateWithFlags(&ln.ev_join[c], cudaEventDisableTiming), "lane event");
                }
            }
            ln.scratch = eng.scratch + (((eng.scratch_bytes / n_lanes) * l) & ~(size_t)255);
            ln.scratch_bytes = (eng.scratch_bytes / n_lanes) & ~(size_t)255;
            ln.arena = eng.arena + (((eng.arena_bytes / n_lanes) * l) & ~(size_t)255);
            ln.arena_bytes = (eng.arena_bytes / n_lanes) & ~(size_t)255;
            ln.alloc.reset(ln.arena_bytes);
            ln.timing = !(getenv("B200_KERNEL_TIMERS") && atoi(getenv("B200_KERNEL_TIMERS")) == 0);
            ln.lst = b200_stats{};
            ln.rc = 0;
            ln.error.clear();
            ln.members.clear();
            ln.inflight = false;
        }
        for (unsigned l = 0; l < n_lanes; l++)
            for (uint32_t i = lane_lo(l); i < lane_lo(l + 1); i++) lanes[l].members.push_back(i);
        // row lookup tables (scatter_kernel): NQ slots of n_words64 entries, zeroed once per batch.  A lane owns the slots of its query
        // range and lends each to at most one activation per step; entries carry the tag of the use that wrote them (12 bits, so a slot
        // serves 4094 steps), which makes the leftovers of earlier uses read as misses.  Activations without a slot search their rows.
        use_rowtab = hix.n_words64 <= (1u << 20) && !getenv("B200_NO_ROWTAB");
        if (use_rowtab) {
            CU(eng.d_rowtab.reserve((size_t)NQ * hix.n_words64), "row lookup tables");
            CU(cudaMemsetAsync(eng.d_rowtab.p, 0, (size_t)NQ * hix.n_words64 * 4, eng.stream), "zero row lookup tables");
        }
        slot_tag.assign(NQ, 0);
        lane_acts.resize(n_lanes);
        return B200_OK;
    }
    int lane_fail(Lane &ln, int code, const char *msg) {
        ln.error = msg;
        return fail(code, msg);
    }

    // pack the pending work of a lane and enqueue it (no synchronisation). returns <0 on error, 0 idle, 1 launched
    int launch(Lane &ln) {
        auto t_pack = clk::now();
        Step s;
        int rc = schedule(ln, s);
        if (rc <= 0) return rc;
        if ((rc = pack(ln, s)) < 0) return rc;
        if ((rc = enqueue(ln, s)) < 0) return rc;
        ln.lst.host_ms[3] += ms_since(t_pack);
        return 1;
    }
    // pass 1 (serial, light): which pending activations join the lane's step; their sizes, offsets and device memory.  Returns <0 on
    // error, 0 when the lane has nothing to do, 1 otherwise.
    int schedule(Lane &ln, Step &s) {
        ln.act_q.clear();
        const unsigned li = (unsigned)(&ln - lanes);
        std::vector<std::unique_ptr<Pending>> &acts = lane_acts[li];
        acts.clear();
        std::vector<Cand> &cand_q = s.cand_q;
        for (auto i : ln.members) {
            QState &q = *qs[i];
            for (auto &f : q.freed) ln.alloc.give(f.first, f.second);  // levels left since the lane's previous step
            q.freed.clear();
            for (auto &pd : q.pendings) cand_q.push_back(Cand{i, pd.get()});
            if (!q.emits.empty()) s.emit_q.push_back(i);
        }
        if (r->candidates || facets || fsearch) {
            // SearchResult::candidates, copied and counted for the facets before any block freed above can be written again
            std::vector<Engine::FacetJob> fjobs;
            for (auto i : ln.members) {
                QState &q = *qs[i];
                if (!q.cand_src) continue;
                if (r->candidates) {
                    CU(cudaMemcpyAsync(r->candidates + (size_t)i * r->candidates_words, q.cand_src, (size_t)hix.n_words64 * 8, cudaMemcpyDeviceToHost,
                                       ln.stream),
                       "D2H candidates");
                    ln.lst.d2h_bytes += (size_t)hix.n_words64 * 8;
                }
                if (fsearch && eng.fs_slot[i] >= 0) {
                    CU(cudaMemcpyAsync(eng.d_fs_qcand.p + (size_t)eng.fs_slot[i] * hix.n_words64, q.cand_src, (size_t)hix.n_words64 * 8,
                                       cudaMemcpyDeviceToDevice, ln.stream),
                       "D2D facet search candidates");
                }
                if (facets && q.status == 0)
                    for (uint32_t k = b->facet_begin[i]; k < b->facet_begin[i + 1]; k++) fjobs.push_back(Engine::FacetJob{q.cand_src, b->facet_fid[k], k});
                q.cand_src = nullptr;
            }
            if (!fjobs.empty()) {
                const int rc = eng.facet_enqueue(&ln, fjobs, fout, b->facet_max_values, ln.d_facet, ln.d_facet_slots);
                if (rc != B200_OK) return rc;
            }
        }
        // longest first: the parallel-for over these queries ends when its slowest query does, and host time per query grows
        // with the size of its query graph
        std::stable_sort(cand_q.begin(), cand_q.end(), [&](const Cand &x, const Cand &y) { return x.pd->L->graph.nodes.size() > y.pd->L->graph.nodes.size(); });
        if (cand_q.empty() && s.emit_q.empty()) return 0;
        s.plan.reserve(cand_q.size());
        // An activation joins the step when its per-step scratch (condition matrix, DP table, path table) and its persistent block
        // (universe rows + bucket columns) fit; otherwise it waits for a later step of the lane (scratch is reused every step, the
        // arena is refilled as queries leave levels).  New queries (first activation) are only admitted while the arena is less
        // than ~60 % full, so that the queries already descending can finish.  When nothing at all fits and the lane is idle, the
        // waiting query with the largest demand fails alone with B200_ERR_CAPACITY and the others go on.
        bool admit_all = false;
        uint32_t next_slot = lane_lo(li);
        const uint32_t slot_end = lane_lo(li + 1);
        for (;;) {
            for (size_t ci = 0; ci < cand_q.size(); ci++) {
                Pending &pd = *cand_q[ci].pd;
                StepOut &o = pd.o;
                Plan pl{};
                pl.jobs = s.n_jobs;
                pl.sets = s.n_sets;
                pl.words = s.n_words;
                pl.colprog = s.n_colprog;
                pl.states = s.n_states;
                pl.edges = s.n_edges;
                pl.costs = s.n_costs_tot;
                pl.prog = s.n_prog;
                pl.probes = s.n_probes;
                pl.res_off = s.res_words;
                uint32_t ld = std::max(1u, pd.parent.cap);
                pl.ld = ld;
                pl.identity = !pd.parent.uw && !pd.parent.out;  // first activation of a query: the universe is the dense documents bitmap itself
                uint32_t n_cols = std::max(1u, o.n_cols);
                uint32_t tab_size = o.want_paths ? 4096u << pd.tab_shift : 1;
                pl.tab_size = tab_size;
                pl.cls = eval_class(n_cols + o.n_pairs + EVAL_EXTRA_SLOTS);
                pl.rpt = 1;  // rows per thread: > 1 only pays for grids far larger than the GPU (it lengthens the tail of small grids); measured
                             // at 10 M documents: 4 rows per thread on the >= 65536-row activations of the smallest class saves 15 % of the pass
                if (eval_rpt_big > 1 && pl.cls == 0 && ld >= 65536) pl.rpt = eval_rpt_big;
                const uint32_t my_tiles = (ld + 128 * pl.rpt - 1) / (128 * pl.rpt);
                size_t persist = pl.identity ? (size_t)ld * 8 * (o.n_costs + 1) : (size_t)ld * 4 + 256 + (size_t)ld * 8 + 256 + (size_t)ld * 8 * (o.n_costs + 1);
                size_t cbytes = (size_t)ld * 8 * n_cols, sbytes = pl.cls < EVAL_CLASSES ? 0 : (size_t)ld * 8 * o.n_pairs, tbytes = (size_t)tab_size * 8;
                // zeroed zone (condition matrix + path table) grows from the front of the lane's scratch, the DP table from the back
                pl.coff = (s.z_used + 255) & ~(size_t)255;
                pl.toff = (pl.coff + cbytes + 255) & ~(size_t)255;
                size_t s_need = (sbytes + 255) & ~(size_t)255;
                pd.demand = persist + cbytes + tbytes + s_need;
                if (pl.toff + tbytes + s_need + s.s_used > ln.scratch_bytes) continue;               // next step
                if (pl.identity && !admit_all && ln.alloc.used * 5 > ln.alloc.total * 3) continue;  // admission
                size_t aoff = ln.alloc.take(persist);
                if (aoff == SIZE_MAX) continue;
                pl.pb = ln.arena + aoff;
                pd.L->a_off = aoff;
                pd.L->a_len = persist;
                pl.rt_slot = UINT32_MAX;
                if (use_rowtab && !pl.identity && ld >= rowtab_min_rows) {
                    while (next_slot < slot_end && slot_tag[next_slot] >= 4094) next_slot++;
                    if (next_slot < slot_end) {
                        pl.rt_slot = next_slot;
                        pl.rt_tag = ++slot_tag[next_slot];
                        next_slot++;
                    }
                }
                s.n_jobs += (uint32_t)o.jobs.size();
                s.n_sets += (uint32_t)o.pairsets.size();
                s.n_words += (uint32_t)o.words.size();
                s.n_colprog += (uint32_t)o.colprog.size();
                s.n_states += (uint32_t)o.dp_states.size();
                s.n_edges += (uint32_t)o.dp_edges.size();
                s.n_costs_tot += (uint32_t)o.cost_vals.size();
                s.n_prog += (uint32_t)o.prog.size();
                s.want_paths_cls[pl.cls] = s.want_paths_cls[pl.cls] || o.want_paths;
                pl.tiles = s.n_tiles_cls[pl.cls];  // within its class; the class bases are added below
                s.n_tiles_cls[pl.cls] += my_tiles;
                s.n_tiles += my_tiles;
                for (auto &ps : o.pairsets) s.n_probes += ps.n_left * ps.n_right;
                s.res_words += 4 + o.n_costs;  // rows | n_costs + 1 bucket counts | path-table saturation flag | last walked bucket
                pl.n_seg = pl.identity ? 1u : std::max(1u, (pd.parent.rows + COMPACT_SEG - 1) / COMPACT_SEG);
                pl.ctiles = s.n_ctiles;
                s.n_ctiles += pl.n_seg;
                s.multi_segment = s.multi_segment || pl.n_seg > 1;
                s.z_used = pl.toff + tbytes;
                s.s_used += s_need;
                pl.soff_from_end = s.s_used;
                ln.act_q.push_back(cand_q[ci].qi);
                s.sched.push_back(ci);
                ln.lst.posting_bytes += o.posting_bytes;
                // algorithmic bytes of the evaluation: condition columns in, universe word in, bucket columns out (the DP table is on-chip)
                uint64_t mb = (uint64_t)ld * 8 * (n_cols + o.n_costs + 2);
                ln.lst.matrix_bytes += mb;
                s.eval_bytes += mb;
                if (!pl.identity) s.compact_bytes += (uint64_t)pd.parent.rows * 8 + (uint64_t)ld * 12;
                s.fill_bytes += o.posting_bytes;
                if (work_hist) {  // B200_WORK_HIST=1: where the step's work comes from (developer statistics, see tools/)
                    const int kind = pd.L->kind;
                    const int ub = ld >= 65536 ? 3 : (ld >= 4096 ? 2 : (ld >= 128 ? 1 : 0));
                    std::lock_guard<std::mutex> g(work_hist->mu);
                    for (auto &jb : o.jobs) {
                        if (jb.chunk) continue;
                        const ListRef &lr = hix.lists[jb.list];
                        int cb = 0;
                        while ((1u << cb) < lr.card && cb < 31) cb++;
                        auto &cell = work_hist->lists[ub][lr.dense ? 32 : cb];
                        cell[0]++;
                        cell[1] += lr.dense ? (uint64_t)hix.n_words64 * 8 : (uint64_t)lr.card * 4;
                    }
                    auto &ev = work_hist->eval[kind][ub];
                    ev[0]++;
                    ev[1] += ld;
                    ev[2] += (uint64_t)ld * o.prog.size();
                    ev[3] += (uint64_t)ld * n_cols;
                    for (auto &ps : o.pairsets) work_hist->probes[ub] += (uint64_t)ps.n_left * ps.n_right;
                }
                s.plan.push_back(pl);
            }
            if (!ln.act_q.empty() || !s.emit_q.empty()) break;
            // the lane is idle (launch is only called between its steps) and nothing fits; nothing was scheduled, so the pass
            // starts over from the same state
            if (!admit_all) {
                admit_all = true;
                continue;
            }
            size_t worst = 0;
            for (size_t k = 1; k < cand_q.size(); k++)
                if (cand_q[k].pd->demand > cand_q[worst].pd->demand) worst = k;
            const uint32_t wq = cand_q[worst].qi;
            QState &q = *qs[wq];
            q.status = B200_ERR_CAPACITY;
            q.error = "a single ranking-rule step of this query needs more device memory than the lane owns (B200_ARENA_MB / B200_SCRATCH_MB)";
            cand_q.erase(std::remove_if(cand_q.begin(), cand_q.end(), [&](const Cand &c) { return c.qi == wq; }), cand_q.end());
            abandon(q);
            for (auto &f : q.freed) ln.alloc.give(f.first, f.second);
            q.freed.clear();
            ln.lst.deferred++;
            if (cand_q.empty()) return 0;
            admit_all = false;
        }
        ln.lst.deferred += cand_q.size() - ln.act_q.size();
        // the scheduled activations leave their queries' pending lists for the lane's step
        for (auto ci : s.sched) {
            QState &q = *qs[cand_q[ci].qi];
            for (auto &up : q.pendings)
                if (up.get() == cand_q[ci].pd) {
                    acts.push_back(std::move(up));
                    break;
                }
        }
        for (auto ci : s.sched) {
            auto &pv = qs[cand_q[ci].qi]->pendings;
            pv.erase(std::remove(pv.begin(), pv.end(), nullptr), pv.end());
        }
        for (uint32_t c = 0; c <= EVAL_CLASSES; c++) s.tile_base[c + 1] = s.tile_base[c] + s.n_tiles_cls[c];
        for (auto &pl : s.plan) pl.tiles += s.tile_base[pl.cls];
        return 1;
    }
    // pass 2 (parallel): the step blob, written straight into the lane's pinned buffer
    int pack(Lane &ln, Step &s) {
        ln.lst.device_steps++;
        const std::vector<std::unique_ptr<Pending>> &acts = lane_acts[(unsigned)(&ln - lanes)];
        const size_t NA = ln.act_q.size();
        for (auto qi : s.emit_q) s.n_emits += (uint32_t)qs[qi]->emits.size();
        // section offsets inside the step blob
        size_t off = 0;
        auto section = [&](size_t bytes) {
            size_t o0 = (off + 15) & ~(size_t)15;
            off = o0 + bytes;
            return o0;
        };
        s.o_acts = section(NA * sizeof(ActDesc));
        s.o_sets = section((size_t)s.n_sets * sizeof(PairSet));
        s.o_words = section((size_t)s.n_words * 4);
        s.o_colprog = section((size_t)s.n_colprog * sizeof(ColOp));
        s.o_states = section((size_t)s.n_states * sizeof(DpState));
        s.o_edges = section((size_t)s.n_edges * sizeof(DpEdge));
        s.o_costs = section((size_t)s.n_costs_tot * 2);
        s.o_prog = section((size_t)s.n_prog * 4);
        s.o_tiles = section((size_t)s.n_tiles * sizeof(TileDesc));
        s.o_ctiles = section((size_t)s.n_ctiles * sizeof(CompactTile));
        s.o_emits = section((size_t)s.n_emits * sizeof(EmitDesc));
        s.o_jobs = section((size_t)s.n_jobs * sizeof(Job));
        s.o_nstatic = section(16);
        s.nbytes = off + 16;
        if (s.nbytes > ln.h_step_cap) {
            if (ln.h_step) cudaFreeHost(ln.h_step);
            ln.h_step_cap = s.nbytes * 2;
            CU(cudaMallocHost((void **)&ln.h_step, ln.h_step_cap), "pinned step buffer");
        }
        uint8_t *hb = ln.h_step;
        ln.pool->run(NA, [&](size_t a) {
            Pending &pd = *acts[a];
            Level &L = *pd.L;
            StepOut &o = pd.o;
            const Plan &pl = s.plan[a];
            ActDesc d;
            memset(&d, 0, sizeof d);
            d.p_uw = pd.parent.uw;
            d.p_ub = pd.parent.ub;
            d.p_out = pd.parent.out;
            d.p_rows = pd.parent.rows;
            d.p_ld = pd.parent.ld;
            d.p_col_lo = pd.parent.col;
            d.p_col_hi = pd.parent.col + 1;
            uint32_t ld = pl.ld;
            d.ld = ld;
            d.n_cols = std::max(1u, o.n_cols);
            d.n_costs = o.n_costs;
            d.n_states = (uint32_t)o.dp_states.size();
            d.want_paths = o.want_paths;
            d.tab_size = pl.tab_size;
            d.all_conditional = o.all_conditional;
            d.S = reinterpret_cast<unsigned long long *>(ln.scratch + ln.scratch_bytes - pl.soff_from_end);
            d.tab = reinterpret_cast<unsigned long long *>(ln.scratch + pl.toff);
            d.C = reinterpret_cast<unsigned long long *>(ln.scratch + pl.coff);
            if (pl.identity) {
                d.uw = nullptr;
                d.ub = const_cast<unsigned long long *>(pd.parent.ub);
                d.out = reinterpret_cast<unsigned long long *>(pl.pb);
            } else {
                d.uw = reinterpret_cast<uint32_t *>(pl.pb);
                d.ub = reinterpret_cast<unsigned long long *>(pl.pb + (((size_t)ld * 4 + 255) & ~(size_t)255));
                d.out = d.ub + (((size_t)ld + 31) & ~(size_t)31);
            }
            d.row_tab = nullptr;
            d.row_tag = 0;
            if (pl.rt_slot != UINT32_MAX) {
                d.row_tag = pl.rt_tag;
                d.row_tab = eng.d_rowtab.p + (size_t)pl.rt_slot * hix.n_words64;
            }
            L.uw = d.uw;
            L.ub = d.ub;
            L.out = d.out;
            L.ld = ld;
            d.colprog_off = pl.colprog;
            d.colprog_len = (uint32_t)o.colprog.size();
            d.state_off = pl.states;
            d.edge_off = pl.edges;
            d.cost_off = pl.costs;
            d.prog_off = pl.prog;
            d.prog_len = (uint32_t)o.prog.size();
            d.n_pairs = o.n_pairs;
            d.need = pd.need;
            d.root_rmin = o.dp_states.empty() ? 0 : o.dp_states[0].rmin;
            d.root_rcount = o.dp_states.empty() ? 0 : o.dp_states[0].rcount;
            if (!o.prog.empty()) memcpy(hb + s.o_prog + (size_t)pl.prog * 4, o.prog.data(), o.prog.size() * 4);
            d.res_off = pl.res_off;
            L.res_off = pl.res_off;
            memcpy(hb + s.o_acts + a * sizeof(ActDesc), &d, sizeof d);
            if (!o.colprog.empty()) memcpy(hb + s.o_colprog + (size_t)pl.colprog * sizeof(ColOp), o.colprog.data(), o.colprog.size() * sizeof(ColOp));
            if (!o.dp_states.empty()) memcpy(hb + s.o_states + (size_t)pl.states * sizeof(DpState), o.dp_states.data(), o.dp_states.size() * sizeof(DpState));
            if (!o.dp_edges.empty()) memcpy(hb + s.o_edges + (size_t)pl.edges * sizeof(DpEdge), o.dp_edges.data(), o.dp_edges.size() * sizeof(DpEdge));
            if (!o.cost_vals.empty()) memcpy(hb + s.o_costs + (size_t)pl.costs * 2, o.cost_vals.data(), o.cost_vals.size() * 2);
            if (!o.words.empty()) memcpy(hb + s.o_words + (size_t)pl.words * 4, o.words.data(), o.words.size() * 4);
            Job *jd = reinterpret_cast<Job *>(hb + s.o_jobs) + pl.jobs;
            for (size_t k = 0; k < o.jobs.size(); k++) {
                jd[k] = o.jobs[k];
                jd[k].act = (uint32_t)a;
            }
            PairSet *sd = reinterpret_cast<PairSet *>(hb + s.o_sets) + pl.sets;
            uint32_t pb = pl.probes;
            for (size_t k = 0; k < o.pairsets.size(); k++) {
                sd[k] = o.pairsets[k];
                sd[k].act = (uint32_t)a;
                sd[k].left_off += pl.words;
                sd[k].right_off += pl.words;
                sd[k].probe_base = pb;
                pb += sd[k].n_left * sd[k].n_right;
            }
            TileDesc *td = reinterpret_cast<TileDesc *>(hb + s.o_tiles) + pl.tiles;
            for (uint32_t r0 = 0, k = 0; r0 < ld; r0 += 128 * pl.rpt, k++) td[k] = TileDesc{(uint32_t)a, r0, pl.rpt, 0};
            CompactTile *ct = reinterpret_cast<CompactTile *>(hb + s.o_ctiles) + pl.ctiles;
            for (uint32_t sg = 0; sg < pl.n_seg; sg++) ct[sg] = CompactTile{(uint32_t)a, sg, pl.ctiles, pl.n_seg};
        });
        {
            EmitDesc *ed = reinterpret_cast<EmitDesc *>(hb + s.o_emits);
            size_t k = 0;
            for (auto qi : s.emit_q) {
                QState &q = *qs[qi];
                for (auto &e : q.emits) {
                    EmitDesc d = e;
                    d.dst = eng.d_docids_out.p + (size_t)qi * std::max(1u, length) + (uint32_t)(uintptr_t)e.dst;
                    ed[k++] = d;
                }
                q.emits.clear();
            }
        }
        uint32_t n_static = s.n_jobs;
        memcpy(hb + s.o_nstatic, &n_static, 4);
        return B200_OK;
    }
    // the step's copies and kernels on the lane's streams
    int enqueue(Lane &ln, const Step &s) {
        const size_t NA = ln.act_q.size();
        const uint32_t res_words = s.res_words, n_tiles = s.n_tiles, n_ctiles = s.n_ctiles, n_emits = s.n_emits;
        const size_t nbytes = s.nbytes;
        CU(ln.d_step.reserve(nbytes), "step buffer");
        cudaStream_t st = ln.stream;
        CU(cudaMemcpyAsync(ln.d_step.p, ln.h_step, nbytes, cudaMemcpyHostToDevice, st), "H2D step");
        ln.lst.h2d_bytes += nbytes;
        ln.lst.d2h_bytes += (size_t)res_words * 4 + 8;
        size_t qcap = std::max<size_t>((size_t)s.n_jobs + ((size_t)1 << 20), (size_t)4 << 20);
        CU(ln.d_queue.reserve(qcap), "job queue");
        qcap = ln.d_queue.cap;
        CU(ln.d_qcount.reserve(8), "job counter");
        CU(ln.d_results.reserve(res_words + 4), "results");
        if (res_words + 4 > ln.h_results_cap) {
            if (ln.h_results) cudaFreeHost(ln.h_results);
            ln.h_results_cap = (size_t)(res_words + 4) * 2;
            CU(cudaMallocHost((void **)&ln.h_results, ln.h_results_cap * 4), "pinned results");
        }
        if (s.n_jobs) CU(cudaMemcpyAsync(ln.d_queue.p, ln.d_step.p + s.o_jobs, (size_t)s.n_jobs * sizeof(Job), cudaMemcpyDeviceToDevice, st), "jobs to queue");
        CU(cudaMemcpyAsync(ln.d_qcount.p, ln.d_step.p + s.o_nstatic, 4, cudaMemcpyDeviceToDevice, st), "job count");
        const ActDesc *dacts = reinterpret_cast<const ActDesc *>(ln.d_step.p + s.o_acts);
        // 1. emissions queued before this step's activations
        if (ln.timing) CU(cudaEventRecord(ln.e0, st), "event");
        if (n_emits) {
            size_t m0 = ln.mark();
            CU(launch_emit(st, reinterpret_cast<const EmitDesc *>(ln.d_step.p + s.o_emits), n_emits), "emit");
            ln.time_kernel(ln.lst, B200_K_EMIT, m0, ln.mark(), (uint64_t)n_emits * 64);
        }
        if (NA) {
            CU(cudaMemsetAsync(ln.d_results.p, 0, (size_t)(res_words + 4) * 4, st), "zero results");
            CU(cudaMemsetAsync(ln.scratch, 0, s.z_used, st), "zero condition matrix");
            CU(ln.d_pathbuf.reserve(PATH_CAP), "path buffer");
            CU(cudaMemsetAsync(ln.d_qcount.p + 1, 0, 16, st), "zero path count and the scatter cursors");
            size_t t0 = ln.mark();
            CU(ln.d_segcount.reserve(n_ctiles + 1), "segment counts");
            CU(launch_compact(st, reinterpret_cast<const CompactTile *>(ln.d_step.p + s.o_ctiles), n_ctiles, s.multi_segment, dacts, ln.d_segcount.p,
                              ln.d_results.p),
               "compact");
            if (s.multi_segment) ln.lst.kernel_launches++;  // act_count_kernel
            size_t t1 = ln.mark();
            ln.time_kernel(ln.lst, B200_K_COMPACT, t0, t1, s.compact_bytes);
            CU(launch_pair_probe(st, reinterpret_cast<const PairSet *>(ln.d_step.p + s.o_sets), s.n_sets, s.n_probes,
                                 reinterpret_cast<const uint32_t *>(ln.d_step.p + s.o_words), dix.pair_keys, hix.pair_keys.size(), hix.pair_list_base,
                                 dix.lists, dacts, ln.d_results.p, ln.d_queue.p, ln.d_qcount.p, (uint32_t)qcap),
               "pair probe");
            size_t t2 = ln.mark();
            if (s.n_probes) ln.time_kernel(ln.lst, B200_K_PAIR_PROBE, t1, t2, (uint64_t)s.n_probes * 8 * 23);
            CU(ln.d_bigq.reserve(qcap), "big-job queue");
            CU(launch_scatter(st, (uint32_t)eng.sm_count * 5, ln.d_queue.p, ln.d_qcount.p, (uint32_t)qcap, dacts, ln.d_results.p, dix.lists, dix.pool,
                              ln.d_bigq.p),
               "scatter");
            ln.lst.kernel_launches++;
            size_t t3 = ln.mark();
            ln.time_kernel(ln.lst, B200_K_SCATTER, t2, t3, s.fill_bytes);
            // the classes are independent (different activations): class 0 stays on the lane's stream, the others run beside it on
            // forked streams and are joined before the results are copied back
            CU(ln.d_tile_summary.reserve(2 * (size_t)n_tiles + 2), "tile summaries");
            uint32_t n_forked = 0;
            for (uint32_t c = 1; c <= EVAL_CLASSES; c++) n_forked += s.n_tiles_cls[c] ? 1 : 0;
            if (n_forked) CU(cudaEventRecord(ln.ev_fork, st), "fork");
            for (uint32_t c = 0; c <= EVAL_CLASSES; c++) {
                if (!s.n_tiles_cls[c]) continue;
                cudaStream_t cs = c == 0 ? st : ln.cls_stream[c];
                if (c) CU(cudaStreamWaitEvent(cs, ln.ev_fork, 0), "fork wait");
                const TileDesc *tl = reinterpret_cast<const TileDesc *>(ln.d_step.p + s.o_tiles) + s.tile_base[c];
                CU(launch_eval(cs, (int)c, tl, s.n_tiles_cls[c], dacts, ln.d_results.p, reinterpret_cast<const ColOp *>(ln.d_step.p + s.o_colprog),
                               reinterpret_cast<const uint16_t *>(ln.d_step.p + s.o_costs), reinterpret_cast<const uint32_t *>(ln.d_step.p + s.o_prog),
                               ln.d_tile_summary.p + 2 * (size_t)s.tile_base[c]),
                   "eval");
                // pass 2 right behind it on the same stream: all tiles of an activation are in one class, so its counts are final
                if (s.want_paths_cls[c]) {
                    CU(launch_walk(cs, (int)c, tl, s.n_tiles_cls[c], dacts, ln.d_results.p, reinterpret_cast<const ColOp *>(ln.d_step.p + s.o_colprog),
                                   reinterpret_cast<const DpState *>(ln.d_step.p + s.o_states), reinterpret_cast<const DpEdge *>(ln.d_step.p + s.o_edges),
                                   reinterpret_cast<const uint16_t *>(ln.d_step.p + s.o_costs), reinterpret_cast<const uint32_t *>(ln.d_step.p + s.o_prog),
                                   ln.d_tile_summary.p + 2 * (size_t)s.tile_base[c], ln.d_pathbuf.p, ln.d_qcount.p + 1, (uint32_t)PATH_CAP),
                       "walk");
                    ln.lst.kernel_launches++;
                }
                ln.lst.eval_class_launches[c]++;
                ln.lst.eval_class_tiles[c] += s.n_tiles_cls[c];
                if (c) {
                    ln.lst.kernel_launches++;
                    CU(cudaEventRecord(ln.ev_join[c], cs), "join");
                    CU(cudaStreamWaitEvent(st, ln.ev_join[c], 0), "join wait");
                }
            }
            ln.time_kernel(ln.lst, B200_K_EVAL_PATHS, t3, ln.mark(), s.eval_bytes);
            CU(cudaMemcpyAsync(ln.h_results, ln.d_results.p, (size_t)res_words * 4, cudaMemcpyDeviceToHost, st), "D2H results");
            CU(cudaMemcpyAsync(ln.h_results + res_words, ln.d_qcount.p, 16, cudaMemcpyDeviceToHost, st), "D2H counters");
        }
        if (ln.timing) CU(cudaEventRecord(ln.e1, st), "event");
        ln.res_words = res_words;
        ln.qcap = qcap;
        ln.inflight = true;
        return B200_OK;
    }

    // wait for a lane's step, fetch its results and advance its queries
    int finish(Lane &ln) {
        auto t_wait = clk::now();
        CU(cudaStreamSynchronize(ln.stream), "step sync");
        ln.inflight = false;
        {
            float ms = 0;
            if (ln.timing) cudaEventElapsedTime(&ms, ln.e0, ln.e1);
            ln.lst.device_ms += ms;
            ln.resolve_timers(ln.lst);
        }
        const std::vector<uint32_t> &act_q = ln.act_q;
        std::vector<std::unique_ptr<Pending>> &acts = lane_acts[(unsigned)(&ln - lanes)];
        const uint32_t res_words = ln.res_words;
        if (!act_q.empty()) {
            if (ln.h_results[res_words] > ln.qcap) return lane_fail(ln, B200_ERR_CAPACITY, "scatter job queue overflow");
            uint32_t np = ln.h_results[res_words + 1];
            if (np > PATH_CAP) return lane_fail(ln, B200_ERR_CAPACITY, "surviving-path buffer overflow");
            std::vector<PathOut> pouts(np);
            if (np) {
                CU(cudaMemcpyAsync(pouts.data(), ln.d_pathbuf.p, (size_t)np * sizeof(PathOut), cudaMemcpyDeviceToHost, ln.stream), "D2H paths");
                CU(cudaStreamSynchronize(ln.stream), "sync paths");
                ln.lst.d2h_bytes += (size_t)np * sizeof(PathOut);
            }
            for (auto &pd : acts) pd->L->surv.clear();
            for (auto &po : pouts) {
                Level &L = *acts[po.act]->L;
                SurvPath sp;
                sp.cost_idx = po.cost_idx;
                sp.edges.assign(po.edges, po.edges + std::min<uint32_t>(po.len, MAX_WALK));
                L.surv.push_back(std::move(sp));
            }
        }
        ln.lst.host_ms[4] += ms_since(t_wait);
        auto t_adv = clk::now();
        const bool dbg = getenv("B200_DEBUG") != nullptr;
        std::vector<ActOut> outs(acts.size());
        // 1. every activation on its own (activations of one query run on different threads: they only touch their own node, their
        //    ActOut and disjoint entries of the query's score table); sequential-mode queries have one activation and own their state
        ln.pool->run(acts.size(), [&](size_t a) {
            QState &q = *qs[act_q[a]];
            Pending &pd = *acts[a];
            ActOut &out = outs[a];
            Level &L = *pd.L;
            const uint32_t *res = ln.h_results + L.res_off;
            L.rows = res[0];
            size_t nc = L.cost_vals.size();
            L.counts.assign(res + 1, res + 1 + nc + 1);
            L.universe_count = 0;
            for (auto c : L.counts) L.universe_count += c;
            L.cursor = 0;
            L.walked_m = res[1 + nc + 2];
            if (res[1 + nc + 1] != 0) {
                // more distinct surviving paths than the de-duplication table holds: some were not reported.  Run the activation again
                // with a table 16x larger (its work description is still in place); give up at 16 M slots.
                if (L.a_off != SIZE_MAX) out.freed.emplace_back(L.a_off, L.a_len);
                L.a_off = SIZE_MAX;
                if (pd.tab_shift >= 12) {
                    out.status = B200_ERR_CAPACITY;
                    out.error = "more distinct surviving paths in one ranking-rule step than the device path table holds";
                    return;
                }
                pd.tab_shift += 4;
                out.retry = true;
                return;
            }
            if (dbg) {
                std::string msg = "[b200 debug] q" + std::to_string(act_q[a]) + " rule " + std::to_string(L.rule_idx) + " kind " + std::to_string(L.kind) +
                                  " rows " + std::to_string(L.rows) + "/" + std::to_string(L.ld) + " states " + std::to_string(L.n_states) + " edges " +
                                  std::to_string(L.sedges.size()) + " conds " + std::to_string(L.conds.size()) + " cols " + std::to_string(pd.o.n_cols) +
                                  " jobs " + std::to_string(pd.o.jobs.size()) + " costs:";
                for (size_t k = 0; k < L.cost_vals.size(); k++) msg += " " + std::to_string(L.cost_vals[k]) + "=" + std::to_string(L.counts[k]);
                msg += " rest=" + std::to_string(L.counts.back()) + " surv " + std::to_string(L.surv.size());
                fprintf(stderr, "%s\n", msg.c_str());
            }
            try {
                ProfScope ps = profile(PROF_ADVANCE);
                if (pd.node)
                    expand(q, pd.node, out);
                else if (rule_buckets)
                    collect_rule_buckets(q);
                else
                    advance(q);
            } catch (const TooComplex &t) {
                out.status = B200_ERR_CAPACITY;
                out.error = t.why;
            }
        });
        // 2. fold the outcomes into the queries, one thread per query
        std::vector<uint32_t> order(act_q.size());
        for (size_t a = 0; a < order.size(); a++) order[a] = (uint32_t)a;
        std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return act_q[x] < act_q[y]; });
        std::vector<uint32_t> grp;  // start of every query's run in `order`
        for (size_t k = 0; k < order.size(); k++)
            if (k == 0 || act_q[order[k]] != act_q[order[k - 1]]) grp.push_back((uint32_t)k);
        grp.push_back((uint32_t)order.size());
        ln.pool->run(grp.size() - 1, [&](size_t g) {
            QState &q = *qs[act_q[order[grp[g]]]];
            for (uint32_t k = grp[g]; k < grp[g + 1]; k++) {
                ActOut &out = outs[order[k]];
                for (auto &f : out.freed) q.freed.push_back(f);
                if (out.status != 0 && q.status == 0) {
                    q.status = out.status;
                    q.error = out.error;
                }
                if (out.retry) q.pendings.push_back(std::move(acts[order[k]]));
                for (auto &e : out.emits) q.emits.push_back(e);
                for (auto &p : out.pendings) q.pendings.push_back(std::move(p));
                q.outstanding += (uint32_t)out.nodes.size();
                for (auto &n : out.nodes) q.nodes.push_back(std::move(n));
                q.n_results += out.n_results;
                if (out.expanded) q.outstanding--;
            }
            if (q.status != 0)
                abandon(q);
            else if (q.tree && q.outstanding == 0 && q.pendings.empty() && !q.done) {
                q.scores.resize(q.n_results);
                q.nodes.clear();
                q.done = true;
            }
        });
        ln.lst.host_ms[5] += ms_since(t_adv);
        return 0;
    }

    int drive(unsigned dr) {
        cudaError_t ce = cudaSetDevice(eng.device);
        if (ce != cudaSuccess) return cuda_fail(ce, "cudaSetDevice");
        Lane *mine = lanes + dr * lanes_per_driver;
        for (unsigned k = 0; k < lanes_per_driver; k++) {
            int rc = launch(mine[k]);
            if (rc < 0) return rc;
        }
        for (;;) {
            bool any = false;
            for (unsigned k = 0; k < lanes_per_driver; k++) {
                Lane &ln = mine[k];
                if (!ln.inflight) continue;
                any = true;
                int rc = finish(ln);
                if (rc < 0) return rc;
                rc = launch(ln);
                if (rc < 0) return rc;
            }
            if (!any) return 0;
        }
    }
    // run driver dr to the end; its outcome becomes its lanes' (fold_lane_stats reports it)
    void run_driver(unsigned dr) {
        const int rc = drive(dr);
        for (unsigned k = 0; k < lanes_per_driver; k++) lanes[dr * lanes_per_driver + k].rc = std::min(lanes[dr * lanes_per_driver + k].rc, rc);
    }
    // Waves: a driver starts stepping as soon as the terms of ITS queries are derived, while the main thread derives the next
    // driver's (the derivation sweep is serial device + host work at the head of the call).  B200_WAVES caps the number of waves.
    int drive_waves() {
        std::vector<std::thread> drivers;
        unsigned n_waves = std::min(2u, n_drivers);
        if (const char *env = getenv("B200_WAVES")) n_waves = (unsigned)std::max(1, std::min((int)n_drivers, atoi(env)));
        int rc_prep = B200_OK;
        for (unsigned wv = 0; wv < n_waves && rc_prep == B200_OK; wv++) {
            const unsigned d0 = n_drivers * wv / n_waves, d1 = n_drivers * (wv + 1) / n_waves;
            const uint32_t lo = lane_lo(d0 * lanes_per_driver), hi = lane_lo(d1 * lanes_per_driver);
            rc_prep = derive_range(lo, hi);
            if (rc_prep != B200_OK) break;
            start_range(lo, hi);
            eng.kw_derived.store(wv + 1 == n_waves ? Engine::KW_DERIVED_ALL : (int)wv + 1, std::memory_order_release);
            cudaError_t ce = cudaStreamSynchronize(eng.stream);  // row-table memset and derivations visible to the lanes
            if (ce != cudaSuccess) {
                rc_prep = cuda_fail(ce, "sync");
                break;
            }
            for (unsigned dr = d0; dr < d1; dr++) drivers.emplace_back([this, dr]() { run_driver(dr); });
        }
        for (auto &t : drivers) t.join();
        return rc_prep;
    }
    // fold the lanes' statistics (host phases of different lanes overlap in time); returns the first lane's error
    int fold_lane_stats() {
        if (facets)  // facet kernels enqueued by a lane's last schedule() run after its last step: their timers are still open
            for (unsigned l = 0; l < n_lanes; l++) {
                CU(cudaStreamSynchronize(lanes[l].stream), "sync facets");
                lanes[l].resolve_timers(lanes[l].lst);
            }
        for (unsigned l = 0; l < n_lanes; l++) {
            const b200_stats &x = lanes[l].lst;
            stats.kernel_launches += x.kernel_launches;
            stats.device_steps += x.device_steps;
            stats.posting_bytes += x.posting_bytes;
            stats.matrix_bytes += x.matrix_bytes;
            stats.device_ms += x.device_ms;
            stats.h2d_bytes += x.h2d_bytes;
            stats.d2h_bytes += x.d2h_bytes;
            stats.deferred += x.deferred;
            for (int k = 0; k < 9; k++) {
                stats.eval_class_launches[k] += x.eval_class_launches[k];
                stats.eval_class_tiles[k] += x.eval_class_tiles[k];
            }
            stats.arena_peak_bytes = std::max<uint64_t>(stats.arena_peak_bytes, lanes[l].alloc.peak * n_lanes);
            for (int k = 0; k < B200_K_COUNT; k++) {
                stats.kernel_ms[k] += x.kernel_ms[k];
                stats.kernel_count[k] += x.kernel_count[k];
                stats.kernel_bytes[k] += x.kernel_bytes[k];
            }
            for (int k = 3; k <= 5; k++) stats.host_ms[k] += x.host_ms[k] / n_drivers;  // per driver thread (drivers run concurrently)
        }
        for (unsigned l = 0; l < n_lanes; l++)
            if (lanes[l].rc < 0) return lanes[l].rc;
        if (r->candidates || facets || fsearch)
            for (unsigned l = 0; l < n_lanes; l++) CU(cudaStreamSynchronize(lanes[l].stream), "sync candidates");
        return B200_OK;
    }
    // ---- GeoSort as the first rule (geo.cu): the first rows of each query's geo order, as far as the result window needs them
    // The order in which GeoSort's cache hands out the documents of G = universe AND geo is a tuple order (DESIGN.md §3): the
    // first geo_m in rtree order, the rest in iterative order.  Its buckets are runs of that order (the chain of next_bucket,
    // documents/geo_sort.rs:137-228), so the rows are produced from rank 0 up to the end of the bucket that holds the window's
    // last rank: first up to that rank, then further while the chain goes on.
    static constexpr double GEO_MARGIN_M = 1.0;  // GeoSortParameter::distance_error_margin
    // the chain over rows [0, have): ends[k] = one past the last row of bucket k; a bucket is complete when a row breaks the chain
    // after it, when it holds max_bucket_size rows, or when the rows are all of G
    static void geo_chain(const QState &q, uint64_t cap, std::vector<uint32_t> &ends) {
        const uint32_t have = (uint32_t)q.geo_docs.size();
        ends.clear();
        for (uint32_t s = 0; s < have;) {
            const double d0 = q.geo_dist[s];
            uint32_t e = s + 1;
            // `(d0 - d).abs() > margin` ends the bucket (documents/geo_sort.rs:177-180): a NaN distance joins it
            while (e < have && e - s < cap && !(std::fabs(d0 - q.geo_dist[e]) > GEO_MARGIN_M)) e++;
            ends.push_back(e);
            s = e;
        }
    }
    // The iterative keys of the queries whose windows first reach their iterative part in this round (descs in mode 1 or 2): the
    // documents geo_ambiguous_kernel lists are decided with libm into the query's patch.  Then every window gets its query's patch.
    int geo_patches(std::vector<GeoDesc> &descs, const std::vector<std::pair<uint32_t, bool>> &owner) {
        std::vector<uint32_t> fresh;  // one window per query to list
        for (size_t k = 0; k < descs.size(); k++) {
            QState &q = *qs[owner[k].first];
            if (descs[k].mode == 0 || q.geo_patched) continue;
            q.geo_patched = true;
            fresh.push_back((uint32_t)k);
        }
        if (!fresh.empty()) {
            const uint32_t nf = (uint32_t)fresh.size();
            uint32_t cap = 1024;
            std::vector<uint32_t> count(nf);
            for (int attempt = 0; attempt < 2; attempt++) {
                std::vector<GeoDesc> ds(nf);
                CU(eng.d_geo_u32.reserve((size_t)nf * (cap + 1)), "alloc geo ambiguous");
                CU(eng.d_geo_desc.reserve(nf), "alloc geo ambiguous");
                for (uint32_t f = 0; f < nf; f++) {
                    ds[f] = descs[fresh[f]];
                    ds[f].amb_cap = cap;
                    ds[f].amb = eng.d_geo_u32.p + nf + (size_t)f * cap;
                    ds[f].amb_count = eng.d_geo_u32.p + f;
                }
                CU(cudaMemsetAsync(eng.d_geo_u32.p, 0, nf * 4, eng.stream), "memset geo ambiguous");
                CU(cudaMemcpyAsync(eng.d_geo_desc.p, ds.data(), nf * sizeof(GeoDesc), cudaMemcpyHostToDevice, eng.stream), "H2D geo ambiguous");
                const size_t m0 = eng.mark();
                CU(launch_geo_ambiguous(eng.stream, eng.d_geo_desc.p, nf), "geo_ambiguous");
                eng.time_kernel(B200_K_GEO, m0, eng.mark(), 0);
                CU(cudaMemcpyAsync(count.data(), eng.d_geo_u32.p, nf * 4, cudaMemcpyDeviceToHost, eng.stream), "D2H geo ambiguous");
                CU(cudaStreamSynchronize(eng.stream), "sync geo ambiguous");
                stats.h2d_bytes += nf * sizeof(GeoDesc);
                stats.d2h_bytes += nf * 4;
                const uint32_t most = *std::max_element(count.begin(), count.end());
                if (most <= cap) break;
                cap = most;
            }
            std::vector<uint32_t> amb((size_t)nf * cap);
            CU(cudaMemcpyAsync(amb.data(), eng.d_geo_u32.p + nf, amb.size() * 4, cudaMemcpyDeviceToHost, eng.stream), "D2H geo ambiguous");
            CU(cudaStreamSynchronize(eng.stream), "sync geo ambiguous");
            stats.d2h_bytes += amb.size() * 4;
            for (uint32_t f = 0; f < nf; f++) {
                QState &q = *qs[owner[fresh[f]].first];
                const SortRule &rule = q.sort_rules[0];
                for (uint32_t j = 0; j < count[f]; j++) {
                    const uint32_t doc = amb[(size_t)f * cap + j];
                    const uint32_t m = geo_floor_host(geo_distance_host(rule.lat, rule.lng, hix.geo.lat[doc], hix.geo.lng[doc]));
                    q.geo_patch.push_back((unsigned long long)doc << 32 | m);
                }
                std::sort(q.geo_patch.begin(), q.geo_patch.end());
            }
        }
        std::vector<unsigned long long> all;
        std::map<uint32_t, size_t> at;  // query -> offset of its patch in `all`
        for (size_t k = 0; k < descs.size(); k++) {
            const QState &q = *qs[owner[k].first];
            if (descs[k].mode == 0 || q.geo_patch.empty()) continue;
            auto it = at.emplace(owner[k].first, all.size());
            if (it.second) all.insert(all.end(), q.geo_patch.begin(), q.geo_patch.end());
            descs[k].patch = reinterpret_cast<const unsigned long long *>((uintptr_t)it.first->second);  // offsets, made pointers below
            descs[k].n_patch = (uint32_t)q.geo_patch.size();
        }
        if (all.empty()) return B200_OK;
        CU(eng.d_geo_patch.reserve(all.size()), "alloc geo patch");
        CU(cudaMemcpyAsync(eng.d_geo_patch.p, all.data(), all.size() * 8, cudaMemcpyHostToDevice, eng.stream), "H2D geo patch");
        CU(cudaStreamSynchronize(eng.stream), "sync geo patch");  // `all` is pageable and local
        stats.h2d_bytes += all.size() * 8;
        for (GeoDesc &d : descs)
            if (d.n_patch) d.patch = eng.d_geo_patch.p + (uintptr_t)d.patch;
        return B200_OK;
    }
    int geo_windows() {
        const GeoParams gp{b->geo_strategy, b->geo_cache_size ? b->geo_cache_size : 1000u,
                           b->geo_max_bucket_size ? b->geo_max_bucket_size : 1000ull};
        std::vector<uint32_t> gq;
        for (uint32_t i = 0; i < NQ; i++) {
            const QState &q = *qs[i];
            if (q.sort_pending && q.status == 0 && q.sort_rules[0].geo) gq.push_back(i);
        }
        if (gq.empty()) return B200_OK;
        const uint32_t W = hix.n_words64;
        // 1. n = |universe AND geo| per query
        {
            std::vector<GeoCount> cs(gq.size());
            CU(eng.d_geo_count.reserve(gq.size()), "alloc geo counts");
            CU(eng.d_geo_u32.reserve(gq.size()), "alloc geo counts");
            for (size_t k = 0; k < gq.size(); k++) cs[k] = GeoCount{universe_of(*qs[gq[k]]), eng.d_geo_ub, W, eng.d_geo_u32.p + k};
            CU(cudaMemcpyAsync(eng.d_geo_count.p, cs.data(), cs.size() * sizeof(GeoCount), cudaMemcpyHostToDevice, eng.stream), "H2D geo counts");
            const size_t m0 = eng.mark();
            CU(launch_geo_count(eng.stream, eng.d_geo_count.p, (uint32_t)gq.size()), "geo_count");
            eng.time_kernel(B200_K_GEO, m0, eng.mark(), 0);
            std::vector<uint32_t> n(gq.size());
            CU(cudaMemcpyAsync(n.data(), eng.d_geo_u32.p, n.size() * 4, cudaMemcpyDeviceToHost, eng.stream), "D2H geo counts");
            CU(cudaStreamSynchronize(eng.stream), "sync geo counts");
            stats.h2d_bytes += cs.size() * sizeof(GeoCount);
            stats.d2h_bytes += n.size() * 4;
            stats.kernel_bytes[B200_K_GEO] += (uint64_t)gq.size() * W * 16;
            for (size_t k = 0; k < gq.size(); k++) {
                QState &q = *qs[gq[k]];
                q.geo_n = n[k];
                // documents in rtree order (documents/geo_sort.rs:48-63,80-118): Dynamic(c) fills the cache from the rtree while at
                // least c candidates remain, c at a time, and sorts the rest iteratively in one fill
                q.geo_m = gp.strategy == 2 ? q.geo_n : gp.strategy == 1 ? 0u : (q.geo_n >= gp.cache_size ? q.geo_n - q.geo_n % gp.cache_size : 0u);
            }
        }
        // 2. rows of the order, in rounds, until every query's window ends in a complete bucket
        const uint32_t doc_bits = hix.n_docs > 1 ? 32u - (uint32_t)__builtin_clz(hix.n_docs - 1) : 0u;
        std::vector<uint32_t> want(NQ, 0), need(NQ, 0);  // rows asked for; rows the window itself covers
        std::vector<uint32_t> active;
        for (uint32_t i : gq) {
            QState &q = *qs[i];
            const uint32_t ehi = (uint32_t)std::min<uint64_t>(q.univ_count, (uint64_t)q.sort_hi + 1), elo = q.sort_lo > 0 ? q.sort_lo - 1 : 0;
            if (elo < q.geo_n) {
                want[i] = need[i] = std::min(q.geo_n, ehi);
                active.push_back(i);
            }
        }
        while (!active.empty()) {
            std::vector<GeoDesc> descs;
            std::vector<std::pair<uint32_t, bool>> owner;  // query, split select
            size_t rows = 0;
            for (uint32_t i : active) {
                QState &q = *qs[i];
                const SortRule &rule = q.sort_rules[0];
                const bool need_split = q.geo_m > 0 && q.geo_m < q.geo_n && want[i] > q.geo_m && !q.geo_split_known;
                GeoDesc d{};
                d.ub = universe_of(q);
                d.geo = eng.d_geo_ub;
                d.pts = eng.d_geo_pts;
                d.n_words = W;
                // rtree target: lat_lng_to_xyz of the point, or of opposite_of(point) when descending (documents/geo_sort.rs:96-118,280-290)
                double la = rule.lat, ln = rule.lng;
                if (!rule.asc) {
                    la = -la;
                    ln = ln > 0. ? ln - 180. : ln + 180.;
                }
                const double to_rad = M_PI / 180.0, rla = la * to_rad, rln = ln * to_rad;
                d.q[0] = std::cos(rla) * std::cos(rln);
                d.q[1] = std::cos(rla) * std::sin(rln);
                d.q[2] = std::sin(rla);
                d.t_lat = rule.lat;
                d.t_lng = rule.lng;
                d.t_cos_lat = std::cos(rule.lat * to_rad);
                d.asc = rule.asc ? 1 : 0;
                d.doc_max = doc_bits ? (uint32_t)((1ull << doc_bits) - 1) : 0u;
                const uint32_t have = (uint32_t)q.geo_docs.size();
                uint32_t lo = have, hi = want[i];
                if (need_split) {
                    d.mode = 0;
                    lo = q.geo_m - 1;
                    hi = q.geo_m;
                } else if (q.geo_m == q.geo_n || want[i] <= q.geo_m)
                    d.mode = 0;
                else if (q.geo_m == 0)
                    d.mode = 1;
                else {
                    d.mode = 2;
                    d.split_key = q.geo_split_key;
                    d.split_doc = q.geo_split_doc;
                }
                const bool iter_desc = d.mode != 0 && !rule.asc;
                const uint32_t bits[5] = {d.mode == 2 ? 1u : 0u, d.mode == 1 ? 0u : 32u, d.mode == 1 ? GEO_FLOOR_BITS : 32u, iter_desc ? doc_bits : 0u, doc_bits};
                for (int w = 0; w < 5; w++) d.bits[w] = bits[w];
                for (uint32_t at = lo; at < hi; at += SORT_WINDOW) {
                    d.lo = at;
                    d.hi = std::min<uint32_t>(hi, at + SORT_WINDOW);
                    d.dst = reinterpret_cast<uint32_t *>((uintptr_t)rows);  // row offsets, made pointers below
                    rows += d.hi - d.lo;
                    descs.push_back(d);
                    owner.emplace_back(i, need_split);
                }
            }
            const size_t n = descs.size();
            int rc = geo_patches(descs, owner);
            if (rc != B200_OK) return rc;
            CU(eng.d_geo_desc.reserve(n), "alloc geo windows");
            CU(eng.d_geo_u32.reserve(rows + 2 * n), "alloc geo rows");
            CU(eng.d_geo_key.reserve(rows), "alloc geo rows");
            for (size_t k = 0; k < n; k++) {
                const size_t off = (uintptr_t)descs[k].dst;
                descs[k].dst = eng.d_geo_u32.p + off;
                descs[k].dst_key = eng.d_geo_key.p + off;
                descs[k].info = eng.d_geo_u32.p + rows + 2 * k;
            }
            CU(cudaMemcpyAsync(eng.d_geo_desc.p, descs.data(), n * sizeof(GeoDesc), cudaMemcpyHostToDevice, eng.stream), "H2D geo windows");
            const size_t m0 = eng.mark();
            CU(launch_geo_window(eng.stream, eng.d_geo_desc.p, (uint32_t)n), "geo_window");
            eng.time_kernel(B200_K_GEO, m0, eng.mark(), 0);
            std::vector<uint32_t> u32(rows + 2 * n);
            std::vector<unsigned long long> key(rows);
            CU(cudaMemcpyAsync(u32.data(), eng.d_geo_u32.p, u32.size() * 4, cudaMemcpyDeviceToHost, eng.stream), "D2H geo rows");
            CU(cudaMemcpyAsync(key.data(), eng.d_geo_key.p, rows * 8, cudaMemcpyDeviceToHost, eng.stream), "D2H geo rows");
            CU(cudaStreamSynchronize(eng.stream), "sync geo rows");
            eng.resolve_timers();
            stats.h2d_bytes += n * sizeof(GeoDesc);
            stats.d2h_bytes += u32.size() * 4 + rows * 8;
            std::vector<size_t> dist_at(n, SIZE_MAX);  // per window: where its rows' distances go in its query's geo_dist
            for (size_t k = 0; k < n; k++) {
                QState &q = *qs[owner[k].first];
                const GeoDesc &d = descs[k];
                const size_t off = d.dst - eng.d_geo_u32.p, nr = d.hi - d.lo;
                // algorithmic bytes: every pass reads the two bitmaps and a GeoPoint per document of G; the rows are written out
                stats.kernel_bytes[B200_K_GEO] += (uint64_t)u32[rows + 2 * k] * (W * 16ull + q.geo_n * (uint64_t)sizeof(GeoPoint)) + nr * 12ull;
                if (u32[rows + 2 * k + 1] != nr) {
                    q.status = B200_ERR_CUDA;
                    q.error = "internal: geo window collected a different number of documents than its rank range";
                    continue;
                }
                if (owner[k].second) {
                    q.geo_split_known = true;
                    q.geo_split_key = key[off];
                    q.geo_split_doc = u32[off];
                    continue;
                }
                q.geo_docs.insert(q.geo_docs.end(), u32.begin() + off, u32.begin() + off + nr);
                dist_at[k] = q.geo_dist.size();
                q.geo_dist.resize(q.geo_dist.size() + nr);
            }
            // the chain's distances, with libm as the reference computes them (windows write disjoint ranges)
            pfor(n, [&](size_t k) {
                if (dist_at[k] == SIZE_MAX) return;
                QState &q = *qs[owner[k].first];
                const SortRule &rule = q.sort_rules[0];
                const uint32_t *docs = u32.data() + (descs[k].dst - eng.d_geo_u32.p);
                for (uint32_t r = 0; r < descs[k].hi - descs[k].lo; r++)
                    q.geo_dist[dist_at[k] + r] = geo_distance_host(rule.lat, rule.lng, hix.geo.lat[docs[r]], hix.geo.lng[docs[r]]);
            });
            std::vector<uint32_t> next, ends;
            for (uint32_t i : active) {
                QState &q = *qs[i];
                if (q.status != 0) continue;
                const uint32_t have = (uint32_t)q.geo_docs.size();
                if (have < want[i]) {  // waited for its split
                    next.push_back(i);
                    continue;
                }
                geo_chain(q, gp.max_bucket_size, ends);
                const size_t k = std::upper_bound(ends.begin(), ends.end(), need[i] - 1) - ends.begin();  // the bucket of the last rank
                const uint32_t e = ends[k], s = k ? ends[k - 1] : 0;
                if (e < have || e - s == gp.max_bucket_size || have == q.geo_n) continue;  // that bucket is complete
                want[i] = std::min<uint32_t>(q.geo_n, have + std::max<uint32_t>(have, 256));
                next.push_back(i);
            }
            active.swap(next);
        }
        return B200_OK;
    }
    // ---- sort windows of the placeholder searches with sort rules (sort.cu), on the handle's stream
    // A query's ranks [sort_lo, sort_hi) are produced with one more rank on each side where the universe has it: under Skip a bucket
    // of at most one document is returned with the scores of the rules above it only (bucket_sort.rs:299-312), and whether a
    // document's group of equal keys is a singleton shows in its neighbours.  Without a GeoSort rule those ranks are one segment of
    // the universe's (keys, docid) order.  With a leading GeoSort rule (geo_windows) they are cut into segments along its buckets:
    // each geo bucket is ordered by the following rules' (keys, docid) over its docid list, and the ranks past the geo documents by
    // the same over the universe without them (the Null bucket); the GeoSort rule's key is the bucket's index.
    int sort_windows() {
        struct Seg {
            uint32_t q, ext_row;    // query, first extended-window row
            uint32_t first_level;   // 1: level 0 is a GeoSort rule whose key is `bucket`
            uint32_t bucket;
        };
        std::vector<SortDesc> descs;
        std::vector<Seg> owner;  // per window
        std::vector<uint32_t> lists;  // docids of the geo buckets the windows read, uploaded with the windows
        std::vector<std::pair<size_t, size_t>> list_of;  // per window: (offset into lists, length), length 0 = none
        size_t key_words = 0, id_words = 0;
        const uint32_t doc_bits = hix.n_docs > 1 ? 32u - (uint32_t)__builtin_clz(hix.n_docs - 1) : 0u;
        std::vector<uint32_t> q_elo(NQ, 0);
        std::vector<std::vector<uint32_t>> geo_p0(NQ);  // per query: the first docid of each geo bucket
        auto add_windows = [&](QState &q, const SortDesc &proto, uint32_t lo, uint32_t hi, Seg seg, size_t list_off, size_t list_len) {
            const uint32_t Lf = (uint32_t)q.sort_rules.size() - seg.first_level;
            for (uint32_t at = lo; at < hi; at += SORT_WINDOW) {
                SortDesc d = proto;
                d.lo = at;
                d.hi = std::min<uint32_t>(hi, at + SORT_WINDOW);
                d.dst = reinterpret_cast<uint32_t *>((uintptr_t)id_words);  // offsets, made pointers below
                id_words += d.hi - d.lo;
                d.dst_keys = reinterpret_cast<uint32_t *>((uintptr_t)key_words);
                key_words += (size_t)(d.hi - d.lo) * Lf;
                descs.push_back(d);
                Seg s = seg;
                s.ext_row += at - lo;
                owner.push_back(s);
                list_of.emplace_back(list_off, list_len);
            }
        };
        for (uint32_t i = 0; i < NQ; i++) {
            QState &q = *qs[i];
            if (!q.sort_pending || q.status != 0) continue;
            const uint32_t L = (uint32_t)q.sort_rules.size(), first = q.sort_rules[0].geo ? 1u : 0u;
            const uint32_t elo = q.sort_lo > 0 ? q.sort_lo - 1 : 0, ehi = (uint32_t)std::min<uint64_t>(q.univ_count, (uint64_t)q.sort_hi + 1);
            q_elo[i] = elo;
            SortDesc proto{};
            proto.ub = universe_of(q);
            proto.n_words = hix.n_words64;
            proto.n_levels = L - first;
            for (uint32_t l = first; l < L; l++) {
                auto it = hix.sort_fields.find(q.sort_rules[l].fid);
                if (it == hix.sort_fields.end()) continue;  // no value anywhere: one Null bucket
                const uint32_t V = it->second.n_values();
                proto.keys[l - first] = it->second.d_key[q.sort_rules[l].asc ? 0 : 1];
                proto.bits[l - first] = V ? 32u - (uint32_t)__builtin_clz(V) : 0u;
            }
            proto.bits[L - first] = doc_bits;
            if (!first) {
                add_windows(q, proto, elo, ehi, Seg{i, 0, 0, 0}, 0, 0);
                continue;
            }
            // geo buckets over the rows geo_windows produced, then the Null bucket
            const uint64_t cap = b->geo_max_bucket_size ? b->geo_max_bucket_size : 1000ull;
            std::vector<uint32_t> ends;
            if (elo < q.geo_n) geo_chain(q, cap, ends);
            for (uint32_t bucket = 0, bs = 0; bucket < ends.size() && bs < ehi; bs = ends[bucket++]) {
                const uint32_t be = ends[bucket];
                geo_p0[i].push_back(q.geo_docs[bs]);
                if (be > elo) {
                    SortDesc d = proto;
                    d.n_ids = be - bs;  // d.ids: set below from list_of
                    const size_t off = lists.size();
                    lists.insert(lists.end(), q.geo_docs.begin() + bs, q.geo_docs.begin() + be);
                    const uint32_t lo = std::max(elo, bs), hi = std::min(ehi, be);
                    add_windows(q, d, lo - bs, hi - bs, Seg{i, lo - elo, 1, bucket}, off, be - bs);
                }
            }
            if (ehi > q.geo_n) {
                SortDesc d = proto;
                d.exclude = eng.d_geo_ub;
                const uint32_t lo = std::max(elo, q.geo_n);
                add_windows(q, d, lo - q.geo_n, ehi - q.geo_n, Seg{i, lo - elo, 1, 0xffffffffu}, 0, 0);
            }
        }
        if (descs.empty()) return B200_OK;
        const size_t n = descs.size();
        CU(eng.d_sort_keys.reserve(std::max<size_t>(1, key_words + id_words + lists.size())), "alloc sort keys");
        CU(eng.d_sort_info.reserve(2 * n), "alloc sort info");
        CU(eng.d_sort_desc.reserve(n), "alloc sort windows");
        uint32_t *d_lists = eng.d_sort_keys.p + key_words + id_words;
        for (size_t k = 0; k < n; k++) {
            descs[k].dst_keys = eng.d_sort_keys.p + (uintptr_t)descs[k].dst_keys;
            descs[k].dst = eng.d_sort_keys.p + key_words + (uintptr_t)descs[k].dst;
            descs[k].info = eng.d_sort_info.p + 2 * k;
            if (list_of[k].second) descs[k].ids = d_lists + list_of[k].first;
        }
        if (!lists.empty())
            CU(cudaMemcpyAsync(d_lists, lists.data(), lists.size() * 4, cudaMemcpyHostToDevice, eng.stream), "H2D geo buckets");
        CU(cudaMemcpyAsync(eng.d_sort_desc.p, descs.data(), n * sizeof(SortDesc), cudaMemcpyHostToDevice, eng.stream), "H2D sort windows");
        const size_t m0 = eng.mark();
        CU(launch_sort_window(eng.stream, eng.d_sort_desc.p, (uint32_t)n), "sort_window");
        eng.time_kernel(B200_K_SORT, m0, eng.mark(), 0);
        std::vector<uint32_t> keys(key_words + id_words), info(2 * n);
        CU(cudaMemcpyAsync(keys.data(), eng.d_sort_keys.p, (key_words + id_words) * 4, cudaMemcpyDeviceToHost, eng.stream), "D2H sort keys");
        CU(cudaMemcpyAsync(info.data(), eng.d_sort_info.p, 2 * n * 4, cudaMemcpyDeviceToHost, eng.stream), "D2H sort info");
        CU(cudaStreamSynchronize(eng.stream), "sync sort");
        eng.resolve_timers();
        stats.h2d_bytes += n * sizeof(SortDesc) + lists.size() * 4;
        stats.d2h_bytes += (key_words + id_words) * 4 + 2 * n * 4;
        // the extended windows: per query its rows' docids and all L keys
        std::vector<std::vector<uint32_t>> ext_ids(NQ), ext_keys(NQ);
        for (uint32_t i = 0; i < NQ; i++) {
            QState &q = *qs[i];
            if (!q.sort_pending || q.status != 0) continue;
            const uint32_t n_ext = (uint32_t)std::min<uint64_t>(q.univ_count, (uint64_t)q.sort_hi + 1) - q_elo[i];
            ext_ids[i].assign(n_ext, 0);
            ext_keys[i].assign((size_t)n_ext * q.sort_rules.size(), 0);
        }
        for (size_t k = 0; k < n; k++) {
            const SortDesc &d = descs[k];
            const Seg &sg = owner[k];
            QState &q = *qs[sg.q];
            const uint32_t rows = d.hi - d.lo, Lf = d.n_levels, L = (uint32_t)q.sort_rules.size();
            // algorithmic bytes: every pass reads the universe (words, or a list) and one key per document; the window writes docids + keys
            const uint64_t set_bytes = d.ids ? d.n_ids * 4ull : hix.n_words64 * 8ull * (d.exclude ? 2 : 1);
            stats.kernel_bytes[B200_K_SORT] += (uint64_t)info[2 * k] * (set_bytes + (d.ids ? d.n_ids : q.univ_count) * 4ull) + (uint64_t)rows * 4 * (Lf + 1);
            if (info[2 * k + 1] != rows) {
                q.status = B200_ERR_CUDA;
                q.error = "internal: sort window collected a different number of documents than its rank range";
                continue;
            }
            const uint32_t *ids = keys.data() + key_words + (d.dst - (eng.d_sort_keys.p + key_words));
            const uint32_t *kp = keys.data() + (d.dst_keys - eng.d_sort_keys.p);
            for (uint32_t r = 0; r < rows; r++) {
                const size_t e = sg.ext_row + r;
                ext_ids[sg.q][e] = ids[r];
                if (sg.first_level) ext_keys[sg.q][e * L] = sg.bucket;
                for (uint32_t l = 0; l < Lf; l++) ext_keys[sg.q][e * L + sg.first_level + l] = kp[(size_t)r * Lf + l];
            }
        }
        for (uint32_t i = 0; i < NQ; i++) {
            QState &q = *qs[i];
            if (!q.sort_pending || q.status != 0) continue;
            const uint32_t L = (uint32_t)q.sort_rules.size(), elo = q_elo[i];
            const uint32_t n_ext = (uint32_t)ext_ids[i].size();
            const uint32_t *kp = ext_keys[i].data();
            auto shares = [&](uint32_t a, uint32_t b, uint32_t n_keys) {  // keys [0, n_keys) of ext rows a and b agree
                for (uint32_t l = 0; l < n_keys; l++)
                    if (kp[(size_t)a * L + l] != kp[(size_t)b * L + l]) return false;
                return true;
            };
            q.sort_ids.assign(ext_ids[i].begin() + (q.sort_lo - elo), ext_ids[i].begin() + (q.sort_hi - elo));
            for (uint32_t j = 0; j < q.sort_hi - q.sort_lo; j++) {
                const uint32_t e = q.sort_lo - elo + j;
                // Under Skip a document leaves bucket_sort early at the first rule l (top down) where either
                //  - the rule's remaining universe is that document alone (bucket_sort.rs:196-204): it is the last of its group of
                //    equal keys [0, l) and no other document of that group shares its key l -> the scores of the rules above l;
                //  - the rule's bucket holding it has no other document (:299-312) -> the scores of rules [0, l].
                uint32_t n_sc = L;
                if (skip_scoring)
                    for (uint32_t l = 0; l < L; l++) {
                        const bool has_prev = e > 0, has_next = e + 1 < n_ext;
                        const bool last_of_group = !(has_next && shares(e, e + 1, l));
                        const bool alone = !(has_prev && shares(e, e - 1, l + 1)) && !(has_next && shares(e, e + 1, l + 1));
                        if (last_of_group && alone) {
                            n_sc = l;
                            break;
                        }
                        if (alone) {
                            n_sc = l + 1;
                            break;
                        }
                    }
                std::vector<EScore> &sc = q.scores[j];
                sc.clear();
                for (uint32_t l = 0; l < n_sc; l++) {
                    const SortRule &rule = q.sort_rules[l];
                    const uint32_t key = kp[(size_t)e * L + l];
                    if (rule.geo) {  // ScoreDetails::GeoSort: the bucket's first point, None for the Null bucket
                        sc.push_back(EScore{B200_S_GEO_SORT, key == 0xffffffffu ? key : geo_p0[i][key], rule.asc ? 2u : 0u, -1.f});
                        continue;
                    }
                    auto it = hix.sort_fields.find(rule.fid);
                    bool is_string = false;
                    uint32_t key_index = 0xffffffffu;
                    if (it != hix.sort_fields.end() && key < it->second.n_values()) it->second.decode(rule.asc, key, is_string, key_index);
                    sc.push_back(EScore{B200_S_SORT, key_index, (uint32_t)rule.fid << 2 | (rule.asc ? 2u : 0u) | (is_string ? 1u : 0u), -1.f});
                }
            }
        }
        return B200_OK;
    }
    int write_results() {
        std::vector<uint32_t> out_ids((size_t)NQ * std::max(1u, length));
        CU(cudaMemcpyAsync(out_ids.data(), eng.d_docids_out.p, out_ids.size() * 4, cudaMemcpyDeviceToHost, eng.stream), "D2H docids");
        stats.d2h_bytes += out_ids.size() * 4;
        stats.h2d_bytes += (size_t)b->lemma_off[b->token_begin[NQ]] + (size_t)b->token_begin[NQ] * 5 + (size_t)NQ * 4;
        CU(cudaStreamSynchronize(eng.stream), "sync");
        if (facets && facet_outputs) {
            std::vector<std::string> err;
            const int rc = eng.facet_results(fout, b->facet_fid, *r, err);
            if (rc != B200_OK) return rc;
            for (uint32_t i = 0; i < NQ; i++) {
                QState &q = *qs[i];
                for (uint32_t k = b->facet_begin[i]; k < b->facet_begin[i + 1]; k++) {
                    if (q.status == 0 && !err[k].empty()) {  // this slot needs more than facet_cap entries: the query fails alone
                        q.status = B200_ERR_CAPACITY;
                        q.error = err[k];
                    }
                    if (q.status != 0) r->facet_n_num[k] = r->facet_n_str[k] = r->facet_has_stats[k] = 0;
                }
            }
        }
        for (uint32_t i = 0; i < NQ; i++) {
            QState &q = *qs[i];
            if (r->status) r->status[i] = q.status;
            if (q.status != 0) {
                r->n_hits[i] = 0;
                if (r->n_candidates) r->n_candidates[i] = 0;
                eng.last_error = q.error;
                continue;
            }
            r->n_hits[i] = q.n_results;
            if (q.sort_pending)
                for (uint32_t k = 0; k < q.n_results; k++) out_ids[(size_t)i * std::max(1u, length) + k] = q.sort_ids[k];
            if (r->n_candidates) r->n_candidates[i] = q.n_candidates;
            if (r->degraded) r->degraded[i] = q.degraded ? 1 : 0;
            if (r->used_negative_operator) r->used_negative_operator[i] = q.used_negative ? 1 : 0;
            for (uint32_t k = 0; k < q.n_results; k++) {
                r->docids[(size_t)i * length + k] = out_ids[(size_t)i * std::max(1u, length) + k];
                if (r->n_scores) {
                    const auto &sc = q.scores[k];
                    size_t ns = std::min<size_t>(sc.size(), B200_MAX_SCORES);
                    r->n_scores[(size_t)i * length + k] = (uint8_t)ns;
                    for (size_t s = 0; s < ns; s++) {
                        size_t at = ((size_t)i * length + k) * B200_MAX_SCORES + s;
                        r->score_kind[at] = sc[s].kind;
                        r->score_rank[at] = sc[s].rank;
                        r->score_max[at] = sc[s].max_rank;
                        r->score_sim[at] = sc[s].sim;
                    }
                }
            }
        }
        return B200_OK;
    }
    // B200_WORK_HIST / B200_PROFILE reports of the batch
    void debug_reports() {
        if (work_hist) {
            static const char *ucls[4] = {"ld<128", "ld<4096", "ld<65536", "ld>=65536"};
            static const char *kinds[10] = {"words", "typo", "proximity", "fid", "position", "exactness", "exact_attr", "resolve", "freq", "?"};
            for (int u = 0; u < 4; u++) {
                fprintf(stderr, "[b200 work] scatter lists, universe %s (pair probes %llu):\n", ucls[u], (unsigned long long)work_hist->probes[u]);
                for (int c = 0; c < 33; c++)
                    if (work_hist->lists[u][c][0])
                        fprintf(stderr, "    %s%-2d lists %9llu  bytes %8.1f MB\n", c == 32 ? "dense " : "card<=2^", c == 32 ? 0 : c,
                                (unsigned long long)work_hist->lists[u][c][0], work_hist->lists[u][c][1] / 1e6);
            }
            for (int k = 0; k < 10; k++)
                for (int u = 0; u < 4; u++)
                    if (work_hist->eval[k][u][0])
                        fprintf(stderr, "[b200 work] eval %-10s %-10s acts %7llu rows %10llu row*ops %12llu row*cols %11llu\n", kinds[k], ucls[u],
                                (unsigned long long)work_hist->eval[k][u][0], (unsigned long long)work_hist->eval[k][u][1],
                                (unsigned long long)work_hist->eval[k][u][2], (unsigned long long)work_hist->eval[k][u][3]);
        }
        if (prof)
            fprintf(stderr, "[b200 profile] thread-ms: build_from_paths %.2f  prepare_graph_rule %.2f  request_activation %.2f  advance(total) %.2f\n",
                    prof_ns[0] / 1e6, prof_ns[1] / 1e6, prof_ns[2] / 1e6, prof_ns[3] / 1e6);
    }
    // tear the per-query state down off the critical path
    void reap() {
        for (auto &t : eng.reapers)
            if (t.joinable()) t.join();
        eng.reapers.clear();
        {
            const size_t n_reapers = 4, per = (qs.size() + n_reapers - 1) / n_reapers;
            for (size_t r0 = 0; r0 < qs.size(); r0 += std::max<size_t>(1, per)) {
                auto *dead = new std::vector<std::unique_ptr<QState>>();
                for (size_t i = r0; i < std::min(qs.size(), r0 + per); i++) dead->push_back(std::move(qs[i]));
                eng.reapers.emplace_back([dead]() { delete dead; });
            }
        }
    }
    // after the step loop: statistics, sort windows, results and reports; the per-query state is freed in the background
    int finish_batch() {
        int rc = fold_lane_stats();
        if (rc == B200_OK) rc = geo_windows();
        if (rc == B200_OK) rc = sort_windows();
        if (rc != B200_OK) return rc;
        const auto t_out = clk::now();
        if ((rc = write_results()) != B200_OK) return rc;
        debug_reports();
        reap();
        stats.host_ms[6] += ms_since(t_out);
        stats.host_ms[7] += ms_since(t_total);
        return B200_OK;
    }
};

}  // namespace

// The sort rules of query qi (search/new/mod.rs:351-416, 651-716): the `Sort` criterion expands to the query's `sort` list at its
// position, once; Asc(f) / Desc(f) criteria add one rule each; a field sorted earlier in the list is skipped; every `_geoPoint`
// entry adds a GeoSort rule.  Sort is built for
// placeholder keyword searches; every other search with sort rules is refused with B200_ERR_UNSUPPORTED rather than answered without
// them.  Returns B200_OK with the rules in `out`, or the code the query fails with and `why`.
int Engine::sort_rules(const b200_query_batch *b, uint32_t qi, bool semantic, bool placeholder, std::vector<SortRule> &out, const char *&why) const {
    bool has_sort_criterion = false, has_custom = false;
    for (int c : hix.settings.criteria) {
        has_sort_criterion |= c == B200_C_SORT;
        has_custom |= (c & 0x30000) != 0;
    }
    const uint32_t s0 = b->sort_begin ? b->sort_begin[qi] : 0, s1 = b->sort_begin ? b->sort_begin[qi + 1] : 0;
    if (s1 > s0 && !has_sort_criterion) {  // check_sort_criteria (search/new/mod.rs:998-1016)
        why = "SortRankingRuleMissing: a sort list was given but the ranking rules do not contain `sort`";
        return B200_ERR_INVALID;
    }
    if (semantic) {  // get_ranking_rules_for_vector (search/new/mod.rs:419-508)
        if (s1 == s0 && !has_custom) return B200_OK;
        why = "sort rules in a semantic search (sort list or Asc/Desc criteria) are not built";
        return B200_ERR_UNSUPPORTED;
    }
    if (s1 > s0 && (!b->sort_fid || !b->sort_asc)) {
        why = "sort_begin without sort_fid / sort_asc";
        return B200_ERR_INVALID;
    }
    bool has_geo = false;
    for (uint32_t k = s0; k < s1 && b->sort_geo; k++) has_geo |= b->sort_geo[k] != 0;
    if (has_geo && !b->sort_geo_point) {
        why = "sort_geo without sort_geo_point";
        return B200_ERR_INVALID;
    }
    if (has_geo && (b->geo_strategy < 0 || b->geo_strategy > 2)) {
        why = "geo_strategy is not 0 (Dynamic), 1 (AlwaysIterative) or 2 (AlwaysRtree)";
        return B200_ERR_INVALID;
    }
    std::vector<SortRule> sr;
    std::vector<uint16_t> sorted;
    bool sort_done = false;
    auto add = [&](uint16_t fid, bool asc) {
        // 0xFFFF stands for every field absent from the fields map: its entries are never "already sorted" (the caller,
        // which sees the names, drops a repeated absent name)
        if (fid != 0xFFFF && std::find(sorted.begin(), sorted.end(), fid) != sorted.end()) return;
        sorted.push_back(fid);
        sr.push_back(SortRule{fid, asc});
    };
    for (int c : hix.settings.criteria) {
        if (c == B200_C_SORT && !sort_done) {
            sort_done = true;
            for (uint32_t k = s0; k < s1; k++) {
                if (b->sort_geo && b->sort_geo[k])  // one GeoSort rule per entry, never deduplicated (geo_sorted is never set)
                    sr.push_back(SortRule{0xFFFF, b->sort_asc[k] != 0, true, b->sort_geo_point[2 * k], b->sort_geo_point[2 * k + 1]});
                else
                    add(b->sort_fid[k], b->sort_asc[k] != 0);
            }
        } else if (c & 0x10000)
            add((uint16_t)(c & 0xffff), true);
        else if (c & 0x20000)
            add((uint16_t)(c & 0xffff), false);
    }
    if (sr.empty()) return B200_OK;
    if (b->mode != 0)
        why = "sort in a semantic or hybrid search (needs the ScoreValue::Sort comparator of hybrid.rs)";
    else if (!placeholder)
        why = "sort rule in a search with query terms (sort is built for placeholder searches)";
    else if (sr.size() > B200_MAX_SCORES)
        why = "more than B200_MAX_SCORES sort rules";
    else if (b->stop_after >= 0)
        why = "stop_after together with a sort rule (the sort window is one device step; its polls are not counted)";
    else if (std::any_of(sr.begin() + 1, sr.end(), [](const SortRule &x) { return x.geo; }))
        why = "GeoSort rule after the first rule of the stack (it is built as the first rule only)";
    else {
        out = std::move(sr);
        return B200_OK;
    }
    return B200_ERR_UNSUPPORTED;
}

int Engine::keyword_batch(const b200_query_batch *b, b200_results *r, uint32_t offset, uint32_t limit, int scoring) {
    CU(cudaSetDevice(device), "cudaSetDevice");
    AffinityScope on_gpu_socket(affinity);  // before any thread of this call is created
    KeywordBatch kb(*this, b, r, offset, limit, scoring);
    kb.parse();
    kb.resolve_sort_rules();
    kb.check_facets();
    int rc = kb.stage_universes();
    if (rc == B200_OK) rc = kb.setup_lanes();
    if (rc == B200_OK) rc = kb.setup_facets();
    if (rc == B200_OK) rc = kb.setup_facet_search();
    if (rc == B200_OK) rc = kb.drive_waves();
    if (rc == B200_OK) rc = kb.finish_batch();
    return rc;
}

// ================================================================================================ S1: the RankingRule seam
void free_graph(GraphObj *g) { delete g; }

struct Engine::RuleRun {
    std::vector<RuleBucket> buckets;
    size_t cursor = 0;
    ~RuleRun() {
        for (auto &b : buckets) delete b.child;
    }
};

// QueryGraph::from_query (query_graph.rs:96-187) over located_query_terms_from_tokens (parse_query.rs:28-202), with every term's
// derivations computed (compute_derivations.rs:21-37): what bucket_sort hands to the first ranking rule
int Engine::graph_from_tokens(const b200_query_batch *one, GraphObj **out) {
    *out = nullptr;
    if (one->n_queries != 1) return fail(B200_ERR_INVALID, "graph_from_tokens takes exactly one query");
    CU(cudaSetDevice(device), "cudaSetDevice");
    AffinityScope on_gpu_socket(affinity);
    b200_results none{};
    KeywordBatch kb(*this, one, &none, 0, 1, 0);
    kb.parse();
    // Sort rules are resolved as in a search, so on an index whose criteria hold Asc/Desc a query with terms is refused with
    // B200_ERR_UNSUPPORTED (sort is built for placeholder searches only).
    kb.resolve_sort_rules();
    int rc = kb.stage_universes();
    if (rc == B200_OK) rc = kb.derive_range(0, 1);
    if (rc != B200_OK) return rc;
    const QState &q = *kb.qs[0];
    if (q.status != 0) return fail(q.status, q.error);
    *out = new GraphObj(q.ctx, q.graph);
    return B200_OK;
}

// RankingRule::start_iteration (ranking_rules.rs:35-45) for one of the graph-based rules or ExactAttribute: all buckets of the rule
// over `universe` are evaluated at once (one device step) and served by rule_next
int Engine::rule_start(int rule_kind, int tms, const GraphObj *query, const uint64_t *universe, uint64_t n_universe_words, RuleRun **out) {
    *out = nullptr;
    static const int kinds[7] = {RK_WORDS, RK_TYPO, RK_PROXIMITY, RK_FID, RK_POSITION, RK_EXACT_ATTRIBUTE, RK_EXACTNESS};
    if (rule_kind < 0 || rule_kind > 6 || !query) return fail(B200_ERR_INVALID, "rule_start: unknown rule kind or null query graph");
    static const uint32_t zeros[2] = {0, 0};
    static const uint8_t kind0[1] = {0};
    b200_query_batch b{};
    b.n_queries = 1;
    b.token_begin = zeros;
    b.token_kind = kind0;
    b.lemma_off = zeros;
    b.lemma_bytes = "";
    b.terms_matching_strategy = tms;
    b.limit = 1;
    b.words_limit = 10;
    b.stop_after = -1;
    const uint64_t *up[1] = {universe};
    if (universe) {
        b.universes = up;
        b.n_universe_words = n_universe_words;
    }
    uint32_t docids[1], n_hits[1];
    int32_t status[1];
    uint64_t n_cand[1];
    b200_results r{};
    r.docids = docids;
    r.n_hits = n_hits;
    r.status = status;
    r.n_candidates = n_cand;
    CU(cudaSetDevice(device), "cudaSetDevice");
    AffinityScope on_gpu_socket(affinity);
    std::unique_ptr<RuleRun> run(new RuleRun());
    KeywordBatch kb(*this, &b, &r, 0, 1, 0);
    kb.rule_buckets = &run->buckets;
    QState &q = *kb.qs[0];
    static_cast<QTerms &>(q.ctx) = query->ctx;
    q.graph = query->graph;
    // Sort rules are resolved as in a search.  The query graph is never parsed here, so it is never a placeholder: on an index whose
    // criteria hold Asc/Desc every rule_start is refused with B200_ERR_UNSUPPORTED.
    kb.resolve_sort_rules();
    int rc = kb.stage_universes();
    if (rc == B200_OK) rc = kb.setup_lanes();
    if (rc == B200_OK) {
        if (!q.done) kb.start_rule(q, kinds[rule_kind]);
        CU(cudaStreamSynchronize(stream), "sync");  // row-table memset visible to the lane
        kb.run_driver(0);
        rc = kb.finish_batch();
    }
    if (rc != B200_OK) return rc;
    if (status[0] != 0) return fail(status[0], last_error);
    *out = run.release();
    return B200_OK;
}

}  // namespace b200

namespace b200 {
int rule_next_impl(Engine::RuleRun *run, uint64_t n_words64, const uint64_t *universe, uint64_t *out_bitmap, uint64_t n_words, uint32_t *rank,
                   uint32_t *max_rank, GraphObj **out_query) {
    if (run->cursor >= run->buckets.size()) return 1;
    RuleBucket &b = run->buckets[run->cursor++];
    if (rank) *rank = b.rank;
    if (max_rank) *max_rank = b.max_rank;
    if (out_bitmap)
        for (uint64_t w = 0; w < n_words; w++) out_bitmap[w] = w < n_words64 ? (b.bitmap[w] & (universe ? universe[w] : ~0ull)) : 0ull;
    if (out_query) {
        *out_query = b.child;
        b.child = nullptr;
    }
    return 0;
}
void rule_end_impl(Engine::RuleRun *run) { delete run; }
}  // namespace b200
