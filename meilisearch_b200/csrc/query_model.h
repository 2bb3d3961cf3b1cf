// Host-side query model of the engine: terms, term subsets, query graph, ranking-rule graph.
// GPU-native restatement (word ids are dictionary ranks, derivations arrive from the device):
//   crates/milli/src/search/new/query_term/{mod.rs,ntypo_subset.rs,parse_query.rs,compute_derivations.rs:170-253}
//   crates/milli/src/search/new/query_graph.rs
//   crates/milli/src/search/new/ranking_rule_graph/{build.rs,mod.rs} and the six rule directories
// Scope: words, soft/hard separators, prefix, typos, n-grams, split words, user phrases, synonyms, the negative operator
// (DESIGN.md §1 lists what is reported as B200_ERR_UNSUPPORTED).
#pragma once
#include <algorithm>
#include <cstdint>
#include <map>
#include <string>
#include <vector>

#include "host_index.h"

namespace b200 {

enum { N_ALL = 0, N_SUBSET = 1, N_NOTHING = 2 };

struct ETerm {  // QueryTerm (query_term/mod.rs:43-54)
    std::string original;
    bool is_ngram = false;
    std::vector<std::string> ngram_words;
    uint8_t max_lev = 0;
    bool is_prefix = false;
    bool empty_term = false;  // longer than MAX_WORD_LENGTH
    int32_t exact = -1;       // dictionary rank of `original`, or -1
    std::vector<uint32_t> prefix_of;
    int32_t prefix_db = -1;   // prefix id
    std::vector<uint32_t> one_typo, two_typo;
    int32_t phrase = -1;             // zero_typo.phrase: the user phrase this term stands for (phrase id)
    std::vector<uint32_t> synonyms;  // zero_typo.synonyms (phrase ids)
    int32_t split = -1;              // one_typo.split_words (phrase id of the 2-word split)
    int32_t lev_slot = -1;           // index into the device derivation batch
    bool allows_split_words() const { return phrase < 0; }
};

// Phrase (query_term/phrase.rs): dictionary ranks; -1 = stop-word hole; -2 = a word that is not in the dictionary
struct EPhrase {
    std::vector<int32_t> words;
};

struct ESubset {  // NTypoTermSubset
    uint8_t kind = N_NOTHING;
    std::vector<uint32_t> words;    // sorted
    std::vector<uint32_t> phrases;  // sorted phrase ids
    bool contains_word(uint32_t w) const { return kind == N_ALL || (kind == N_SUBSET && std::binary_search(words.begin(), words.end(), w)); }
    bool contains_phrase(uint32_t p) const { return kind == N_ALL || (kind == N_SUBSET && std::binary_search(phrases.begin(), phrases.end(), p)); }
    bool is_empty() const { return kind == N_NOTHING || (kind == N_SUBSET && words.empty() && phrases.empty()); }
    void intersect(const ESubset &o) {
        if (kind == N_ALL)
            *this = o;
        else if (kind == N_SUBSET) {
            if (o.kind == N_SUBSET) {
                std::vector<uint32_t> r;
                std::set_intersection(words.begin(), words.end(), o.words.begin(), o.words.end(), std::back_inserter(r));
                words.swap(r);
                std::vector<uint32_t> rp;
                std::set_intersection(phrases.begin(), phrases.end(), o.phrases.begin(), o.phrases.end(), std::back_inserter(rp));
                phrases.swap(rp);
            } else if (o.kind == N_NOTHING)
                *this = ESubset{};
        }
    }
    bool operator==(const ESubset &o) const { return kind == o.kind && words == o.words && phrases == o.phrases; }
    void key(std::string &s) const {  // binary identity key (cheap: no number formatting)
        s.push_back((char)('A' + kind));
        uint32_t nw = (uint32_t)words.size();
        s.append(reinterpret_cast<const char *>(&nw), 4);
        if (!words.empty()) s.append(reinterpret_cast<const char *>(words.data()), words.size() * 4);
        uint32_t np = (uint32_t)phrases.size();
        s.append(reinterpret_cast<const char *>(&np), 4);
        if (np) s.append(reinterpret_cast<const char *>(phrases.data()), phrases.size() * 4);
    }
};

struct ETermSubset {
    uint32_t term = 0;
    ESubset zero, one, two;
    bool mandatory = false;
    static ETermSubset full(uint32_t t) {
        ETermSubset s;
        s.term = t;
        s.zero.kind = s.one.kind = s.two.kind = N_ALL;
        return s;
    }
    void intersect(const ETermSubset &o) {
        zero.intersect(o.zero);
        one.intersect(o.one);
        two.intersect(o.two);
    }
};

struct ELocated {  // LocatedQueryTermSubset
    ETermSubset ts;
    uint16_t ps = 0, pe = 0;
    uint8_t t0 = 0, t1 = 0;
    uint32_t n_term_ids() const { return (uint32_t)t1 - t0 + 1; }
    void key(std::string &s) const {
        s.append(reinterpret_cast<const char *>(&ts.term), 4);
        s.push_back(ts.mandatory ? '!' : '.');
        ts.zero.key(s);
        ts.one.key(s);
        ts.two.key(s);
        s.append(reinterpret_cast<const char *>(&ps), 2);
        s.append(reinterpret_cast<const char *>(&pe), 2);
        s.push_back((char)t0);
        s.push_back((char)t1);
        s.push_back('|');
    }
    std::string key() const {
        std::string s;
        s.reserve(48);
        key(s);
        return s;
    }
};

enum { ND_TERM = 0, ND_DELETED = 1, ND_START = 2, ND_END = 3 };
struct ENode {
    int kind = ND_DELETED;
    ELocated term;
    std::vector<uint16_t> pred, succ;  // ascending
};
struct EGraph {
    uint16_t root = 0, end = 1;
    std::vector<ENode> nodes;
};

inline void sorted_insert(std::vector<uint16_t> &v, uint16_t x) {
    auto it = std::lower_bound(v.begin(), v.end(), x);
    if (it == v.end() || *it != x) v.insert(it, x);
}
inline void sorted_remove(std::vector<uint16_t> &v, uint16_t x) {
    auto it = std::lower_bound(v.begin(), v.end(), x);
    if (it != v.end() && *it == x) v.erase(it);
}

// score kinds = b200_score_kind
struct EScore {
    uint8_t kind;
    uint32_t rank, max_rank;
    float sim;
};

}  // namespace b200
