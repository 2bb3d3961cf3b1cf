// Banded restricted Damerau-Levenshtein (OSA) distance and the character-class filter, shared by term derivation (kernels.cu, over
// bytes) and facet search (facet_search.cu, over Unicode scalar values).
#pragma once
#include <cstdint>

namespace b200 {

// Returns min(distance, k+1), k <= 2.  prefix: min over prefixes of w.
template <class C>
__device__ __forceinline__ int banded_osa(const C *q, int m, const C *w, int n, int k, bool prefix) {
    const int INF = k + 1;
    // column j holds D[i][j] for i = j + b - k, b in [0, 2k]
    int c2[5], c1[5], c0[5];
#pragma unroll
    for (int b = 0; b < 5; b++) {
        int i = b - k;
        c1[b] = (b <= 2 * k && i >= 0 && i <= m) ? (i < INF ? i : INF) : INF;
        c2[b] = INF;
    }
    int best = INF;
    if (prefix && m <= k) best = m;  // empty prefix (never happens for words long enough to have typos)
    int jmax = n;
    if (jmax > m + k) jmax = m + k;
    if (!prefix && (n > m + k || n < m - k)) return INF;
    if (prefix && n < m - k) return INF;
    for (int j = 1; j <= jmax; j++) {
        C wc = w[j - 1];
        C wp = j > 1 ? w[j - 2] : 0;
        int rowmin = INF;
#pragma unroll
        for (int b = 0; b < 5; b++) {
            int v = INF;
            if (b <= 2 * k) {
                int i = j + b - k;
                if (i >= 0 && i <= m) {
                    if (i == 0)
                        v = j;
                    else {
                        int del = (b > 0) ? c0[b - 1] + 1 : INF;              // D[i-1][j] + 1
                        int ins = (b < 2 * k) ? c1[b + 1] + 1 : INF;          // D[i][j-1] + 1
                        int sub = c1[b] + (q[i - 1] != wc ? 1 : 0);           // D[i-1][j-1] + cost
                        v = min(del, min(ins, sub));
                        if (i > 1 && j > 1 && q[i - 1] == wp && q[i - 2] == wc) v = min(v, c2[b] + 1);  // D[i-2][j-2] + 1
                    }
                    if (v > INF) v = INF;
                }
            }
            c0[b] = v;
            rowmin = min(rowmin, v);
        }
        if (prefix) {
            int b = m - j + k;
            if (b >= 0 && b <= 2 * k) best = min(best, c0[b]);
        }
#pragma unroll
        for (int b = 0; b < 5; b++) {
            c2[b] = c1[b];
            c1[b] = c0[b];
        }
        if (rowmin >= INF && !prefix) {
            // both this and (via c2) an earlier column may still matter for a transposition; stop only when two columns are dead
            int m2 = INF;
#pragma unroll
            for (int b = 0; b < 5; b++) m2 = min(m2, c2[b]);
            if (m2 >= INF) return INF;
        }
    }
    if (prefix) return best;
    int b = m - n + k;
    return (b >= 0 && b <= 2 * k) ? c1[b] : INF;
}

// Character-class signature: bit (c & 31) for every character.  If OSA(q, w) <= k then at most k classes of q are missing from w
// (every edit removes at most one class; a transposition none), and — outside prefix mode — vice versa.  Sound with collisions.
template <class C>
__device__ __forceinline__ uint32_t char_signature(const C *s, int n) {
    uint32_t m = 0;
    for (int i = 0; i < n; i++) m |= 1u << (s[i] & 31);
    return m;
}

}  // namespace b200
