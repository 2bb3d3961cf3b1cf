"""GPU parity tests (run with -m gpu on an H100): the CUDA path through the C ABI vs the CPU oracle and the
reference goldens.  Integer/bit work must match exactly; vector scores within 1e-4 relative."""
import numpy as np
import pytest

from tests.helpers import image_from_corpus, load_goldens, synthetic_image
from tests.test_oracle_goldens import check_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mb():
    import meilisearch_b200 as m

    m.load_library()
    return m


@pytest.fixture(scope="module")
def synth():
    return synthetic_image(60000, 25000, seed=11)


def _edit(rng, w):
    k = rng.integers(4)
    if len(w) < 2:
        k = 1
    p = int(rng.integers(len(w)))
    c = chr(ord("a") + int(rng.integers(26)))
    if k == 0:
        return w[:p] + c + w[p + 1:]
    if k == 1:
        return w[:p] + c + w[p:]
    if k == 2:
        return w[:p] + w[p + 1:]
    p = min(p, len(w) - 2)
    return w[:p] + w[p + 1] + w[p] + w[p + 2:]


def test_derive_matches_oracle(mb, synth):
    from oracle.pyoracle import OracleIndex

    rng = np.random.default_rng(5)
    words = []
    for _ in range(300):
        w = synth.word(int(rng.integers(synth.n_words)))
        for _ in range(int(rng.integers(3))):
            w = _edit(rng, w) or w
        if len(w) >= 3:
            words.append(w)
    words += ["a" * 5, "zzzzzzzzz", synth.word(0), synth.word(synth.n_words - 1)]
    ix = mb.Index(synth)
    o = OracleIndex(synth)
    for max_typo in (1, 2):
        for is_prefix in (0, 1):
            got = ix.derive(words, [max_typo] * len(words), [is_prefix] * len(words))
            for w, (g1, g2) in zip(words, got):
                o1, o2 = o.derive(w, max_typo, is_prefix)
                assert list(g1) == list(o1), (w, max_typo, is_prefix, "one")
                assert list(g2) == list(o2), (w, max_typo, is_prefix, "two")


def test_derive_caps(mb):
    # MAX_ONE_TYPO_COUNT / MAX_TWO_TYPOS_COUNT and the first-letter quirk (limits.rs:7-9, compute_derivations.rs:129-166)
    from corpus.pyindexgen import IndexImage
    from oracle.pyoracle import OracleIndex

    img = IndexImage(1)
    base = "abcdefghij"
    docs = []
    for a in "abcdefghijklmnopqrstuvwxyz":
        for b in "abcdefghijklmnopqrstuvwxyz":
            docs.append(base[:4] + a + base[5:8] + b + base[9:])   # <= 2 substitutions, same first letter
        docs.append(a + base[1:])                                   # first-letter substitutions
    img.add_text(0, 0, " ".join(docs))
    img.build()
    ix, o = mb.Index(img), OracleIndex(img)
    for w, p in ((base, 0), (base, 1), ("xbcdefghij", 0)):
        (g1, g2), = ix.derive([w], [2], [p])
        o1, o2 = o.derive(w, 2, p)
        assert list(g1) == list(o1) and list(g2) == list(o2)
        assert len(o1) <= 150 and len(o2) <= 50


def test_nns_matches_oracle(mb, synth):
    from oracle.pyoracle import OracleIndex

    rng = np.random.default_rng(1)
    n, d = 30000, 768
    emb = rng.standard_normal((n, d)).astype(np.float32)
    emb[100] = emb[50]          # an exact tie: equal distances must come out in docid order
    docids = rng.permutation(n).astype(np.uint32)
    ix = mb.Index(synth)
    ix.set_embeddings(emb, docids)
    o = OracleIndex(synth)
    o.set_embeddings(emb.astype(np.float16).astype(np.float32), docids)   # the oracle scans the same fp16-rounded rows
    q = rng.standard_normal((11, d)).astype(np.float32)
    q[3] = emb[50]
    cand = np.zeros((n + 63) // 64, np.uint64)
    keep = rng.random(n) < 0.1
    for doc in np.nonzero(keep)[0]:
        cand[doc >> 6] |= np.uint64(1) << np.uint64(doc & 63)
    for cw in (None, cand):
        ids, dist, cnt = ix.nns_by_vector(q, 100, cw)
        for i in range(len(q)):
            oid, od = o.nns(q[i], 100, cw)
            assert cnt[i] == len(oid)
            # 1e-4 relative on the similarity score (north_star); ids equal except where oracle scores tie within tolerance
            assert np.allclose(1 - dist[i, : cnt[i]], 1 - od, rtol=1e-4, atol=1e-6)
            diff = [k for k in range(len(oid)) if ids[i, k] != oid[k]]
            for k in diff:
                assert abs(od[k] - dist[i, k]) <= 1e-4 * max(1 - od[k], 1e-3)


def test_nns_tensor_core_batch_matches_oracle(mb, synth, monkeypatch):
    """The batched vector stage (wgmma GEMM + fused top-k) against the oracle and against the GEMV scan."""
    from oracle.pyoracle import OracleIndex

    rng = np.random.default_rng(7)
    for n, d, nq, k in ((20011, 768, 150, 100), (5000, 128, 40, 7), (300, 64, 17, 128)):
        emb = rng.standard_normal((n, d)).astype(np.float32)
        emb[100] = emb[50]
        docids = rng.permutation(n).astype(np.uint32)
        ix = mb.Index(synth)
        ix.set_embeddings(emb, docids)
        o = OracleIndex(synth)
        o.set_embeddings(emb.astype(np.float16).astype(np.float32), docids)
        q = rng.standard_normal((nq, d)).astype(np.float32)
        q[3] = emb[50]
        cand = np.zeros((n + 63) // 64, np.uint64)
        for doc in np.nonzero(rng.random(n) < 0.2)[0]:
            cand[doc >> 6] |= np.uint64(1) << np.uint64(doc & 63)
        for cw in (None, cand):
            monkeypatch.setenv("B200_VEC_GEMM", "1")
            ix.reset_stats()
            ids, dist, cnt = ix.nns_by_vector(q, k, cw)
            assert ix.stats()["kernels"]["vec_gemm_topk"]["count"] >= 1
            monkeypatch.setenv("B200_VEC_GEMM", "0")
            ids2, dist2, cnt2 = ix.nns_by_vector(q, k, cw)
            assert (cnt == cnt2).all()
            # queries are rounded to fp16 for the tensor cores: 1e-4 relative on the similarity (north_star)
            for i in range(nq):
                oid, od = o.nns(q[i], k, cw)
                assert cnt[i] == len(oid)
                assert np.allclose(1 - dist[i, : cnt[i]], 1 - od, rtol=1e-4, atol=2e-5), (n, d, i)
                assert (np.diff(dist[i, : cnt[i]]) >= 0).all()
                assert len(set(ids[i, : cnt[i]].tolist())) == cnt[i]
                for j in np.nonzero(ids[i, : cnt[i]] != oid)[0]:
                    assert abs(od[j] - dist[i, j]) <= 1e-4 * max(1 - od[j], 1e-3) + 2e-5
            assert np.allclose(dist[:, : cnt.min()], dist2[:, : cnt.min()], rtol=1e-4, atol=2e-5)


G = load_goldens()


def test_reference_goldens_on_gpu(mb):
    """Every golden extracted from the reference's ranking-rule tests (docids and, where snapshotted, ScoreDetails) through the CUDA path."""
    ran = 0
    images = {}
    for case in G["cases"]:
        s = case["settings"]
        ci = case["index"]
        if ci not in images:
            images[ci] = image_from_corpus(G["corpora"][ci])
        img = images[ci]
        ix = mb.Index(img, criteria=s.get("criteria"), authorize_typos=s.get("authorize_typos", True), one_typo=s.get("one_typo", 5),
                      two_typos=s.get("two_typos", 9), exact_words=s.get("exact_words", []), synonyms=s.get("synonyms"), weights=s.get("weights"))
        search = (ix.search().query(mb.TokenBatch([case["query"]], img.stop_words)).terms_matching_strategy(case["tms"])
                  .scoring_strategy(case["scoring"]).limit(max(case["limit"], 1)).offset(case["offset"]))
        if case.get("threshold") is not None:
            search = search.ranking_score_threshold(case["threshold"])
        res = search.execute()
        assert res.status[0] == 0
        check_golden(case, res.ids(0), res.scores(0), int(res.n_candidates[0]))
        ix.close()
        ran += 1
    assert ran == len(G["cases"])


@pytest.mark.parametrize("tms,scoring", [("last", "detailed"), ("last", "skip"), ("all", "detailed"), ("frequency", "detailed")])
def test_keyword_batch_matches_oracle(mb, synth, tms, scoring):
    from oracle.pyoracle import OracleIndex

    queries = synth.synthetic_queries(300, seed=21) + ["", "   ", synth.word(5), "zzzzqqqq xxxxyyyy"]
    tokens = mb.TokenBatch(queries)
    ix = mb.Index(synth)
    got = ix.search().query(tokens).terms_matching_strategy(tms).scoring_strategy(scoring).execute()
    want = OracleIndex(synth).search_batch(tokens, tms=tms, scoring=scoring, n_threads=8)
    for q in range(len(queries)):
        assert got.status[q] == 0
        assert got.ids(q) == want.ids(q), (queries[q], tms, scoring)
        assert got.scores(q) == want.scores(q), (queries[q], tms, scoring)
        assert int(got.n_candidates[q]) == int(want.n_candidates[q]), queries[q]


def test_offset_limit(mb, synth):
    from oracle.pyoracle import OracleIndex

    queries = synth.synthetic_queries(40, seed=4, with_typos=False)
    tokens = mb.TokenBatch(queries)
    ix, o = mb.Index(synth), OracleIndex(synth)
    for off, lim in ((0, 5), (3, 7), (15, 20), (0, 100)):
        got = ix.search().query(tokens).offset(off).limit(lim).execute()
        want = o.search_batch(tokens, offset=off, limit=lim)
        for q in range(len(queries)):
            assert got.ids(q) == want.ids(q), (queries[q], off, lim)


def test_two_fields_full_stack(mb):
    from oracle.pyoracle import OracleIndex

    img = synthetic_image(8000, 3000, seed=3, n_fields=2)
    queries = img.synthetic_queries(120, seed=8)
    tokens = mb.TokenBatch(queries)
    crit = ["words", "typo", "proximity", "attribute", "exactness"]
    ix, o = mb.Index(img, criteria=crit), OracleIndex(img, criteria=crit)
    got = ix.search().query(tokens).scoring_strategy("detailed").execute()
    want = o.search_batch(tokens, scoring="detailed")
    for q in range(len(queries)):
        assert got.ids(q) == want.ids(q), queries[q]
        assert got.scores(q) == want.scores(q), queries[q]


def test_hybrid_matches_oracle(mb, synth):
    from oracle.pyoracle import OracleIndex

    rng = np.random.default_rng(2)
    n, d = synth.n_docs, 64
    emb = rng.standard_normal((n, d)).astype(np.float16).astype(np.float32)
    queries = synth.synthetic_queries(50, seed=9)
    tokens = mb.TokenBatch(queries)
    vec = rng.standard_normal((len(queries), d)).astype(np.float16).astype(np.float32)
    ix, o = mb.Index(synth), OracleIndex(synth)
    ix.set_embeddings(emb)
    o.set_embeddings(emb)
    for ratio in (0.1, 0.5, 0.9):
        got = ix.search().query(tokens).semantic(vec).execute_hybrid(ratio)
        want = o.search_batch(tokens, vectors=vec, hybrid=True, semantic_ratio=ratio)
        for q in range(len(queries)):
            assert got.ids(q) == want.ids(q), (queries[q], ratio)
            assert int(got.semantic_hit_count[q]) == int(want.semantic_hits[q])


def test_phrases_negatives_match_oracle(mb, synth):
    from oracle.pyoracle import OracleIndex

    base = synth.synthetic_queries(60, seed=33, with_typos=False)
    queries = []
    for i, q in enumerate(base):
        w = q.split()
        if i % 3 == 0 and len(w) >= 2:
            queries.append('"' + " ".join(w[:2]) + '" ' + " ".join(w[2:]))
        elif i % 3 == 1 and len(w) >= 2:
            queries.append(" ".join(w[:-1]) + " -" + w[-1])
        else:
            queries.append(w[0] + ' "' + " ".join(w[1:]) + '"')
    tokens = mb.TokenBatch(queries)
    ix, o = mb.Index(synth), OracleIndex(synth)
    got = ix.search().query(tokens).scoring_strategy("detailed").execute()
    want = o.search_batch(tokens, scoring="detailed", n_threads=8)
    for q in range(len(queries)):
        assert got.status[q] == 0
        assert got.ids(q) == want.ids(q), queries[q]
        assert got.scores(q) == want.scores(q), queries[q]


def test_only_negative_terms_is_a_placeholder_search_over_the_rest(mb, synth):
    """search/new/mod.rs:719-737: no positive term -> placeholder search over universe minus the negative words' / phrases' documents"""
    from oracle.pyoracle import OracleIndex

    qs = synth.synthetic_queries(6, seed=31, with_typos=False)
    w = [q.split() for q in qs]
    queries = ["-" + w[0][0], "-" + w[1][0] + " -" + w[2][0], '-"' + " ".join(w[3][:2]) + '"', "- " + w[4][0], "-" + w[5][0] + " -zzzzqqqqxxxx"]
    tokens = mb.TokenBatch(queries)
    ix, o = mb.Index(synth), OracleIndex(synth)
    for offset, limit in ((0, 20), (7, 5)):
        got = ix.search().query(tokens).scoring_strategy("detailed").offset(offset).limit(limit).with_candidates().execute()
        want = o.search_batch(tokens, scoring="detailed", offset=offset, limit=limit, n_threads=4)
        for q in range(len(queries)):
            assert got.status[q] == 0
            assert got.ids(q) == want.ids(q), queries[q]
            assert got.scores(q) == want.scores(q), queries[q]
            assert int(got.n_candidates[q]) == int(want.n_candidates[q]), queries[q]
            assert bool(got.used_negative_operator[q]) == bool(want.used_negative_operator[q])
            assert int(np.bitwise_count(got.candidates[q]).sum()) == int(want.n_candidates[q])


def test_unsupported_is_reported_not_faked(mb, synth):
    ix = mb.Index(synth)
    w = synth.synthetic_queries(1, seed=5, with_typos=False)[0].split()[0]
    long_query = " ".join(synth.synthetic_queries(8, seed=6, with_typos=False))
    assert len(long_query.split()) > 12
    res = ix.search().query(["-" + w, "plain", long_query]).words_limit(20).execute()
    assert res.status[0] == 0
    assert res.status[1] == 0
    assert res.status[2] == -4 and res.n_hits[2] == 0
    # with the default words_limit (10) the same long query is in scope
    assert ix.search().query([long_query]).execute().status[0] == 0


def test_large_universe_matches_oracle(mb):
    """More than 8192 x 64 documents: universes span several compaction segments and the emit scan runs many rounds."""
    from oracle.pyoracle import OracleIndex
    from tests.helpers import synthetic_image

    img = synthetic_image(700_000, 60_000, seed=0xB201)
    queries = img.synthetic_queries(48, seed=9)
    tokens = mb.TokenBatch(queries)
    got = mb.Index(img).search().query(tokens).scoring_strategy("detailed").execute()
    want = OracleIndex(img).search_batch(tokens, scoring="detailed", n_threads=8)
    for q in range(len(queries)):
        assert got.status[q] == 0
        assert got.ids(q) == want.ids(q), queries[q]
        assert got.scores(q) == want.scores(q), queries[q]
        assert int(got.n_candidates[q]) == int(want.n_candidates[q])


def test_union_postings_matches_decoded_lists(mb, synth):
    """S2 (b200_union_postings): OR of posting lists AND universe, against the CBO values decoded by the oracle's codec."""
    check_union_postings(mb.Index(synth), synth)


def check_union_postings(ix, synth):
    from oracle.pyoracle import cbo_decode

    rng = np.random.default_rng(3)
    n_words = (synth.n_docs + 63) // 64
    for db in (0, 4, 5):  # word_docids, word_pair_proximity_docids, word_position_docids
        view = synth.dbs[db]
        n_keys = int(view.n_keys)
        # a mix of the longest lists (dense on the device) and random ones
        lens = np.diff(np.asarray(view.val_offsets))
        keys = np.unique(np.concatenate([np.argsort(lens)[-3:], rng.integers(0, n_keys, 40)])).astype(np.uint32)
        want = np.zeros(n_words, np.uint64)
        for k in keys:
            ids = cbo_decode(view.val(int(k)))
            np.bitwise_or.at(want, ids >> 6, np.uint64(1) << (ids & 63).astype(np.uint64))
        got = ix.union_postings(db, keys)
        assert np.array_equal(got, want), db
        universe = rng.integers(0, 2**63, n_words, dtype=np.uint64)
        got_u = ix.union_postings(db, keys, universe)
        assert np.array_equal(got_u, want & universe), db
    assert np.array_equal(ix.union_postings(0, np.zeros(0, np.uint32)), np.zeros(n_words, np.uint64))


# ------------------------------------------------------------------------------------------------ round 2: S0 boundary features
def _same(got, want, q, scores=True, ctx=None):
    assert got.status[q] == 0, ctx
    assert got.ids(q) == want.ids(q), ctx
    if scores:
        assert got.scores(q) == want.scores(q), ctx
    assert int(got.n_candidates[q]) == int(want.n_candidates[q]), ctx


def test_cutoff_goldens_on_gpu(mb):
    """Deadline::with_stop_after(n) known answers of the reference (search/new/tests/cutoff.rs:100-407) through the C ABI."""
    from tests.test_cutoff_goldens import CUTOFF_CASES, cutoff_image, global_score

    ix = mb.Index(cutoff_image(), criteria=["words", "typo"])
    for stop_after, (ids, scores, degraded) in CUTOFF_CASES.items():
        r = ix.search().query(["hello puppy kefir"]).scoring_strategy("detailed").limit(4).deadline(stop_after=stop_after).execute()
        assert r.ids(0) == ids, stop_after
        assert [round(global_score(s), 4) for s in r.scores(0)] == scores, stop_after
        assert bool(r.degraded[0]) == degraded, stop_after
    # cutoff.rs:74-98 degraded_search_cannot_skip_filter
    r = ix.search().query(["hello puppy kefir"]).limit(100).deadline(stop_after=0).universes([np.array([0b00011], np.uint64)]).with_candidates().execute()
    assert r.ids(0) == [0, 1] and int(r.n_candidates[0]) == 2 and r.degraded[0] == 1
    assert int(r.candidates[0, 0]) == 0b00011
    # a zero time budget degrades too (cutoff.rs:58-72)
    assert ix.search().query(["hello puppy kefir"]).limit(3).deadline(budget_ms=0).execute().degraded[0] == 1


def _random_universes(rng, n_docs, n_queries):
    words = (n_docs + 63) // 64
    shared = rng.integers(0, 2**63, words, dtype=np.uint64) & rng.integers(0, 2**63, words, dtype=np.uint64)
    sparse = np.zeros(words, np.uint64)
    for d in rng.integers(0, n_docs, 300):
        sparse[d >> 6] |= np.uint64(1) << np.uint64(d & 63)
    out = []
    for q in range(n_queries):
        out.append([None, shared, sparse, rng.integers(0, 2**63, words, dtype=np.uint64)][q % 4])
    return out


def test_filtered_universe_matches_oracle(mb, synth):
    """S0 `universes` (filtered_universe, search/new/mod.rs:719): keyword, placeholder, semantic and hybrid searches"""
    from oracle.pyoracle import OracleIndex

    rng = np.random.default_rng(12)
    queries = synth.synthetic_queries(80, seed=41) + ["", synth.word(7)]
    tokens = mb.TokenBatch(queries)
    unis = _random_universes(rng, synth.n_docs, len(queries))
    ix, o = mb.Index(synth), OracleIndex(synth)
    for scoring in ("detailed", "skip"):
        got = ix.search().query(tokens).scoring_strategy(scoring).universes(unis).with_candidates().execute()
        want = o.search_batch(tokens, scoring=scoring, universes=unis, n_threads=8)
        for q in range(len(queries)):
            _same(got, want, q, ctx=(queries[q], q % 4))
            cand = got.candidates[q]
            assert int(sum(bin(int(w)).count("1") for w in cand)) == int(want.n_candidates[q])
            if unis[q] is not None:
                assert not (cand & ~unis[q]).any()
            for d in got.ids(q):
                assert (int(cand[d >> 6]) >> (d & 63)) & 1
    # vector side
    d = 64
    emb = rng.standard_normal((synth.n_docs, d)).astype(np.float16).astype(np.float32)
    ix.set_embeddings(emb)
    o.set_embeddings(emb)
    vec = rng.standard_normal((len(queries), d)).astype(np.float16).astype(np.float32)
    got = ix.search().semantic(vec).universes(unis).limit(10).execute()
    want = o.search_batch(mb.TokenBatch([""] * len(queries)), vectors=vec, vector_only=True, universes=unis, limit=10, n_threads=8)
    for q in range(len(queries)):
        assert got.ids(q) == want.ids(q), q
        assert int(got.n_candidates[q]) == int(want.n_candidates[q])
    got = ix.search().query(tokens).semantic(vec).universes(unis).execute_hybrid(0.5)
    want = o.search_batch(tokens, vectors=vec, hybrid=True, semantic_ratio=0.5, universes=unis, n_threads=8)
    for q in range(len(queries)):
        assert got.ids(q) == want.ids(q), (queries[q], q % 4)


@pytest.mark.parametrize("threshold", [0.2, 0.55, 0.8, 0.97])
def test_ranking_score_threshold_matches_oracle(mb, synth, threshold):
    from oracle.pyoracle import OracleIndex

    queries = synth.synthetic_queries(120, seed=51)
    tokens = mb.TokenBatch(queries)
    got = mb.Index(synth).search().query(tokens).scoring_strategy("detailed").ranking_score_threshold(threshold).execute()
    want = OracleIndex(synth).search_batch(tokens, scoring="detailed", threshold=threshold, n_threads=8)
    for q in range(len(queries)):
        _same(got, want, q, ctx=(queries[q], threshold))


@pytest.mark.parametrize("stop_after", [0, 1, 2, 3])
def test_deadline_stop_after_matches_oracle(mb, synth, stop_after):
    """Deadline::with_stop_after(n) on a synthetic corpus.  Early polls fall into the Words / Typo rules, where the engine's bucket
    requests map one to one onto the reference's; deeper in the stack the reference also polls for costs that its skip
    constraints make infeasible (DESIGN.md §3), so larger n are checked through invariants below."""
    from oracle.pyoracle import OracleIndex

    queries = synth.synthetic_queries(100, seed=61)
    tokens = mb.TokenBatch(queries)
    for scoring in ("detailed", "skip"):
        got = mb.Index(synth).search().query(tokens).scoring_strategy(scoring).deadline(stop_after=stop_after).execute()
        want = OracleIndex(synth).search_batch(tokens, scoring=scoring, stop_after=stop_after, n_threads=8)
        for q in range(len(queries)):
            _same(got, want, q, ctx=(queries[q], stop_after, scoring))
            assert int(got.degraded[q]) == int(want.degraded[q]), (queries[q], stop_after)


@pytest.mark.parametrize("stop_after", [5, 8, 13, 40])
def test_deadline_invariants(mb, synth, stop_after):
    """a degraded result returns every candidate it has room for, the sorted prefix equals the undegraded search's, and the
    unsorted tail carries a Skipped score (bucket_sort.rs:206-264)"""
    queries = synth.synthetic_queries(100, seed=62)
    tokens = mb.TokenBatch(queries)
    ix = mb.Index(synth)
    full = ix.search().query(tokens).scoring_strategy("detailed").execute()
    got = ix.search().query(tokens).scoring_strategy("detailed").deadline(stop_after=stop_after).with_candidates().execute()
    for q in range(len(queries)):
        assert got.status[q] == 0
        ids = got.ids(q)
        assert len(set(ids)) == len(ids)
        assert int(got.n_candidates[q]) == int(full.n_candidates[q])
        assert len(ids) == min(20, int(got.n_candidates[q]))
        for d in ids:
            assert (int(got.candidates[q, d >> 6]) >> (d & 63)) & 1
        skipped = [any(s[0] == "skipped" for s in row) for row in got.scores(q)]
        if not got.degraded[q]:
            assert ids == full.ids(q) and not any(skipped)
            continue
        k = skipped.index(True) if any(skipped) else len(ids)
        assert all(skipped[k:])                                  # once the dump starts, everything after it is dumped
        assert ids[:k] == full.ids(q)[:k]                        # what was ranked before the deadline is the true prefix
        assert got.scores(q)[:k] == full.scores(q)[:k]


def test_used_negative_operator(mb, synth):
    w = synth.synthetic_queries(1, seed=5, with_typos=False)[0].split()
    r = mb.Index(synth).search().query([w[0] + " -" + w[-1], w[0]]).execute()
    assert list(r.used_negative_operator) == [1, 0]


def test_count_goldens_on_gpu(mb):
    """typo_tolerance.rs:18-357 hit counts (exact words, exact attributes, min word length) through the CUDA path"""
    ran = 0
    for case in G.get("count_cases", []):
        img = image_from_corpus(G["corpora"][case["index"]])
        s = case["settings"]
        ix = mb.Index(img, criteria=s.get("criteria"), authorize_typos=s.get("authorize_typos", True), one_typo=s.get("one_typo", 5),
                      two_typos=s.get("two_typos", 9), exact_words=s.get("exact_words", []), synonyms=s.get("synonyms"))
        res = ix.search().query(mb.TokenBatch([case["query"]], img.stop_words)).terms_matching_strategy(case.get("tms", "last")).limit(max(case.get("limit", 20), 1)).execute()
        assert res.status[0] == 0
        assert int(res.n_hits[0]) == case["expected_count"], case["source"]
        ix.close()
        ran += 1
    assert ran == len(G.get("count_cases", []))


def test_distribution_shift_matches_oracle(mb, synth):
    """b200_stage_distribution (vector/distribution.rs:103-130) on semantic scores"""
    from oracle.pyoracle import OracleIndex

    rng = np.random.default_rng(3)
    d = 64
    emb = rng.standard_normal((5000, d)).astype(np.float16).astype(np.float32)
    ix, o = mb.Index(synth), OracleIndex(synth)
    ix.set_embeddings(emb, distribution=(0.6, 0.05))
    o.set_embeddings(emb, distribution=(0.6, 0.05))
    vec = rng.standard_normal((9, d)).astype(np.float16).astype(np.float32)
    got = ix.search().semantic(vec).scoring_strategy("detailed").limit(15).execute()
    want = o.search_batch(mb.TokenBatch([""] * 9), vectors=vec, vector_only=True, scoring="detailed", limit=15)
    for q in range(9):
        assert got.ids(q) == want.ids(q)
        gs = [s[0][1] for s in got.scores(q)]
        ws = [s[0][1] for s in want.scores(q)]
        assert np.allclose(gs, ws, rtol=1e-4, atol=1e-6)
        assert all(0 < x <= 1 for x in gs)


def test_prefix_search_disabled_matches_oracle(mb, synth):
    from oracle.pyoracle import OracleIndex

    queries = synth.synthetic_queries(80, seed=71)
    tokens = mb.TokenBatch(queries)
    got = mb.Index(synth, prefix_search=False).search().query(tokens).scoring_strategy("detailed").execute()
    want = OracleIndex(synth, prefix_search=False).search_batch(tokens, scoring="detailed", n_threads=8)
    for q in range(len(queries)):
        _same(got, want, q, ctx=queries[q])


def test_nns_many_ties_and_duplicate_docids(mb, synth):
    """more equal-distance rows than the selection's tie buffer, and several embeddings per document; with docids in row order
    and permuted (then row order says nothing about which tied rows have the smallest docids)"""
    from oracle.pyoracle import OracleIndex

    rng = np.random.default_rng(4)
    n, d = 6000, 64
    emb = rng.standard_normal((n, d)).astype(np.float16).astype(np.float32)
    emb[1000:3500] = emb[999]                      # 2501 identical rows: a tie far longer than any top-k
    ix, o = mb.Index(synth), OracleIndex(synth)
    q = np.stack([emb[999], emb[150], rng.standard_normal(d).astype(np.float32)])
    for layout in ("row order", "permuted"):
        docids = np.arange(n, dtype=np.uint32) if layout == "row order" else rng.permutation(n).astype(np.uint32)
        docids[4000:4200] = docids[100:300]        # 200 documents own two embeddings each
        ix.set_embeddings(emb, docids)
        o.set_embeddings(emb, docids)
        for k in (10, 100):
            ids, dist, cnt = ix.nns_by_vector(q, k)
            for i in range(len(q)):
                oid, od = o.nns(q[i], k)
                assert cnt[i] == len(oid)
                assert np.allclose(dist[i, : cnt[i]], od, rtol=1e-4, atol=2e-6)
                # inside a run of equal distances the order is ascending docid on both sides
                assert list(ids[i, : cnt[i]]) == list(oid), (layout, i, k)


def test_path_table_growth(mb):
    """More distinct surviving paths in one rule step than the 4096-slot table holds: the step is rerun with a larger table"""
    from corpus.pyindexgen import IndexImage
    from oracle.pyoracle import OracleIndex

    # 4 query words, each document holds them at a different combination of positions: the Position rule (about 10 costs per
    # term) sees thousands of distinct (position, position, position, position) paths in its first bucket's universe
    rng = np.random.default_rng(8)
    img = IndexImage(1)
    words = ["alpha", "bravo", "charlie", "delta"]
    filler = ["f%03d" % i for i in range(200)]
    for doc in range(9000):
        toks = [filler[int(x)] for x in rng.integers(0, 200, 40)]
        for w, p in zip(words, sorted(rng.choice(40, 4, replace=False))):
            toks[int(p)] = w
        img.add_text(doc, 0, " ".join(toks))
    img.build()
    crit = ["words", "wordPosition", "exactness"]
    queries = [" ".join(words)]
    tokens = mb.TokenBatch(queries)
    got = mb.Index(img, criteria=crit).search().query(tokens).scoring_strategy("detailed").limit(50).execute()
    want = OracleIndex(img, criteria=crit).search_batch(tokens, scoring="detailed", limit=50)
    _same(got, want, 0)


def test_partial_embeddings_last_bucket(mb, synth):
    """fewer embedded documents than offset + limit: the rest of the universe follows in docid order without a similarity
    (vector_sort.rs:128-160)"""
    from oracle.pyoracle import OracleIndex

    rng = np.random.default_rng(6)
    d = 64
    emb = rng.standard_normal((7, d)).astype(np.float16).astype(np.float32)
    docids = np.array([5, 900, 17, 4000, 33, 2, 12000], np.uint32)
    ix, o = mb.Index(synth), OracleIndex(synth)
    ix.set_embeddings(emb, docids)
    o.set_embeddings(emb, docids)
    vec = rng.standard_normal((3, d)).astype(np.float16).astype(np.float32)
    got = ix.search().semantic(vec).scoring_strategy("detailed").limit(12).execute()
    want = o.search_batch(mb.TokenBatch([""] * 3), vectors=vec, vector_only=True, scoring="detailed", limit=12)
    for q in range(3):
        assert got.ids(q) == want.ids(q)
        assert [s[0][1] is None for s in got.scores(q)] == [s[0][1] is None for s in want.scores(q)]


def test_hybrid_goldens_on_gpu(mb):
    """hybrid.rs:195-430 `simple_search` (hit order, _rankingScore, semanticHitCount at semanticRatio 0.2 / 0.5 / 0.8) through the C ABI"""
    from tests.test_hybrid_goldens import HYBRID_CASES, check, embeddings, hybrid_image

    ix = mb.Index(hybrid_image(), weights=[0, 0, 0])
    ix.set_embeddings(embeddings())
    for ratio in HYBRID_CASES:
        r = ix.search().query(["Captain"]).semantic(np.array([[1.0, 1.0]], np.float32)).scoring_strategy("detailed").execute_hybrid(ratio)
        check(r.ids(0), r.scores(0), int(r.semantic_hit_count[0]), ratio)


def test_hybrid_more_goldens_on_gpu(mb):
    """the other known answers of hybrid.rs (limit_offset, distribution_shift, highlighter, single_document, query_combination:
    tests/test_hybrid_goldens.py MORE_CASES) through the C ABI, routed as the HTTP layer routes them"""
    from tests.test_hybrid_goldens import MORE_CASES, check_more, embeddings, more_image, route

    for case in MORE_CASES:
        _, q, vector, ratio, offset, limit, distribution, n_docs, _, _, _ = case
        ix = mb.Index(more_image(n_docs), weights=[0, 0, 0])
        ix.set_embeddings(embeddings()[:n_docs], distribution=distribution)
        kind = route(q, vector, ratio)
        vec = None if vector is None else np.array([vector], np.float32)
        s = ix.search().scoring_strategy("detailed").offset(offset).limit(limit)
        if kind == "keyword":
            r = s.query([q or ""]).execute()
            sem = None
        elif kind == "semantic":
            r = s.semantic(vec).execute()
            sem = len(r.ids(0))
        else:
            r = s.query([q]).semantic(vec).execute_hybrid(ratio)
            sem = int(r.semantic_hit_count[0])
        check_more(case, r.ids(0), r.scores(0), sem)
        ix.close()


# ------------------------------------------------------------------------------------------------ round 2: S1 / S2 seams
def _bits(words):
    out = []
    for w, v in enumerate(words):
        v = int(v)
        while v:
            b = (v & -v).bit_length() - 1
            out.append(w * 64 + b)
            v &= v - 1
    return out


def test_rule_seam_matches_oracle_buckets(mb):
    """S1 (b200_graph_from_tokens / b200_rule_start / _next / _end): the first two rules are driven bucket by bucket by the
    caller, as bucket_sort does (bucket_sort.rs:123,266,323), and every bucket must hold exactly the documents the oracle scores
    with that rule's rank (ScoringStrategy::Detailed with a limit covering every candidate)."""
    from oracle.pyoracle import OracleIndex

    img = synthetic_image(4000, 1500, seed=19)
    ix, o = mb.Index(img), OracleIndex(img)
    queries = img.synthetic_queries(25, seed=3)
    for query in queries:
        want = o.search_batch(mb.TokenBatch([query]), scoring="detailed", limit=4000)
        by_doc = {d: s for d, s in zip(want.ids(0), want.scores(0))}
        # the universe bucket_sort starts from: the documents of the maximally reduced query graph = the oracle's candidates
        universe = np.zeros((img.n_docs + 63) // 64, np.uint64)
        for d in by_doc:
            universe[d >> 6] |= np.uint64(1) << np.uint64(d & 63)
        assert len(by_doc) == int(want.n_candidates[0])
        g = ix.query_graph(query)
        seen = set()
        for cand, rank, mx, child in g.rule("words", universe):
            docs = _bits(cand)
            for d in docs:
                assert by_doc[d][0] == ("words", rank, mx), (query, d)
            assert not (seen & set(docs))
            seen |= set(docs)
            if child is None:
                assert not docs
                continue
            seen2 = set()
            for cand2, rank2, mx2, child2 in child.rule("typo", cand):
                docs2 = _bits(cand2)
                for d in docs2:
                    assert by_doc[d][1] == ("typo", rank2, mx2), (query, d)
                seen2 |= set(docs2)
                if child2 is not None:
                    child2.close()
            assert seen2 == set(docs), query
            child.close()
        assert seen == set(by_doc), query
        g.close()


def test_proximity_pairs_matches_decoded_lists(mb, synth):
    """S2 (b200_proximity_pairs): forward + backward pair lookups of two word sets, against the CBO values decoded by the oracle's codec"""
    from oracle.pyoracle import cbo_decode

    ix = mb.Index(synth)
    db = synth.dbs[4]
    key_of = {db.key(i): i for i in range(int(db.n_keys))}
    word_rank = {synth.word(i): i for i in range(synth.n_words)}
    rng = np.random.default_rng(14)
    n_words = (synth.n_docs + 63) // 64
    # word sets drawn from real pair keys so that many probes hit
    picks = rng.integers(0, int(db.n_keys), 60)
    left, right = set(), set()
    for i in picks:
        k = db.key(int(i))
        w1, w2 = k[1:].split(b"\0")
        left.add(word_rank[w1.decode()])
        right.add(word_rank[w2.decode()])
    left, right = sorted(left), sorted(right)
    universe = rng.integers(0, 2**63, n_words, dtype=np.uint64)
    for fwd, bwd in ((1, 0), (2, 1), (3, 2), (0, 1)):
        want = np.zeros(n_words, np.uint64)
        for l in left:
            for r in right:
                for prox, a, b in ((fwd, l, r), (bwd, r, l)):
                    if not prox:
                        continue
                    k = bytes([prox]) + synth.word(a).encode() + b"\0" + synth.word(b).encode()
                    if k in key_of:
                        ids = cbo_decode(db.val(key_of[k]))
                        np.bitwise_or.at(want, ids >> 6, np.uint64(1) << (ids & 63).astype(np.uint64))
        assert want.any() or fwd == 0
        assert np.array_equal(ix.proximity_pairs(left, right, fwd, bwd), want), (fwd, bwd)
        assert np.array_equal(ix.proximity_pairs(left, right, fwd, bwd, universe), want & universe), (fwd, bwd)


def test_limit_zero_reports_candidates(mb, synth):
    """limit 0 still reports SearchResult::candidates (estimatedTotalHits and facets rely on it, bucket_sort.rs:52-64,104-116)"""
    from oracle.pyoracle import OracleIndex

    queries = synth.synthetic_queries(30, seed=81)
    tokens = mb.TokenBatch(queries)
    full = OracleIndex(synth).search_batch(tokens, limit=20, n_threads=8)
    got = mb.Index(synth).search().query(tokens).limit(0).execute()
    for q in range(len(queries)):
        assert got.status[q] == 0 and got.n_hits[q] == 0
        assert int(got.n_candidates[q]) == int(full.n_candidates[q]), queries[q]


def test_malformed_input_is_rejected(mb, synth):
    """the ABI checks what it is given: a truncated roaring value and a repeated stage_finish are errors, not crashes"""
    import copy

    class Img:
        pass
    bad = Img()
    for k in ("n_docs", "n_words", "n_fields", "dict_bytes", "dict_offsets", "documents_ids_cbo"):
        setattr(bad, k, getattr(synth, k))
    bad.dbs = list(synth.dbs)
    db0 = copy.copy(synth.dbs[0])
    lens = np.diff(np.asarray(db0.val_offsets))
    big = int(np.argmax(lens))                       # a roaring-encoded value (> 7 docids)
    assert lens[big] > 28
    vb = np.array(db0.val_bytes, copy=True)
    vb[int(db0.val_offsets[big]) + 4] = 0xFF          # container count 255+: the descriptors would run past the value
    vb[int(db0.val_offsets[big]) + 5] = 0xFF
    db0.val_bytes = vb
    bad.dbs[0] = db0
    with pytest.raises(mb.B200Error) as e:
        mb.Index(bad)
    assert e.value.code == -3
    ix = mb.Index(synth)
    assert ix._l.b200_stage_finish(ix._h) == -6        # B200_ERR_STATE
