"""The keyword path in the configurations the rest of the suite leaves at their defaults, against the CPU oracle: queries of
6-12 words in every DP slot class, every lane layout, the sequential bucket sort, device-memory budgets small enough to defer and
fail activations, both extremes of the posting-list forms, row lookup tables on and off, and several rows per thread.  Docids,
score tuples, candidate counts and statuses must equal the oracle's, and each test checks through Index.stats() that the path it
is named for ran."""
import math
import os
import random

import numpy as np
import pytest

from tests.helpers import synthetic_image

pytestmark = pytest.mark.gpu

# every knob these tests set; cleared before each test so that the caller's environment cannot change which path a test runs
KNOBS = ("B200_ARENA_MB", "B200_SCRATCH_MB", "B200_DENSE_DIV", "B200_DRIVERS", "B200_LANES_PER_DRIVER", "B200_WAVES", "B200_NO_TREE",
         "B200_NO_ROWTAB", "B200_ROWTAB_MIN", "B200_EVAL_RPT", "B200_SINGLE_LANE")
FULL = ["words", "typo", "proximity", "attribute", "wordPosition", "exactness"]
STOP = ("the", "of", "and")
ERR_CAPACITY = -5
MB = 1 << 20
N_MADE = 32768  # 512 rows of 64 documents: a query's first activation spans four 128-row tiles


@pytest.fixture(autouse=True)
def _default_knobs(monkeypatch):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)


@pytest.fixture(scope="module")
def mb():
    import meilisearch_b200 as m

    m.load_library()
    return m


@pytest.fixture(scope="module")
def synth():
    return synthetic_image(60000, 25000, seed=11)


def _edit(r, w):
    p, c = r.randrange(len(w)), chr(97 + r.randrange(26))
    k = r.randrange(3)
    return w[:p] + c + w[p + 1:] if k == 0 else (w[:p] + c + w[p:] if k == 1 else w[:p] + w[p + 1:])


@pytest.fixture(scope="module")
def made():
    return made_image()


def made_image():
    """A corpus for long queries: 3 fields; the 64 documents of a row share one of 6 topics of 14 words and hold 0-6 of them per
    field at positions drawn per document, some as a typo, a longer word (prefix match) or glued to the next topic word (n-gram),
    between filler words and stop words.  -> (image, topics)"""
    from corpus.pyindexgen import IndexImage

    r = random.Random(0x5EED)
    word = lambda lo, hi: "".join(chr(97 + r.randrange(26)) for _ in range(r.randint(lo, hi)))
    topics = [[word(5, 11) for _ in range(14)] for _ in range(6)]
    filler = [word(3, 8) for _ in range(3000)]
    img = IndexImage(3, 0, STOP)
    for d in range(N_MADE):
        words = topics[(d >> 6) % len(topics)]
        for f in range(3):
            toks = [filler[min(len(filler) - 1, int(r.expovariate(1 / 300)))] for _ in range(r.randint(4, 28))]
            for i in r.sample(range(len(words)), r.randint(0, 6)):
                w, x = words[i], r.random()
                if x < 0.15:
                    w = _edit(r, w)
                elif x < 0.25:
                    w += r.choice(("s", "ing", "er"))
                elif x < 0.35 and i + 1 < len(words):
                    w += words[i + 1]
                toks.insert(r.randint(0, len(toks)), w)
            for _ in range(r.randint(0, 2)):
                toks.insert(r.randint(0, len(toks)), r.choice(STOP))
            img.add_text(d, f, " ".join(toks))
    return img.build(), topics


def made_queries(topics, n, seed, lo=6, hi=12):
    """n queries of lo-hi words of one topic: half in topic order (consecutive words form the corpus' n-grams), some with a typo, a
    truncated last word (prefix) or stop words among them"""
    r = random.Random(seed)
    out = []
    for _ in range(n):
        t = topics[r.randrange(len(topics))]
        k = r.randint(lo, hi)
        n_stop = r.randint(0, min(2, k - lo))
        idx = r.sample(range(len(t)), k - n_stop)
        if r.random() < 0.5:
            idx.sort()
        ws = [t[i] for i in idx]
        if r.random() < 0.3:
            j = r.randrange(len(ws))
            ws[j] = _edit(r, ws[j])
        if r.random() < 0.3 and len(ws[-1]) > 4:
            ws[-1] = ws[-1][: r.randint(3, len(ws[-1]) - 1)]
        for _ in range(n_stop):
            ws.insert(r.randint(1, len(ws)), r.choice(STOP))
        out.append(" ".join(ws))
    return out


def joined_queries(img, n, seed):
    """n queries of 6-12 words made by joining the corpus' synthetic queries"""
    r = random.Random(seed)
    words = " ".join(img.synthetic_queries(4 * n, seed=seed)).split()
    out, i = [], 0
    while len(out) < n:
        k = r.randint(6, 12)
        assert i + k <= len(words)
        out.append(" ".join(words[i:i + k]))
        i += k
    return out


@pytest.fixture(scope="module")
def oracle():
    return oracle_cache()


def oracle_cache():
    """want(image, queries, criteria, tms, scoring, offset, limit): the oracle's answer, computed once per module"""
    from meilisearch_b200 import TokenBatch
    from oracle.pyoracle import OracleIndex

    indexes, memo = {}, {}

    def want(img, queries, crit=None, tms="last", scoring="detailed", offset=0, limit=20):
        key = (id(img), tuple(queries), tuple(crit or ()), tms, scoring, offset, limit)
        if key not in memo:
            ik = (id(img), tuple(crit or ()))
            if ik not in indexes:
                indexes[ik] = OracleIndex(img, criteria=crit)
            memo[key] = indexes[ik].search_batch(TokenBatch(queries, img.stop_words), tms=tms, scoring=scoring, offset=offset, limit=limit,
                                                 words_limit=12, n_threads=os.cpu_count() or 1)
        return memo[key]

    return want


def search(ix, img, queries, tms="last", scoring="detailed", offset=0, limit=20, candidates=False):
    from meilisearch_b200 import TokenBatch

    s = ix.search().query(TokenBatch(queries, img.stop_words)).terms_matching_strategy(tms).scoring_strategy(scoring)
    s = s.offset(offset).limit(limit).words_limit(12)
    return (s.with_candidates() if candidates else s).execute()


def same(got, want, queries, ctx, only=None, candidates=False):
    """the queries `only` (default: all) have status 0 and the oracle's docids, score tuples and candidate counts"""
    for q in range(len(queries)) if only is None else only:
        c = (ctx, q, queries[q])
        assert got.status[q] == 0, c + (int(got.status[q]),)
        assert got.ids(q) == want.ids(q), c
        assert got.scores(q) == want.scores(q), c
        assert int(got.n_candidates[q]) == int(want.n_candidates[q]), c
        if candidates:
            cand = got.candidates[q]
            assert int(np.bitwise_count(cand).sum()) == int(want.n_candidates[q]), c
            assert all((int(cand[d >> 6]) >> (d & 63)) & 1 for d in got.ids(q)), c


# offset/limit windows: 37/50 and 0/1000 put walk_kernel's `need` cut inside buckets
WINDOWS = [("last", "detailed", 0, 20), ("all", "detailed", 37, 50), ("frequency", "detailed", 0, 1000), ("last", "skip", 37, 50),
           ("frequency", "skip", 0, 20), ("all", "skip", 0, 1000)]


def test_long_queries_in_every_dp_class(mb, synth, made, oracle):
    """Queries of 6-12 words under full criteria stacks: activations of every shared-memory slot class and of the global-memory DP
    (class 8), walks over more than 64 condition columns (Position over 12 terms and their n-grams, each found at many positions)
    and rows whose needed documents carry more than 8 condition patterns (each document of a row holds the topic words at positions
    of its own).  No statistic counts the last two."""
    img_m, topics = made
    batches = [(synth, joined_queries(synth, 60, seed=7)), (img_m, made_queries(topics, 80, seed=3))]
    launches = np.zeros(9, np.int64)
    for crit in (FULL, None):
        for img, queries in batches:
            ix = mb.Index(img, criteria=crit)
            for tms, scoring, off, lim in WINDOWS:
                got = search(ix, img, queries, tms, scoring, off, lim, candidates=lim == 50)
                same(got, oracle(img, queries, crit, tms, scoring, off, lim), queries, (crit, tms, scoring, off, lim), candidates=lim == 50)
            launches += ix.stats()["eval_class_launches"]
            ix.close()
    print("eval_class_launches", launches.tolist())
    assert (launches > 0).all(), launches


@pytest.fixture(scope="module")
def lane_batch(synth):
    """620 queries, short and long mixed"""
    queries = synth.synthetic_queries(560, seed=23) + joined_queries(synth, 60, seed=29)
    random.Random(5).shuffle(queries)
    return queries


LAYOUTS = [None, (1, 1), (2, 1), (3, 1), (4, 2), (2, 4), (3, 3), (3, 4)]


@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda x: "default" if x is None else "%dx%d" % x)
def test_lane_layouts(mb, synth, oracle, lane_batch, monkeypatch, layout):
    """(drivers, lanes per driver) and derivation waves: every lane the batch is split over is driven.  (3, 3) and (3, 4) ask for
    more than the 8 lanes there are."""
    want = oracle(synth, lane_batch)
    ix = mb.Index(synth)
    n_drivers, per_driver = (4, 1) if layout is None else layout
    if layout is not None:
        monkeypatch.setenv("B200_DRIVERS", str(n_drivers))
        monkeypatch.setenv("B200_LANES_PER_DRIVER", str(per_driver))
    for waves in (1, 2, 4):
        monkeypatch.setenv("B200_WAVES", str(waves))
        ix.reset_stats()
        got = search(ix, synth, lane_batch)
        same(got, want, lane_batch, (layout, waves))
        assert ix.stats()["device_steps"] >= n_drivers * min(per_driver, 8 // n_drivers)


def test_sequential_bucket_sort(mb, synth, made, oracle, lane_batch, monkeypatch):
    """B200_NO_TREE=1: one needed bucket per device step instead of every needed bucket of a level"""
    img_m, topics = made
    cases = [(img_m, made_queries(topics, 80, seed=3), FULL, None), (synth, lane_batch, None, None), (synth, lane_batch, None, (3, 4))]
    for img, queries, crit, layout in cases:
        if layout is not None:
            monkeypatch.setenv("B200_DRIVERS", str(layout[0]))
            monkeypatch.setenv("B200_LANES_PER_DRIVER", str(layout[1]))
        want = oracle(img, queries, crit)
        ix = mb.Index(img, criteria=crit)
        steps = {}
        for no_tree in (False, True):
            if no_tree:
                monkeypatch.setenv("B200_NO_TREE", "1")
            ix.reset_stats()
            same(search(ix, img, queries), want, queries, (crit, layout, no_tree))
            steps[no_tree] = ix.stats()["device_steps"]
            monkeypatch.delenv("B200_NO_TREE", raising=False)
        print("device_steps tree / sequential", crit, layout, steps[False], steps[True])
        assert steps[True] > steps[False], steps
        ix.close()


def staged(mb, img, monkeypatch, arena=None, scratch=None):
    """a new Index whose arena / scratch (whole MB, None = default) is read at staging"""
    for k, v in (("B200_ARENA_MB", arena), ("B200_SCRATCH_MB", scratch)):
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))
    return mb.Index(img)


def check_budget(mb, img, queries, want, monkeypatch, arena, scratch):
    """search under the budget: activations were deferred; every query either equals the oracle or failed with B200_ERR_CAPACITY
    and no hits -> (failed queries, those of them that also fail when searched alone under the same budget)"""
    ix = staged(mb, img, monkeypatch, arena, scratch)
    got = search(ix, img, queries)
    st = ix.stats()
    assert st["deferred"] > 0, (arena, scratch)
    failed = [q for q in range(len(queries)) if got.status[q] != 0]
    for q in failed:
        assert got.status[q] == ERR_CAPACITY and got.n_hits[q] == 0, (arena, scratch, q, int(got.status[q]))
    same(got, want, queries, (arena, scratch), only=[q for q in range(len(queries)) if q not in failed])
    alone = [q for q in failed if search(ix, img, [queries[q]]).status[0] != 0]
    ix.close()
    print("budget arena_mb=%s scratch_mb=%s: %d queries, %d deferred, %d failed %s, %d of them fail alone %s"
          % (arena, scratch, len(queries), st["deferred"], len(failed), failed, len(alone), alone))
    return failed, alone


@pytest.fixture(scope="module")
def big():
    return synthetic_image(700_000, 60_000, seed=0xB201)


@pytest.mark.parametrize("corpus", ["synth", "big"])
def test_memory_budgets(mb, synth, big, oracle, monkeypatch, corpus):
    """One lane under B200_ARENA_MB at 1/2 and 1/4 of the batch's arena peak and B200_SCRATCH_MB at 1/2 and 1/4 of the smallest
    power-of-two budget under which no activation waits; on 700 k documents also the arena at 1/10 and 1/20 of the peak.
    Activations are deferred; every query equals the oracle or fails with B200_ERR_CAPACITY and no hits.  A query that fails
    under a scratch budget fails alone too (one of its steps does not fit the lane).  Under a starved arena, queries that hold
    blocks can wait on each other: the one failed to break that would succeed alone."""
    img = synth if corpus == "synth" else big
    monkeypatch.setenv("B200_DRIVERS", "1")
    queries = img.synthetic_queries(60, seed=43) + joined_queries(img, 20, seed=47)
    want = oracle(img, queries)
    ix = staged(mb, img, monkeypatch)
    same(search(ix, img, queries), want, queries, "no budget")
    st = ix.stats()
    assert st["deferred"] == 0
    peak = st["arena_peak_bytes"]
    ix.close()
    scratch = 1024
    while True:
        ix = staged(mb, img, monkeypatch, scratch=scratch)
        search(ix, img, queries)
        deferred = ix.stats()["deferred"]
        ix.close()
        if deferred or scratch == 1:
            break
        scratch //= 2
    assert deferred > 0
    fits = scratch * 2
    print("%s: arena peak %d bytes; scratch: nothing waits at %d MB" % (corpus, peak, fits))
    arena = lambda div: math.ceil(peak / div / MB)
    budgets = [(arena(2), None), (arena(4), None), (None, max(1, fits // 2)), (None, max(1, fits // 4)), (arena(4), max(1, fits // 4))]
    if corpus == "big":
        budgets += [(arena(10), None), (arena(20), None)]
    n_failed = 0
    for a, s in budgets:
        failed, alone = check_budget(mb, img, queries, want, monkeypatch, a, s)
        if a is None:
            assert failed == alone, (a, s, failed, alone)
        n_failed += len(failed)
    assert n_failed > 0 or corpus == "synth"


def test_capacity_failure_is_one_query(mb, big, oracle, monkeypatch):
    """a scratch budget one MB short of what a 12-term query's widest step needs, while the 2-word queries of the same batch fit:
    that query fails alone with B200_ERR_CAPACITY and every other query is exact"""
    img = big
    monkeypatch.setenv("B200_DRIVERS", "1")
    short = [q for q in img.synthetic_queries(120, seed=53, with_typos=False) if len(q.split()) == 2][:30]
    long_q = " ".join(" ".join(img.synthetic_queries(12, seed=59, with_typos=False)).split()[:12])
    queries = short[:15] + [long_q] + short[15:]
    k = queries.index(long_q)

    def statuses(scratch, qs):
        ix = staged(mb, img, monkeypatch, scratch=scratch)
        st = [int(s) for s in search(ix, img, qs).status]
        ix.close()
        return st

    lo, hi = 1, 256
    assert statuses(hi, [long_q]) == [0]
    while lo < hi:  # the smallest budget under which the long query runs alone
        mid = (lo + hi) // 2
        if statuses(mid, [long_q]) == [0]:
            hi = mid
        else:
            lo = mid + 1
    print("the 12-term query needs %d MB of scratch" % lo)
    assert lo > 1
    assert statuses(lo - 1, [long_q]) == [ERR_CAPACITY]
    ix = staged(mb, img, monkeypatch, scratch=lo - 1)
    got = search(ix, img, queries)
    assert got.status[k] == ERR_CAPACITY and got.n_hits[k] == 0
    same(got, oracle(img, queries), queries, lo - 1, only=[q for q in range(len(queries)) if q != k])


@pytest.mark.parametrize("dense_div", [8, 1 << 30])
def test_posting_list_forms_and_row_tables(mb, synth, made, oracle, monkeypatch, dense_div):
    """B200_DENSE_DIV=8 stores only lists of more than n_docs / 8 documents as bitmaps, 2^30 every list of more than 64; each under
    row lookup tables for activations of at least 64 rows (the default), for every activation (B200_ROWTAB_MIN=1) and for none"""
    from tests.test_gpu_parity import check_union_postings

    img_m, topics = made
    batches = [(synth, synth.synthetic_queries(100, seed=61) + joined_queries(synth, 20, seed=67)),
               (img_m, made_queries(topics, 60, seed=71, lo=2))]
    for img, queries in batches:
        ix = mb.Index(img)
        default_bytes = ix.stats()["hbm_bytes_staged"]
        ix.close()
        monkeypatch.setenv("B200_DENSE_DIV", str(dense_div))
        ix = mb.Index(img, criteria=FULL)
        assert ix.stats()["hbm_bytes_staged"] != default_bytes
        if img is synth:
            check_union_postings(ix, synth)
        want = oracle(img, queries, FULL)
        for knob in (None, "B200_ROWTAB_MIN", "B200_NO_ROWTAB"):
            if knob is not None:
                monkeypatch.setenv(knob, "1")
            same(search(ix, img, queries, candidates=True), want, queries, (dense_div, knob), candidates=True)
            monkeypatch.delenv(knob or "B200_NO_ROWTAB", raising=False)
        ix.close()
        monkeypatch.delenv("B200_DENSE_DIV")


def test_rows_per_thread(mb, oracle, monkeypatch):
    """64 * (65536 + 300) - 5 documents: the first activation has more than 65 536 rows, a partial last tile at every row count
    per thread, and its tiles take B200_EVAL_RPT rows per thread"""
    from corpus.pyindexgen import synthetic_image as cached_image

    img = cached_image(64 * (65536 + 300) - 5, 100_000, seed=0xB2E7)
    queries = img.synthetic_queries(24, seed=73)
    want = oracle(img, queries)
    ix = mb.Index(img)
    tiles = {}
    for rpt in (1, 2, 4, 8):
        monkeypatch.setenv("B200_EVAL_RPT", str(rpt))
        ix.reset_stats()
        same(search(ix, img, queries), want, queries, rpt)
        tiles[rpt] = ix.stats()["eval_class_tiles"][0]
    print("class-0 tiles per rows per thread", tiles)
    assert tiles[1] > tiles[2] > tiles[4] > tiles[8], tiles
