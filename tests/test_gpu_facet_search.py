"""GPU: facet search (facet_search.cu, b200_facet_search_batch) against the CPU specification (tests/facet_search_spec.py) over the
same candidates: keyword and placeholder search candidates and random bitmaps, every query kind, both orders and several
maxValuesPerFacet, on a field built for count ties at the cut and originals that differ between documents."""
import numpy as np
import pytest

import meilisearch_b200 as mb
from corpus.facets import FacetImage
from corpus.pyindexgen import IndexImage
from tests.facet_search_spec import facet_search

pytestmark = pytest.mark.gpu

CRITERIA = ["words", "typo", "proximity", "attributeRank", "sort", "wordPosition", "exactness"]
EXACT = ["tag07", "brand001"]
GENRES = ["Adventure", "adventure", "Àdventure", "ADVENTURE ", "Action", "Comedy", "comédie", "Comédie", "Drama", "Horror", "Crime",
          "Romance", "Thriller", "Science Fiction", "Fantasy", "Animation", "Documentary", "Family", "War", "Western"]


def make(n_docs):
    img = IndexImage(1)
    img.add_synthetic(n_docs, 2000)
    img.build()
    fac = FacetImage().add_synthetic(n_docs).add_synthetic_search(n_docs, n_values=min(n_docs, 4000))
    rng = np.random.default_rng(11)
    # `genre`: 20 originals over 16 normalised keys and 13 hyper-normalised strings, drawn so that small candidate sets tie
    for d, k in enumerate(rng.integers(0, len(GENRES), n_docs)):
        fac.add_facet(d, "genre", GENRES[k])
    fac.build()
    fac.build_search()
    return img, fac


@pytest.fixture(scope="module")
def small():
    img, fac = make(40_000)
    return img, fac, mb.Index(img, criteria=CRITERIA, facets=fac, exact_words=EXACT)


def bitmap(n_docs, docs):
    bits = np.zeros(((n_docs + 63) // 64) * 64, np.uint8)
    bits[np.asarray(sorted(docs), np.int64)] = 1
    return np.packbits(bits, bitorder="little").view(np.uint64)


def docs_of(bm, n_docs):
    return np.nonzero(np.unpackbits(bm.view(np.uint8), bitorder="little")[:n_docs])[0].tolist()


QUERIES = [None, "", "a", "ad", "adv", "advnture", "avdenture", "comedie", "com", "brand0", "brand01", "brnd012", "tag07", "tag0",
           "tga07", "xyz", "s", "sci", "science fic", "b", "ab", "abcdefghijkl"]


def compare(ix, fac, cands, sets, name, queries, order, max_values, typos=True):
    fid = fac.fields[name]
    got, status = ix.facet_search(cands, name, queries, order=order, max_values=max_values, typos=typos)
    qs = queries if isinstance(queries, list) else [queries] * len(cands)
    for i, (docs, q) in enumerate(zip(sets, qs)):
        assert status[i] == 0, (name, q, ix.last_error())
        want = facet_search(fac, fid, docs, q, order=order, max_values=max_values, field_typos=typos, exact_words=EXACT)
        assert got[i] == want, (name, q, order, max_values, typos, len(docs))


@pytest.mark.parametrize("order", ["alpha", "count"])
@pytest.mark.parametrize("max_values", [0, 1, 3, 100])
def test_random_bitmaps(small, order, max_values):
    img, fac, ix = small
    rng = np.random.default_rng(max_values)
    sets = [[], [int(rng.integers(img.n_docs))]] + [sorted(rng.choice(img.n_docs, size, replace=False).tolist()) for size in (3000, 20000)]
    cands = [bitmap(img.n_docs, s) for s in sets] + [None]
    sets.append(list(range(img.n_docs)))
    for name in ("genre", "brand", "tags", "model"):
        for q in QUERIES:
            compare(ix, fac, cands, sets, name, q, order, max_values)
        compare(ix, fac, cands, sets, name, "adv", order, max_values, typos=False)


def test_search_candidates(small):
    img, fac, ix = small
    queries = img.synthetic_queries(6, seed=5) + [""] * 2
    res = ix.search().query(queries).with_candidates().execute()
    sets = [docs_of(res.candidates[q], img.n_docs) for q in range(len(queries))]
    for order in ("alpha", "count"):
        for q in (None, "", "ad", "adventure", "comedi", "brnd00"):
            compare(ix, fac, list(res.candidates), sets, "genre", q, order, 3)
            compare(ix, fac, list(res.candidates), sets, "brand", q, order, 10)


def test_one_query_per_bitmap_and_shared_bitmaps(small):
    img, fac, ix = small
    rng = np.random.default_rng(9)
    docs = sorted(rng.choice(img.n_docs, 5000, replace=False).tolist())
    bm = bitmap(img.n_docs, docs)
    queries = ["ad", None, "", "comdie", "tag07"]
    compare(ix, fac, [bm] * len(queries), [docs] * len(queries), "genre", queries, "count", 2)


def test_errors(small):
    img, fac, ix = small
    got, status = ix.facet_search([None], "genre", "a" * 65)
    assert status[0] == mb.B200Error(-4, "").code and got == [[]]
    got, status = ix.facet_search([None, None], "genre", [None, "ad"], max_values=10, cap=1)  # 16 and 2 hits
    assert list(status) == [-5, -5]
    got, status = ix.facet_search([None], "nope", None)
    assert status[0] == 0 and got == [[]]
    got, status = ix.facet_search([None], "price", None)  # a number field: no FST
    assert status[0] == 0 and got == [[]]


def test_stats_and_no_side_effects(small):
    img, fac, ix = small
    ix.reset_stats()
    ix.facet_search([None], "model", "ab")
    k = ix.stats()["kernels"]["facet_search"]
    assert k["count"] == 3 and k["ms"] > 0
    a = ix.search().query(img.synthetic_queries(4, seed=3)).execute()
    b = ix.search().query(img.synthetic_queries(4, seed=3)).execute()
    for q in range(4):
        assert a.ids(q) == b.ids(q)


def test_large_corpus():
    img, fac = make(700_000)
    ix = mb.Index(img, criteria=CRITERIA, facets=fac, exact_words=EXACT)
    rng = np.random.default_rng(2)
    sets = [sorted(rng.choice(img.n_docs, 20000, replace=False).tolist())]
    cands = [bitmap(img.n_docs, sets[0]), None]
    sets.append(list(range(img.n_docs)))
    for order in ("alpha", "count"):
        for q in (None, "ab", "abc", "brand00", "genre"):
            compare(ix, fac, cands, sets, "model", q, order, 100)
            compare(ix, fac, cands, sets, "genre", q, order, 3)


def test_staged_escapes_missing_keys_and_no_originals():
    """set values written with \\u escapes and surrogate pairs, out of order and with duplicates, an entry whose first key
    facet_id_string_docids lacks (the rest of that entry is skipped), and no originals at all (every value falls back)"""
    import json

    from corpus.facets import _db

    fac = FacetImage()
    vals = ['Café "q"', "emoji 🎉 fan", "back\\slash", "Plain", "Émoji 🎉 fan"]
    for d in range(300):
        fac.add_facet(d, "f", vals[d % len(vals)])
    fac.build()
    fac.build_search()
    entries = []
    for i in range(fac.norm_db.n_keys):
        keys = json.loads(fac.norm_db.val(i).decode())
        if fac.norm_db.key(i)[2:] == b"plain":
            keys = ["", *keys]  # "" sorts first and is not a level-0 key
        entries.append((fac.norm_db.key(i), json.dumps(keys[::-1] + keys, ensure_ascii=True).encode()))
    fac.norm_db, fac.orig_db = _db(entries), _db([])
    img = IndexImage(1)
    img.add_synthetic(300, 50)
    img.build()
    ix = mb.Index(img, facets=fac)
    docs = list(range(300))
    for q in (None, "", "caf", "emoji", "emoj", "plain", "back"):
        for order in ("alpha", "count"):
            got, status = ix.facet_search([None], "f", q, order=order, max_values=10)
            assert status[0] == 0
            spec = facet_search(fac, fac.fields["f"], docs, q, order=order, max_values=10)
            assert got[0] == spec, (q, order)
    assert ix.facet_search([None], "f", "plain")[0] == [[]]
    bad = FacetImage()
    bad.add_facet(0, "f", "x")
    bad.build()
    bad.build_search()
    bad.norm_db = _db([(bad.norm_db.key(0), b'["x",')])
    with pytest.raises(mb.B200Error) as e:
        mb.Index(img, facets=bad)
    assert e.value.code == -3
