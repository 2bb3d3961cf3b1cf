"""The references of the vector stage (tests/vec_spec.py) on the CPU: the exact-arithmetic generator keeps its promise, and R1,
the float32 replica of the device formula, agrees with the oracle's `nns_by_vector` (the specification) on exact inputs, zero
and near-zero norms and the zero query included."""
import numpy as np
import pytest

from oracle.pyoracle import OracleIndex
from tests import vec_spec as vs
from tests.helpers import synthetic_image

ULP = 2.0 ** -24  # spacing of f32 in [0.5, 1): one ulp of the cosine's halves, the scale every distance is computed at


@pytest.fixture(scope="module")
def img():
    return synthetic_image(500, 300, seed=21)


@pytest.mark.parametrize("d", [8, 64, 100, 768, 1536])
def test_exact_generator_is_exact(d):
    g = vs.ExactGen(d, seed=d)
    rows = g.mixed_rows(3000, dup=0.1, scaled=0.1, zero=0.03, tiny=0.05)
    q = g.mixed_queries(24, rows)
    dots = vs.exact_dots(rows, q)
    assert np.array_equal(dots.astype(np.float64), q.astype(np.float64) @ rows.astype(np.float64).T)
    for x in (rows, q):
        assert np.array_equal(x.astype(np.float16).astype(np.float32), x)  # staged and wgmma-rounded values are the same
        s32 = np.einsum("ij,ij->i", x, x, dtype=np.float32)
        assert np.array_equal(s32.astype(np.float64), np.einsum("ij,ij->i", x.astype(np.float64), x.astype(np.float64)))
    assert vs.rule_margin_ok(rows, q)
    # the classes the stress cases rely on are present
    norms = np.linalg.norm(rows.astype(np.float64), axis=1)
    assert (norms == 0).any() and (norms == 2.0 ** -24).any()
    qn = np.linalg.norm(q.astype(np.float64), axis=1)
    assert (qn == 0).any() and (qn == 2.0 ** -24).any() and ((qn > 0.5) & (qn <= 1)).any()
    # scaled copies tie exactly with their source for every query of the normal class (a tiny query may see one of them under
    # the norm rule and the other not)
    base = g.rows(50)
    copy = g.scaled(base, 2.0 ** -14)
    assert not np.array_equal(copy, base)
    normal = qn >= 2.0 ** -8
    assert np.array_equal(vs.r1_distances(base, q[normal]), vs.r1_distances(copy, q[normal]))


def test_norm_rule_classes():
    """zero and tiny rows are at distance 0 for zero, tiny and small queries, and computed for large ones"""
    g = vs.ExactGen(64, seed=3)
    rows = np.concatenate([g.tiny(4), np.zeros((2, 64), np.float32), g.rows(10)])
    q = g.mixed_queries(8, rows)
    dist = vs.r1_distances(rows, q)
    qn = np.linalg.norm(q.astype(np.float64), axis=1)
    for i in range(len(q)):
        assert (dist[i, 4:6] == 0).all()
        if qn[i] <= 1:
            assert (dist[i, :4] == 0).all()
        if qn[i] == 0:
            assert (dist[i] == 0).all()


def _clusters(od, gap):
    """maximal runs of positions whose consecutive distances differ by at most `gap`"""
    cut = np.nonzero(np.diff(od.astype(np.float64)) > gap)[0] + 1
    return np.split(np.arange(len(od)), cut)


@pytest.mark.parametrize("d,n,seed", [(8, 2000, 1), (64, 3000, 2), (100, 1500, 3), (768, 1200, 4), (1536, 600, 5)])
def test_r1_matches_oracle_on_exact_inputs(img, d, n, seed):
    g = vs.ExactGen(d, seed=seed)
    rows = g.mixed_rows(n, dup=0.1, scaled=0.1, zero=0.03, tiny=0.05)
    docids = g.docids(n, img.n_docs)
    q = g.mixed_queries(12, rows)
    assert vs.rule_margin_ok(rows, q)
    o = OracleIndex(img)
    o.set_embeddings(rows, docids)
    cand = vs.bitmap(np.nonzero(g.rng.random(img.n_docs + 64) < 0.5)[0])
    for cw in (None, cand):
        rid, rd, rc = vs.r1(rows, docids, q, n, cw)
        for i in range(len(q)):
            oid, od = o.nns(q[i], n, cw)
            assert rc[i] == len(oid), (d, i)
            got_d = rd[i, : rc[i]].astype(np.float64)
            assert np.abs(got_d - od).max(initial=0) <= 2 * ULP, (d, i, np.abs(got_d - od).max())
            # ids: equal wherever the oracle's distances are more than 4 ulp apart; inside a cluster of closer ones, the same set
            for c in _clusters(od, 4 * ULP):
                if len(c) == 1:
                    assert rid[i, c[0]] == oid[c[0]], (d, i, int(c[0]))
                else:
                    assert sorted(rid[i, c].tolist()) == sorted(oid[c].tolist()), (d, i, c[:4])
            # exact ties are ordered by docid on both sides
            ties = od[1:] == od[:-1]
            assert (oid[1:][ties] >= oid[:-1][ties]).all()


def test_r1_zero_query_is_docid_order(img):
    g = vs.ExactGen(64, seed=9)
    rows = g.mixed_rows(2000)
    docids = g.docids(2000, img.n_docs)
    q = np.zeros((1, 64), np.float32)
    ids, dist, cnt = vs.r1(rows, docids, q, 50)
    assert cnt[0] == 50 and (dist[0] == 0).all()
    assert list(ids[0]) == sorted(docids.tolist())[:50]
    o = OracleIndex(img)
    o.set_embeddings(rows, docids)
    oid, od = o.nns(q[0], 50)
    assert list(oid) == list(ids[0]) and (od == 0).all()


def test_certificate_rejects_wrong_results():
    """the R2 certificate accepts the exact answer and refuses a lost row, a wrong distance and a wrong order"""
    rng = np.random.default_rng(0)
    d, n, k = 128, 4000, 20
    rows = rng.standard_normal((n, d)).astype(np.float32)
    docids = rng.permutation(n).astype(np.uint32)
    q = rng.standard_normal((3, d)).astype(np.float32)
    r2 = vs.r2_distances(rows, q, "gemv")
    ids, dist, cnt = vs.topk(r2.astype(np.float32), docids, k)
    vs.check_certificate(ids, dist, cnt, docids, r2, k, d)
    far = np.argsort(r2[0])[k + 50]  # a consistent answer that lost its k-th row for a farther one
    bad, bdist = ids.copy(), dist.copy()
    bad[0, k - 1], bdist[0, k - 1] = docids[far], np.float32(r2[0, far])
    with pytest.raises(AssertionError, match="order|,"):
        vs.check_certificate(bad, bdist, cnt, docids, r2, k, d)
    bd = dist.copy()
    bd[1, 5] += 1e-3
    with pytest.raises(AssertionError):
        vs.check_certificate(ids, bd, cnt, docids, r2, k, d)
    sw = ids.copy()
    sw[2, [0, 1]] = sw[2, [1, 0]]
    sd = dist.copy()
    sd[2, [0, 1]] = sd[2, [1, 0]]
    with pytest.raises(AssertionError):
        vs.check_certificate(sw, sd, cnt, docids, r2, k, d)
    with pytest.raises(AssertionError):
        vs.check_certificate(ids, dist, cnt - 1, docids, r2, k, d)
