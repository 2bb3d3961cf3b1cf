"""The batched vector kernel (run with -m gpu on an H100) computes two 64-row tiles per MMA and drops the second half of a slice's
last block when the slice has an odd number of tiles.  Its top-k must not depend on how the rows are cut into slices: a batch,
its queries sent 64 at a time, and the same batch with fewer CTAs all give identical ids, distances and counts."""
import numpy as np
import pytest

from tests.helpers import synthetic_image

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mb():
    import meilisearch_b200 as m

    m.load_library()
    return m


@pytest.fixture(scope="module")
def img():
    return synthetic_image(3000, 1500, seed=5)


# (rows, d, queries, k): rows not a multiple of 64, fewer row tiles than CTAs per query tile, odd and even tile counts per slice
CASES = [(64 * 37 + 5, 128, 300, 20), (100, 64, 150, 100), (64 * 41, 768, 256, 128), (5001, 64, 1000, 1), (64 * 3 + 63, 768, 17, 7)]


@pytest.mark.parametrize("n,d,nq,k", CASES)
def test_batch_independent_of_slicing(mb, img, monkeypatch, n, d, nq, k):
    rng = np.random.default_rng(n + d + nq + k)
    emb = rng.standard_normal((n, d)).astype(np.float32)
    emb[n // 2:n // 2 + 40] = emb[3]  # a run of equal distances across a tile boundary
    docids = rng.permutation(n).astype(np.uint32)
    q = rng.standard_normal((nq, d)).astype(np.float32)
    q[1] = emb[3]
    cand = np.zeros((n + 63) // 64, np.uint64)
    for doc in np.nonzero(rng.random(n) < 0.3)[0]:
        cand[doc >> 6] |= np.uint64(1) << np.uint64(doc & 63)
    ix = mb.Index(img)
    ix.set_embeddings(emb, docids)
    monkeypatch.setenv("B200_VEC_GEMM", "1")  # also for a short last chunk of 64
    for cw in (None, cand):
        monkeypatch.delenv("B200_VEC_SMS", raising=False)
        ix.reset_stats()
        ids, dist, cnt = ix.nns_by_vector(q, k, cw)
        assert ix.stats()["kernels"]["vec_gemm_topk"]["count"] >= 1
        assert (cnt == min(k, n if cw is None else int(sum(bin(int(w)).count("1") for w in cand)))).all()
        for i in range(nq):
            assert (np.diff(dist[i, : cnt[i]]) >= 0).all()
        chunks = [ix.nns_by_vector(q[i:i + 64], k, cw) for i in range(0, nq, 64)]
        for j, got in enumerate(zip(*chunks)):
            assert np.array_equal(np.concatenate(got), (ids, dist, cnt)[j]), ("chunks of 64", n, d, nq, k, j)
        for sms in ("8", "33"):
            monkeypatch.setenv("B200_VEC_SMS", sms)
            for j, got in enumerate(ix.nns_by_vector(q, k, cw)):
                assert np.array_equal(got, (ids, dist, cnt)[j]), ("B200_VEC_SMS", sms, n, d, nq, k, j)
