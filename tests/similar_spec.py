"""Similar::execute (crates/milli/src/search/similar.rs:66-152) restated over a staged vector store, numpy only.

For target `id` and U = documents_ids AND the caller's universe AND its filter:
  1. the universe is U \\ {id};
  2. the reference calls VectorStore::nns_by_item(id, offset + limit + 1, U \\ {id}) (vector/store.rs:980-1034): one search per store,
     store k holding each document's k-th vector, searched with the target's k-th vector (a store without the target is skipped);
     the stores' lists are concatenated and sorted by distance.  Here a store is a flat list of staged rows, so store k is every
     document's k-th row in staging order, each search is exact (ascending (distance, docid)) and the merged list is sorted by
     (distance, docid);
  3. the list is walked: `seen` starts as {id}, a docid already in it is dropped, otherwise added; the first `offset` survivors are
     skipped; at most `limit` are taken with score 1 - distance (f32), shifted by the distribution if there is one; with a
     threshold, a taken document whose score is below it ends the walk and candidates becomes (candidates \\ {doc}) AND seen;
  4. n_candidates = |candidates|, candidates starting as U \\ {id}; a target without a row, or outside documents_ids (a deleted
     document, which the vector store no longer holds), has no hits.

`distance(query, rows)` is the distance function: `r1` (tests/vec_spec.py, the device formula, exact on ExactGen data) or `f64`."""
import numpy as np

from tests import vec_spec as vs

F32 = np.float32


def r1(query, rows):
    """f32 distances of the device formula (bit for bit on exact-arithmetic data)"""
    return vs.r1_distances(rows, query[None, :])[0]


def f64(query, rows):
    """(1 - cos) / 2 in float64 with the norm rule |q||v| > f32::EPSILON"""
    q = query.astype(np.float64)
    r = rows.astype(np.float64)
    p = np.linalg.norm(q) * np.linalg.norm(r, axis=1)
    with np.errstate(invalid="ignore", divide="ignore"):
        cs = np.clip((r @ q) / p, -1, 1)
    return np.where(p > vs.EPS, (1 - cs) / 2, 0.0)


def shift(distribution, score):
    """DistributionShift::shift (vector/distribution.rs:103-130) in f32"""
    mean, sigma = F32(distribution[0]), F32(distribution[1])
    factor = F32(0.4) / sigma
    offset = F32(0.5) - factor * mean
    s = factor * F32(score) + offset
    if s <= 0:
        s = F32(1.1920929e-7)
    return min(s, F32(1))


def stores(docids):
    """per store k, the rows holding each document's k-th vector"""
    count, out = {}, []
    for r, d in enumerate(docids):
        k = count.get(int(d), 0)
        count[int(d)] = k + 1
        if k == len(out):
            out.append([])
        out[k].append(r)
    return out


def similar(rows, docids, target, universe, *, offset=0, limit=20, threshold=None, distribution=None, distance=r1, documents_ids=None):
    """(hit docids, their f32 scores, n_candidates) of Similar::execute.  rows / docids: the staged store (rows as the f32 values the
    device holds); universe: the docids of U (an iterable); documents_ids: the index's documents (None: every target counts as one)"""
    rows = np.asarray(rows)
    docids = np.asarray(docids, np.int64)
    u = set(int(x) for x in universe) - {int(target)}
    want = offset + limit + 1
    found = []
    for store in stores(docids) if documents_ids is None or int(target) in documents_ids else []:
        store = np.asarray(store, np.int64)
        own = store[docids[store] == target]
        if len(own) == 0:  # by_item: the target is not in this store
            continue
        el = store[np.asarray([int(d) in u for d in docids[store]], bool)] if len(store) else store
        if len(el) == 0:
            continue
        dist = distance(rows[own[0]], rows[el])
        order = np.lexsort((docids[el], dist))[:want]
        found += [(dist[i], int(docids[el[i]])) for i in order]
    found.sort()
    seen, hits, scores, skipped, n_cand = {int(target)}, [], [], 0, len(u)
    for dist, doc in found:
        if len(hits) == limit:
            break
        if doc in seen:
            continue
        seen.add(doc)
        if skipped < offset:
            skipped += 1
            continue
        score = F32(1) - F32(dist) if isinstance(dist, np.float32) else 1.0 - dist
        if distribution is not None:
            score = shift(distribution, score)
        if threshold is not None and float(score) < threshold:
            n_cand = len(seen) - 2  # (candidates \ {doc}) AND seen: the documents walked before this one
            break
        hits.append(doc)
        scores.append(score)
    return hits, scores, n_cand
