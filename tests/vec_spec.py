"""Reference models of the vector stage (`Index.nns_by_vector`), numpy only.

The specification is the oracle's `cosine_distance` / `nns_by_vector` (arroy/hannoy `Cosine`): distance = (1 - cos) / 2 in f32,
cos clamped to [-1, 1], distance 0 unless |q||v| > f32::EPSILON; results ascending by (distance, docid), restricted to the
candidate bitmap.  Two references check the device against it:

R1, a float32 replica of the device formula, for exact-arithmetic inputs (`ExactGen`).  Every component is m * 2^(s - 4) with
m an integer in [-3, 3] and one power-of-two scale s per vector, so every product of a row with a query is an integer multiple of
the same power of two, and every partial sum of their dot is an integer of at most 9 d <= 13 824 < 2^14 such units: the f32 dot is
exact whatever the summation order or accumulator (wgmma's included), and so is every sum of squares.  The components are exact in
fp16 too (multiples of 2^-24, none above 2^15).  With IEEE sqrt and division (the library is built without fast-math), every
distance the device computes is then determined, and both GPU paths must reproduce R1 bit for bit:
    inv = 1 / sqrt(sum x^2) (0 for a zero vector), pn = inv_v * inv_q,
    dd = (1 - clip(dot * pn, -1, 1)) * 0.5 if 0 < pn < 2^23 else 0.
The last condition is the device form of the norm rule: 1 / (|q||v|) < 2^23 <=> |q||v| > 2^-23, up to rounding within an ulp of
the boundary.  `ExactGen` keeps every product |q||v| a factor of 2 away from 2^-23 (`rule_margin_ok`), where both forms agree.

R2, a float64 reference with the documented quantisation, for realistic inputs: rows rounded to fp16, their norms taken from the
rows as staged (f32 rows: the f32 values); the GEMV path takes the dot with the f32 query, the wgmma path with the query rounded
to fp16, both the norm of the f32 query.  A device result is checked as a certificate (`check_certificate`).  The tolerance
TOL(d) = (d + 8) 2^-24 on a distance follows from the usual bound on a float32 sum of d products, |err| <= d u sum|q_i v_i|
<= d u |q||v| with u = 2^-24 (Cauchy-Schwarz): relative to |q||v| the dot is off by at most d u; each sum of squares is off by at
most d u relative, which moves its inverse square root by d u / 2, and the sqrt, the division and the product of the two inverse
norms add about 3 u; so the cosine is off by at most (2 d + 6) u and the distance, half of (1 - cos), by (d + 3) u plus one
rounding.  The slack up to d + 8 covers the clamp and the final rounding.  A dropped k-block, a swizzle error or a lost row moves
distances by orders of magnitude more.
"""
import numpy as np

F32 = np.float32
EPS = 2.0 ** -23  # f32::EPSILON
PN_MAX = F32(2.0 ** 23)


def tol(d):
    return (d + 8) * 2.0 ** -24


# ------------------------------------------------------------------------------------------------ exact-arithmetic inputs
class ExactGen:
    """Rows and queries with exact f32 dots and norms (see the module docstring).

    Norm classes, so that every product |q||v| is a factor of 2 away from EPS = 2^-23:
      normal rows      |v| >= 2^-14 and not in (1, 4)
      normal queries   |q| >= 2^-8 and not in (1, 4)
      tiny vectors     one component +-2^-24 (|x| = 2^-24)
      zero vectors
    Then normal x normal >= 2^-22; tiny x normal is <= 2^-24 (normal norm <= 1) or >= 2^-22 (>= 4); tiny x tiny = 2^-48.
    """

    def __init__(self, d, seed):
        self.d = d
        self.rng = np.random.default_rng(seed)

    @staticmethod
    def band(x, lo):
        """scale each row of x by a power of two so that its norm is >= lo and not in (1, 4); zero rows stay zero"""
        x = x.copy()
        for i in range(len(x)):
            s = float(np.sqrt(np.dot(x[i].astype(np.float64), x[i].astype(np.float64))))
            if s == 0:
                continue
            while s < lo:
                x[i] *= 4
                s *= 4
            if 1 < s < 4:
                x[i] *= 4 if s * 4 <= 48 else 0.25
                s = s * 4 if s * 4 <= 48 else s / 4
        return x

    def _raw(self, n, lo, e_lo, e_hi):
        m = self.rng.integers(-3, 4, (n, self.d)).astype(np.float32)
        e = self.rng.integers(e_lo, e_hi + 1, n)
        return self.band(m * np.exp2(e - 4).astype(np.float32)[:, None], lo)

    def rows(self, n):
        return self._raw(n, 2.0 ** -14, -10, 6)

    def queries(self, n):
        return self._raw(n, 2.0 ** -8, -10, 6)

    def tiny(self, n):
        x = np.zeros((n, self.d), np.float32)
        x[np.arange(n), self.rng.integers(0, self.d, n)] = self.rng.choice([-1.0, 1.0], n) * 2.0 ** -24
        return x

    def scaled(self, x, lo):
        """copies of x scaled by 2^+-k (same cosine with every query, so exact ties), kept in their norm class"""
        k = self.rng.integers(-3, 4, len(x))
        y = x * np.exp2(k).astype(np.float32)[:, None]
        y = self.band(y, lo)
        assert np.abs(y).max(initial=0) <= 2.0 ** 15
        return y

    def mixed_rows(self, n, dup=0.1, scaled=0.05, zero=0.02, tiny=0.02):
        """normal rows with exact duplicates, scaled copies, zero rows and tiny rows mixed in at random positions"""
        x = self.rows(n)
        if n == 0:
            return x
        kinds = self.rng.random(n)
        src = self.rng.integers(0, n, n)
        c1, c2, c3 = dup, dup + scaled, dup + scaled + zero
        a = kinds < c1
        x[a] = x[src[a]]
        b = (kinds >= c1) & (kinds < c2)
        x[b] = self.scaled(x[src[b]], 2.0 ** -14)
        x[(kinds >= c2) & (kinds < c3)] = 0
        t = (kinds >= c3) & (kinds < c3 + tiny)
        x[t] = self.tiny(int(t.sum()))
        return x

    def mixed_queries(self, nq, rows):
        """normal queries, plus (when there is room) queries equal to rows, a zero query, a tiny query and a small one"""
        q = self.queries(nq)
        extra = []
        if len(rows):
            pick = rows[self.rng.integers(0, len(rows), 3)]
            extra += [self.band(pick, 2.0 ** -8)]
        extra += [np.zeros((1, self.d), np.float32), self.tiny(1)]
        small = self.band(self.queries(1), 2.0 ** -8)
        small *= np.float32(2.0 ** -np.ceil(np.log2(max(float(np.linalg.norm(small)), 1e-30))))  # |q| in (1/2, 1]
        extra.append(small.astype(np.float32))
        e = np.concatenate(extra)[: max(0, nq - 1)]
        q[1: 1 + len(e)] = e
        return q

    def docids(self, n, n_docs, dup=0.02, beyond=0.02):
        """a permutation of [0, n) with some duplicate docids and some at or beyond n_docs"""
        ids = self.rng.permutation(max(n, 1))[:n].astype(np.int64)
        r = self.rng.random(n)
        ids[r < dup] = ids[self.rng.integers(0, max(n, 1), int((r < dup).sum()))]
        b = r > 1 - beyond
        ids[b] = n_docs + self.rng.integers(0, 3 * max(n, 64), int(b.sum()))
        return ids.astype(np.uint32)


def exact_dots(rows, queries):
    """queries x rows in float32; exact on ExactGen data (checked by the CPU tests against float64)"""
    return (queries.astype(np.float32) @ rows.astype(np.float32).T).astype(np.float32)


def inv_norms(x):
    """1 / sqrt(sum x^2) in f32 (0 for a zero vector); on exact inputs the f32 sum of squares is exact"""
    s = np.einsum("ij,ij->i", x.astype(np.float64), x.astype(np.float64)).astype(np.float32)
    n = np.sqrt(s)
    out = np.zeros(len(x), np.float32)
    nz = n > 0
    out[nz] = F32(1) / n[nz]
    return out


def rule_margin_ok(rows, queries):
    """every |q||v| with both norms non-zero is a factor of 2 away from EPS"""
    nv = np.sqrt(np.einsum("ij,ij->i", rows.astype(np.float64), rows.astype(np.float64)))
    nq = np.sqrt(np.einsum("ij,ij->i", queries.astype(np.float64), queries.astype(np.float64)))
    p = nq[:, None] * nv[None, :]
    return not ((p > EPS / 2) & (p < EPS * 2)).any()


def r1_distances(rows, queries):
    """[nq, n] f32 distances of the device formula (exact inputs)"""
    with np.errstate(invalid="ignore", over="ignore"):
        pn = inv_norms(queries)[:, None] * inv_norms(rows)[None, :]
        cs = np.clip(exact_dots(rows, queries) * pn, F32(-1), F32(1))
        dd = (F32(1) - cs) * F32(0.5)
    return np.where((pn > 0) & (pn < PN_MAX), dd, F32(0)).astype(np.float32)


def eligible(docids, cand):
    """rows whose docid the candidate bitmap (uint64 words, None = all) holds; bits past its end are absent"""
    if cand is None:
        return np.ones(len(docids), bool)
    cand = np.asarray(cand, np.uint64)
    w = docids.astype(np.int64) >> 6
    ok = w < len(cand)
    out = np.zeros(len(docids), bool)
    out[ok] = ((cand[w[ok]] >> (docids[ok].astype(np.uint64) & np.uint64(63))) & np.uint64(1)).astype(bool)
    return out


def topk(dist, docids, k, cand=None):
    """(ids [nq, k], dist [nq, k], counts [nq]) ordered by (distance, docid), as nns_by_vector returns them"""
    nq = dist.shape[0]
    ids = np.zeros((nq, k), np.uint32)
    dd = np.zeros((nq, k), np.float32)
    cnt = np.zeros(nq, np.uint32)
    el = np.nonzero(eligible(docids, cand))[0]
    for q in range(nq):
        o = el[np.lexsort((docids[el], dist[q, el]))][:k]
        cnt[q] = len(o)
        ids[q, : len(o)] = docids[o]
        dd[q, : len(o)] = dist[q, o]
    return ids, dd, cnt


def r1(rows, docids, queries, k, cand=None):
    return topk(r1_distances(rows, queries), docids, k, cand)


def bitmap(docs, n_words=None):
    docs = np.asarray(docs, np.int64)
    n = n_words if n_words is not None else (int(docs.max(initial=-1)) >> 6) + 1
    w = np.zeros(n, np.uint64)
    for x in docs:
        if (x >> 6) < n:
            w[x >> 6] |= np.uint64(1) << np.uint64(x & 63)
    return w


# ------------------------------------------------------------------------------------------------ float64 certificates
def r2_distances(rows, queries, path, rows_f16=False):
    """[nq, n] float64 distances with the device's quantisation ("gemv" or "wgmma"); rows_f16: staged as fp16 (norms of the
    fp16 values) rather than from f32"""
    r16 = rows.astype(np.float16).astype(np.float64)
    rn = np.linalg.norm(r16 if rows_f16 else rows.astype(np.float64), axis=1)
    q64 = queries.astype(np.float64)
    qd = queries.astype(np.float16).astype(np.float64) if path == "wgmma" else q64
    qn = np.linalg.norm(q64, axis=1)
    p = qn[:, None] * rn[None, :]
    with np.errstate(invalid="ignore", divide="ignore"):
        cs = np.clip((qd @ r16.T) / p, -1, 1)
    return np.where(p > EPS, (1 - cs) / 2, 0.0)


def check_certificate(ids, dist, cnt, docids, r2, k, d, cand=None, ctx=None):
    """The device result of every query against R2: count, order, each distance within TOL(d) of R2's for that row, and no
    eligible row left out that R2 places clearly (by more than 2 TOL) before the last one returned."""
    t = tol(d)
    el = eligible(docids, cand)
    n_el = int(el.sum())
    row_of = {}
    for r in np.nonzero(el)[0]:
        row_of.setdefault(int(docids[r]), []).append(r)
    for q in range(r2.shape[0]):
        c = int(cnt[q])
        assert c == min(k, n_el), (ctx, q, c, k, n_el)
        gi, gd = ids[q, :c], dist[q, :c].astype(np.float64)
        key = gd + 0.0
        assert all((key[i], gi[i]) <= (key[i + 1], gi[i + 1]) for i in range(c - 1)), (ctx, q, "order")
        used = np.zeros(len(docids), bool)
        worst = -np.inf
        for i in range(c):
            rs = [r for r in row_of.get(int(gi[i]), []) if not used[r]]
            assert rs, (ctx, q, i, int(gi[i]), "id not an eligible row")
            r = min(rs, key=lambda r: abs(r2[q, r] - gd[i]))
            assert abs(r2[q, r] - gd[i]) <= t, (ctx, q, i, int(gi[i]), float(gd[i]), float(r2[q, r]), t)
            used[r] = True
            worst = max(worst, r2[q, r])
        left = el & ~used
        if c and left.any():
            assert r2[q, left].min() >= worst - 2 * t, (ctx, q, float(r2[q, left].min()), float(worst))
