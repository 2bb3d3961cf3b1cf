"""SURVEY §8(d) cfg 4 matrix: N in {1e5, 1e6, 1e7} x 768 fp16 rows (i.i.d. N(0,1), L2-normalised), B in {1, 16, 1024} query vectors,
k = 100, with and without a 10 %-density candidate bitmap.  Per cell: kernel time (CUDA events), achieved HBM GB/s (B < 16, GEMV
kernel) or TFLOP/s (B >= 16, wgmma kernel) against the measured peaks, end-to-end ms per batch through the C ABI, and parity
with the CPU oracle on a bounded number of queries (scores within 1e-4 relative; ids equal except where the oracle's scores tie
within that tolerance).  Prints one JSON line per cell."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import meilisearch_b200 as mb
from corpus.pyindexgen import IndexImage, synthetic_embeddings_f16
from meilisearch_b200.tokenizer import TokenBatch
from oracle.pyoracle import OracleIndex

peaks = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}
D, K = 768, 100
sizes = [int(float(x)) for x in os.environ.get("CFG4_N", "1e5,1e6,1e7").split(",")]
for N in sizes:
    img = IndexImage(1)
    img.add_synthetic(N, 100, len_lo=1, len_hi=1, seed=1)   # N documents (docids 0..N-1); the text does not matter here
    img.build()
    emb = synthetic_embeddings_f16(N, D, seed=0xE5BED)
    ix = mb.Index(img)
    ix.set_embeddings(emb)
    o = OracleIndex(img)
    o.set_embeddings(emb)
    rng = np.random.default_rng(N)
    mask = np.zeros((N + 63) // 64, np.uint64)
    keep = np.nonzero(rng.random(N) < 0.1)[0]
    np.bitwise_or.at(mask, keep >> 6, np.uint64(1) << (keep & 63).astype(np.uint64))
    for B in (1, 16, 1024):
        q = rng.standard_normal((B, D), dtype=np.float32)
        for cand, label in ((None, "none"), (mask, "10%")):
            for _ in range(3):
                ix.nns_by_vector(q, K, cand)
            ix.reset_stats()
            reps = 5 if N >= 10**7 else 10
            t0 = time.perf_counter()
            for _ in range(reps):
                ids, dist, cnt = ix.nns_by_vector(q, K, cand)
            wall = time.perf_counter() - t0
            ks = ix.stats()["kernels"]
            cell = {"N": N, "d": D, "B": B, "k": K, "mask": label, "e2e_ms_per_batch": 1e3 * wall / reps}
            if ks["vec_gemm_topk"]["count"]:
                ms = ks["vec_gemm_topk"]["ms"] / ks["vec_gemm_topk"]["count"]
                tf = 2.0 * ((B + 63) // 64 * 64) * N * D / (ms * 1e-3) / 1e12
                cell.update({"kernel": "vec_gemm_topk", "kernel_ms": ms, "tflops": tf, "frac_of_bf16_peak": tf / peaks["bf16_tflops"]})
            else:
                kd = ks["vec_dist"]
                ms = kd["ms"] / kd["count"]
                gbs = kd["bytes"] / (kd["ms"] * 1e-3) / 1e9
                cell.update({"kernel": "vec_dist (+topk_select %.3f ms)" % (ks["topk_select"]["ms"] / max(1, ks["topk_select"]["count"])), "kernel_ms": ms,
                             "launches_per_batch": kd["count"] / reps, "gbs": gbs, "frac_of_hbm_peak": gbs / peaks["hbm_gbs"]})
            # parity on a bounded number of queries
            nchk = min(B, 8 if cand is None else (4 if N < 10**7 else 2))
            bad = 0
            if cand is None:
                want = o.search_batch(TokenBatch([""] * nchk), vectors=np.ascontiguousarray(q[:nchk]), vector_only=True, limit=K, scoring="detailed", n_threads=os.cpu_count() or 1)
                for i in range(nchk):
                    oid = want.ids(i)
                    od = np.array([1.0 - s[0][1] for s in want.scores(i)], np.float32)
                    ok = cnt[i] == len(oid) and np.allclose(1 - dist[i, : cnt[i]], 1 - od, rtol=1e-4, atol=2e-5)
                    for j in np.nonzero(ids[i, : cnt[i]] != np.array(oid, np.uint32))[0] if ok else []:
                        ok = ok and abs(od[j] - dist[i, j]) <= 1e-4 * max(1 - od[j], 1e-3) + 2e-5
                    bad += 0 if ok else 1
            else:
                for i in range(nchk):
                    oid, od = o.nns(q[i], K, cand)
                    ok = cnt[i] == len(oid) and np.allclose(1 - dist[i, : cnt[i]], 1 - od, rtol=1e-4, atol=2e-5)
                    for j in np.nonzero(ids[i, : cnt[i]] != oid)[0] if ok else []:
                        ok = ok and abs(od[j] - dist[i, j]) <= 1e-4 * max(1 - od[j], 1e-3) + 2e-5
                    bad += 0 if ok else 1
            cell["parity"] = {"checked": nchk, "mismatches": bad}
            print(json.dumps(cell), flush=True)
    ix.close()
    del o, emb
