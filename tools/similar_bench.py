"""`/similar` against semantic search on the cfg 3 store (10 M x 768 fp16 rows, seeded): 1024 targets through Index.similar, and a
semantic batch of the same 1024 vectors (the f32 copies of the targets' rows), alternated round by round in one process.  Both scan
with the same k (similar: offset + limit + 2 = 22; semantic: limit 22).  Prints one JSON line per workload: device time per batch
(CUDA events of the library's vector kernels), wall time per batch, queries/s and host-to-device bytes per batch.

usage: python tools/similar_bench.py [--docs N] [--rounds R] [--warmup W]"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import meilisearch_b200 as mb  # noqa: E402
from corpus.pyindexgen import IndexImage, synthetic_embeddings_f16  # noqa: E402

DIM, BATCH, LIMIT = 768, 1024, 20


def gpu_name():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip() if out.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    img = IndexImage(1)
    img.add_synthetic(a.docs, 1000, len_lo=1, len_hi=1, seed=7)  # documents_ids covers every row; the text is not read
    img.build()
    ix = mb.Index(img)
    emb = synthetic_embeddings_f16(a.docs, DIM, seed=0xE5BED)
    ix.set_embeddings(emb)
    targets = np.random.default_rng(5).choice(a.docs, BATCH, replace=False).astype(np.uint32)
    vectors = emb[targets].astype(np.float32)

    def similar():
        return ix.similar(targets, limit=LIMIT)

    def semantic():
        return ix.search().semantic(vectors).limit(LIMIT + 2).execute()

    runs = {"similar": similar, "semantic": semantic}
    acc = {k: {"device_ms": 0.0, "wall_ms": 0.0, "h2d_bytes": 0} for k in runs}
    for r in range(a.warmup + a.rounds):
        for name, fn in runs.items():
            ix.reset_stats()
            t0 = time.perf_counter()
            res = fn()  # returns after the library's stream synchronise
            wall = (time.perf_counter() - t0) * 1e3
            st = ix.stats()
            assert (res.status == 0).all()
            if r >= a.warmup:
                acc[name]["device_ms"] += sum(k["ms"] for k in st["kernels"].values())
                acc[name]["wall_ms"] += wall
                acc[name]["h2d_bytes"] += st["h2d_bytes"]
    card = gpu_name()
    for name, v in acc.items():
        dev, wall = v["device_ms"] / a.rounds, v["wall_ms"] / a.rounds
        print(json.dumps({"workload": name, "docs": a.docs, "dim": DIM, "batch": BATCH, "device_ms": round(dev, 3), "wall_ms": round(wall, 3),
                          "qps_wall": round(BATCH / (wall * 1e-3), 1), "h2d_bytes": v["h2d_bytes"] // a.rounds, "gpu": card}))


if __name__ == "__main__":
    main()
