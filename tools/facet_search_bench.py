"""Facet search throughput: batches of facet-search requests (b200_facet_search_batch) over all documents of a synthetic corpus with
`brand` (500 values) and `model` (a high-cardinality string field).  Three workloads: 1-3 byte prefixes on `model`, typo'd 6-10 byte
queries on `model`, and no query on `brand`.  With --check N, N sampled requests of each workload are compared with the CPU
specification (tests/facet_search_spec.py) before anything is timed.

Prints one JSON line per workload with the card's name and power limit read in the same run: the facet-search kernels' ms per batch
(b200_stats, match + count + select together), end-to-end ms per batch (wall clock around the call, host decoding included),
device and end-to-end requests per second, and the kernels' algorithmic bytes per batch.

usage: python tools/facet_search_bench.py [--docs 10000000] [--values 100000] [--batch 1024] [--steps 5] [--warmup 1] [--check 4]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import meilisearch_b200 as mb  # noqa: E402
from corpus.facets import FacetImage  # noqa: E402
from corpus.pyindexgen import IndexImage  # noqa: E402
from tests.facet_search_spec import facet_search  # noqa: E402


def log(msg):
    print(f"[facet_search_bench] {msg}", file=sys.stderr, flush=True)


def typo(rng, w):
    """one random edit (substitution, deletion, insertion or transposition) inside w"""
    i = int(rng.integers(1, len(w) - 1))
    op = int(rng.integers(4))
    c = chr(ord("a") + int(rng.integers(26)))
    return [w[:i] + c + w[i + 1:], w[:i] + w[i + 1:], w[:i] + c + w[i:], w[:i - 1] + w[i] + w[i - 1] + w[i + 1:]][op]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--values", type=int, default=100_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=4, help="requests per workload checked against the CPU specification")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    t0 = time.time()
    img = IndexImage(1)
    img.add_synthetic(a.docs, 1000)
    img.build()
    fac = FacetImage().add_synthetic(a.docs).add_synthetic_search(a.docs, n_values=a.values)
    fac.build()
    fac.build_search()
    ix = mb.Index(img, facets=fac)
    log(f"staged ({time.time() - t0:.0f} s)")
    rng = np.random.default_rng(5)
    models = sorted(fac.strings[fac.fields["model"]])
    long_models = [m for m in models if 6 <= len(m) <= 10]
    workloads = [
        ("prefix_1_3_bytes", "model", [m[:int(rng.integers(1, 4))] for m in rng.choice(models, a.batch)]),
        ("typo_6_10_bytes", "model", [typo(rng, m) for m in rng.choice(long_models, a.batch)]),
        ("none_brand", "brand", [None] * a.batch),
    ]
    all_docs = range(a.docs)
    for name, field, queries in workloads:
        if a.check:
            got, status = ix.facet_search([None] * a.check, field, queries[:a.check], order="count", max_values=100)
            for i in range(a.check):
                want = facet_search(fac, fac.fields[field], all_docs, queries[i], order="count", max_values=100)
                if status[i] != 0 or got[i] != want:
                    raise SystemExit(f"{name}: request {i} ({queries[i]!r}) differs from the specification")
            log(f"{name}: {a.check} requests match the specification")
        cands = [None] * a.batch
        for _ in range(a.warmup):
            ix.facet_search(cands, field, queries, order="count", max_values=100)
        ix.reset_stats()
        t = time.perf_counter()
        for _ in range(a.steps):
            _, status = ix.facet_search(cands, field, queries, order="count", max_values=100)
        wall = (time.perf_counter() - t) / a.steps * 1e3
        k = ix.stats()["kernels"]["facet_search"]
        dev = k["ms"] / a.steps
        print(json.dumps({"card": card, "workload": name, "docs": a.docs, "values": len(models) if field == "model" else None,
                          "batch": a.batch, "steps": a.steps, "errors": int((status != 0).sum()), "kernel_ms_per_batch": round(dev, 3),
                          "e2e_ms_per_batch": round(wall, 3), "device_qps": round(a.batch / dev * 1e3), "e2e_qps": round(a.batch / wall * 1e3),
                          "algorithmic_bytes_per_batch": k["bytes"] // a.steps}), flush=True)


if __name__ == "__main__":
    main()
