"""Filter programs at scale: a synthetic corpus with `price`, `brand` and `tags` facets, a batch of filters mixing equality, range, IN
and two-level AND / OR (one per query, seeded).  Measures, per batch:

* b200_filter_batch alone: the filter kernel's ms (CUDA events) and its algorithmic GB/s (bytes counted by the library, b200_stats);
* keyword searches with the programs (`filter`), end to end (wall clock around b200_search_batch);
* the same searches given the same sets as host bitmaps (`universes`), which is what a caller that evaluates the filter on the CPU
  sends today (the time to build those bitmaps on the CPU is not included).

The first queries of both searches are checked to return the same documents.  Prints one JSON line with the card's name and power
limit read in the same run.

usage: python tools/filter_bench.py [--docs 10000000] [--batch 1024] [--steps 3] [--warmup 1]"""
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


def log(msg):
    print(f"[filter_bench] {msg}", file=sys.stderr, flush=True)


def filters(n, seed=17):
    rng = np.random.default_rng(seed)
    b = lambda: f"brand{int(rng.zipf(1.3)) % 500:03d}"  # noqa: E731
    out = []
    for q in range(n):
        lo = float(np.round(rng.uniform(0, 200), 1))
        k = q % 5
        if k == 0:
            out.append(f"brand = {b()}")
        elif k == 1:
            out.append(f"price {lo} TO {lo + float(rng.uniform(5, 80)):.1f}")
        elif k == 2:
            out.append("brand IN [" + ", ".join(b() for _ in range(5)) + "]")
        elif k == 3:
            out.append(f"(brand = {b()} OR brand = {b()}) AND price > {lo}")
        else:
            out.append(f"tags = tag{int(rng.integers(60)):02d} AND NOT price < {lo} OR tags = {int(rng.integers(200))}")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    t0 = time.time()
    img = IndexImage(1)
    img.add_synthetic(a.docs, 1000)
    img.build()
    fac = FacetImage().add_synthetic(a.docs)
    fac.build()
    fac.build_presence()
    ix = mb.Index(img, facets=fac)
    log(f"staged ({time.time() - t0:.0f} s)")
    fs = filters(a.batch)
    queries = img.synthetic_queries(a.batch, seed=3)
    rec = {"card": card, "docs": a.docs, "batch": a.batch, "steps": a.steps}
    # the filter kernel alone
    for _ in range(a.warmup):
        bitmaps, status, _ = ix.filter_batch(fs)
    assert (status == 0).all()
    ix.reset_stats()
    t = time.time()
    for _ in range(a.steps):
        ix.filter_batch(fs)
    wall = time.time() - t
    k = ix.stats()["kernels"]["filter"]
    rec["filter_kernel_ms_per_batch"] = round(k["ms"] / a.steps, 3)
    rec["filter_kernel_gb_per_s"] = round(k["bytes"] / (k["ms"] * 1e-3) / 1e9, 1) if k["ms"] else None
    rec["filter_batch_e2e_ms_per_batch"] = round(wall * 1e3 / a.steps, 1)  # includes copying the 1024 bitmaps to the host
    rec["mean_matches"] = float(np.mean([int(np.unpackbits(bitmaps[q].view(np.uint8)).sum()) for q in range(0, a.batch, 64)]))
    # keyword searches: with the programs, and with the same sets as host bitmaps
    universes = [bitmaps[q] for q in range(a.batch)]
    for tag, build in (("program", lambda s: s.filter(fs)), ("universes", lambda s: s.universes(universes))):
        def step():
            r = build(ix.search().query(queries).limit(20)).execute()
            assert (r.status == 0).all()
            return r
        for _ in range(a.warmup):
            step()
        t = time.time()
        for _ in range(a.steps):
            r = step()
        wall = time.time() - t
        rec[f"{tag}_e2e_ms_per_batch"] = round(wall * 1e3 / a.steps, 1)
        rec[f"{tag}_qps"] = round(a.batch * a.steps / wall, 1)
        rec[f"{tag}_ids"] = [r.ids(q) for q in range(8)]
    assert rec.pop("program_ids") == rec.pop("universes_ids"), "a program and its bitmap gave different results"
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
