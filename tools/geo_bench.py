"""GeoSort throughput: placeholder searches sorted by `_geoPoint(lat, lng):asc` then `price:asc`, limit 20, in batches of 1024
over a synthetic corpus whose documents all carry `_geo` (coordinates on a 0.01-degree grid, uniform over the sphere).

Prints one JSON line: device q/s (queries over the CUDA-event time of the geo and sort kernels), end-to-end q/s (wall clock
around b200_search_batch with host buffers), the geo kernels' time and algorithmic bytes/s, and the card's name and power limit
read in the same run.

usage: python tools/geo_bench.py [--docs 10000000] [--batch 1024] [--steps 5] [--warmup 2]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import meilisearch_b200 as mb  # noqa: E402
from corpus.facets import FacetImage  # noqa: E402
from corpus.pyindexgen import IndexImage  # noqa: E402


def log(msg):
    print(f"[geo_bench] {msg}", file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--limit", type=int, default=20)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    t0 = time.time()
    img = IndexImage(1)
    img.add_synthetic(a.docs, 1000)
    img.build()
    log(f"index image built ({time.time() - t0:.0f} s)")
    rng = np.random.default_rng(0x6E0)
    docs = np.arange(a.docs, dtype=np.uint32)
    lat = np.round(np.degrees(np.arcsin(rng.uniform(-1, 1, a.docs))), 2)
    lng = np.round(rng.uniform(-180, 180, a.docs), 2)
    fac = FacetImage()
    fac._bulk("_geo.lat", docs, lat, numbers=True)
    fac._bulk("_geo.lng", docs, lng, numbers=True)
    fac._bulk("price", docs, np.round(rng.gamma(2.0, 40.0, a.docs), 1), numbers=True)
    fac.build()
    log(f"facet databases built ({time.time() - t0:.0f} s)")
    ix = mb.Index(img, criteria=["sort"], facets=fac)
    setup_s = time.time() - t0
    log(f"staged ({setup_s:.0f} s)")
    pts = np.stack([np.degrees(np.arcsin(rng.uniform(-1, 1, a.batch))), rng.uniform(-180, 180, a.batch)], 1)
    sorts = [[f"_geoPoint({p[0]:.6f}, {p[1]:.6f}):asc", "price:asc"] for p in pts]

    def step():
        r = ix.search().query([""] * a.batch).sort(sorts).limit(a.limit).execute()
        assert (r.status == 0).all() and (r.n_hits == a.limit).all()

    for i in range(a.warmup):
        t = time.time()
        step()
        log(f"warm-up batch {i}: {time.time() - t:.2f} s")
    ix.reset_stats()
    t = time.time()
    for _ in range(a.steps):
        step()
    wall = time.time() - t
    k = ix.stats()["kernels"]
    q = a.batch * a.steps
    dev_ms = k["geo"]["ms"] + k["sort"]["ms"]
    print(json.dumps({
        "card": card, "docs": a.docs, "batch": a.batch, "steps": a.steps, "limit": a.limit, "setup_s": round(setup_s, 1),
        "device_qps": round(q / (dev_ms * 1e-3), 1), "e2e_qps": round(q / wall, 1),
        "geo_kernel_ms_per_batch": round(k["geo"]["ms"] / a.steps, 3), "geo_launches_per_batch": k["geo"]["count"] / a.steps,
        "geo_bytes_per_s": round(k["geo"]["bytes"] / (k["geo"]["ms"] * 1e-3), 1),
        "sort_kernel_ms_per_batch": round(k["sort"]["ms"] / a.steps, 3)}))


if __name__ == "__main__":
    main()
