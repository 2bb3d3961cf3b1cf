"""Geo filter throughput: batches of placeholder searches, each with one `_geoRadius` (radii log-uniform from 100 m to 500 km around
random points), over a synthetic corpus whose documents all carry `_geo` (0.01-degree grid, uniform over the sphere); once unsorted,
once sorted by `_geoPoint` around the same point; then a batch of bounding boxes.  A sample of queries is checked against the CPU
specification (tests/geo_filter_spec.py) first.

Prints one JSON line per workload: the geo filter kernels' ms per batch and launches, their algorithmic bytes and the fraction of
HBM peak (3.35 TB/s, H100 SXM data sheet) those bytes would take, device q/s (queries over the CUDA-event time of every kernel of
the batch) and end-to-end q/s (wall clock around b200_search_batch), with the card's name and power limit read in the same run.

usage: python tools/geo_filter_bench.py [--docs 10000000] [--batch 1024] [--steps 3] [--warmup 1] [--check 1]"""
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
from corpus.facets import FacetImage, geo_points  # noqa: E402
from corpus.pyindexgen import IndexImage  # noqa: E402

HBM_PEAK = 3.35e12


def log(msg):
    print(f"[geo_filter_bench] {msg}", file=sys.stderr, flush=True)


def spec_index(fac, n_docs):
    """the CPU specification over the corpus (pure Python: about a minute at 10 M documents)"""
    from tests.geo_filter_spec import GeoFilterIndex
    from tests.geo_spec import GeoIndex
    from tests.sort_spec import FacetDbs

    gix = GeoIndex(geo_points(fac, fac.fields["_geo.lat"], fac.fields["_geo.lng"]))
    return GeoFilterIndex(FacetDbs(fac.f64_db, fac.string_db), gix, n_docs, fac.fields["_geo.lat"], fac.fields["_geo.lng"])


def check(ix, spec, n_docs, clauses, got_cand, sample):
    """the first `sample` queries: candidate counts and b200_geo_filter_batch's bitmaps against the specification"""
    for q in range(sample):
        want = spec.filtered_universe([mb.parse_geo_filter(clauses[q])])
        assert int(got_cand[q]) == len(want), (clauses[q], int(got_cand[q]), len(want))
        out, st = ix.geo_filter([clauses[q]])
        bits = np.unpackbits(out[0].view(np.uint8), bitorder="little")[:n_docs]
        assert st[0] == 0 and set(np.nonzero(bits)[0].tolist()) == want, clauses[q]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--limit", type=int, default=20)
    ap.add_argument("--check", type=int, default=1, help="queries checked against the CPU specification (0: none)")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    t0 = time.time()
    img = IndexImage(1)
    img.add_synthetic(a.docs, 1000)
    img.build()
    rng = np.random.default_rng(0x6E0)
    docs = np.arange(a.docs, dtype=np.uint32)
    fac = FacetImage()
    fac._bulk("_geo.lat", docs, np.round(np.degrees(np.arcsin(rng.uniform(-1, 1, a.docs))), 2), numbers=True)
    fac._bulk("_geo.lng", docs, np.round(rng.uniform(-180, 180, a.docs), 2), numbers=True)
    fac.build()
    ix = mb.Index(img, criteria=["sort"], facets=fac)
    log(f"staged ({time.time() - t0:.0f} s)")
    pts = np.stack([np.degrees(np.arcsin(rng.uniform(-1, 1, a.batch))), rng.uniform(-180, 180, a.batch)], 1)
    radii = np.exp(rng.uniform(np.log(100.0), np.log(500_000.0), a.batch))
    radius = [f"_geoRadius({p[0]:.6f}, {p[1]:.6f}, {r:.3f})" for p, r in zip(pts, radii)]
    sorts = [[f"_geoPoint({p[0]:.6f}, {p[1]:.6f}):asc"] for p in pts]
    half = rng.uniform(0.05, 5.0, (a.batch, 2))
    boxes = [f"_geoBoundingBox([{min(90.0, p[0] + h[0]):.6f}, {((p[1] + h[1] + 180) % 360) - 180:.6f}], "
             f"[{max(-90.0, p[0] - h[0]):.6f}, {((p[1] - h[1] + 180) % 360) - 180:.6f}])" for p, h in zip(pts, half)]
    spec = None
    for name, clauses, sort in (("radius", radius, None), ("radius+geosort", radius, sorts), ("box", boxes, None)):
        def step():
            s = ix.search().query([""] * a.batch).geo_filter([[c] for c in clauses]).limit(a.limit)
            if sort is not None:
                s = s.sort(sort)
            r = s.execute()
            assert (r.status == 0).all()
            return r

        r = step()
        if a.check:
            spec = spec if spec is not None else spec_index(fac, a.docs)
            check(ix, spec, a.docs, clauses, r.n_candidates, min(a.check, a.batch))
            log(f"{name}: {min(a.check, a.batch)} queries match the specification")
        for _ in range(a.warmup):
            step()
        ix.reset_stats()
        t = time.time()
        for _ in range(a.steps):
            step()
        wall = time.time() - t
        st = ix.stats()
        k = st["kernels"]
        q = a.batch * a.steps
        dev_ms = sum(v["ms"] for v in k.values())
        gf = k["geo_filter"]
        rec = {"card": card, "workload": name, "docs": a.docs, "batch": a.batch, "steps": a.steps,
               "geo_filter_ms_per_batch": round(gf["ms"] / a.steps, 3), "geo_filter_launches_per_batch": gf["count"] / a.steps,
               "geo_filter_gb_per_batch": round(gf["bytes"] / a.steps / 1e9, 3),
               "geo_filter_hbm_fraction": round(gf["bytes"] / HBM_PEAK / (gf["ms"] * 1e-3), 4),
               "device_qps": round(q / (dev_ms * 1e-3), 1), "e2e_qps": round(q / wall, 1),
               "mean_candidates": float(np.mean(r.n_candidates))}
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
