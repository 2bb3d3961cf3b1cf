"""Facet distribution throughput: a synthetic corpus with `price`, `brand` and `tags` facets; batches of keyword queries and of
placeholder searches, each timed without facets and with facets = [brand, price, tags].  A sample of queries is checked against the
CPU specification (tests/facet_spec.py), whose time over that sample is what a caller pays today per query on the host.

Prints one JSON line per workload: end-to-end ms per batch with and without facets (wall clock around b200_search_batch), the facet
kernels' ms and launches per batch, the ordinal reads they need per query (the sum over the candidates of each document's values, over the first 16 queries), and the
specification's ms per query, with the card's name and power limit read in the same run.

usage: python tools/facet_bench.py [--docs 10000000] [--batch 1024] [--steps 3] [--warmup 1] [--check 2]"""
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
from tests.facet_spec import facet_values  # noqa: E402

FIELDS = ["brand", "price", "tags"]


def log(msg):
    print(f"[facet_bench] {msg}", file=sys.stderr, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--check", type=int, default=2, help="queries checked against (and timed through) the CPU specification")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    t0 = time.time()
    img = IndexImage(1)
    img.add_synthetic(a.docs, 1000)
    img.build()
    fac = FacetImage().add_synthetic(a.docs)
    fac.build()
    ix = mb.Index(img, facets=fac)
    log(f"staged ({time.time() - t0:.0f} s)")
    # ordinal reads per document: its number of values in each requested field
    per_doc = np.zeros(a.docs, np.int64)
    for name in FIELDS:
        fid = fac.fields[name]
        for tab in (fac.numbers.get(fid, {}), fac.strings.get(fid, {})):
            for docs in tab.values():
                np.add.at(per_doc, np.asarray(docs, np.int64), 1)
    for name, queries in (("keyword", img.synthetic_queries(a.batch, seed=3)), ("placeholder", [""] * a.batch)):
        rec = {"card": card, "workload": name, "docs": a.docs, "batch": a.batch, "steps": a.steps}
        for facets in (False, True):
            def step(cands=False):
                s = ix.search().query(queries).limit(20)
                if facets:
                    s = s.facets(FIELDS)
                if cands:
                    s = s.with_candidates()
                r = s.execute()
                assert (r.status == 0).all()
                return r
            if facets and a.check:
                r = step(True)
                spec_s = 0.0
                for q in range(min(a.check, a.batch)):
                    cand = set(np.nonzero(np.unpackbits(r.candidates[q].view(np.uint8), bitorder="little")[: a.docs])[0].tolist())
                    t = time.time()
                    want = {n: facet_values(fac, fac.fields[n], cand) for n in FIELDS}
                    spec_s += time.time() - t
                    assert r.facet_distribution(q) == want, q
                rec["spec_ms_per_query"] = round(spec_s * 1e3 / min(a.check, a.batch), 1)
                log(f"{name}: {min(a.check, a.batch)} queries match the specification")
            for _ in range(a.warmup):
                step()
            ix.reset_stats()
            t = time.time()
            for _ in range(a.steps):
                r = step()
            wall = time.time() - t
            k = ix.stats()["kernels"]["facet"]
            tag = "facets" if facets else "plain"
            rec[f"{tag}_e2e_ms_per_batch"] = round(wall * 1e3 / a.steps, 2)
            if facets:
                rec["facet_kernel_ms_per_batch"] = round(k["ms"] / a.steps, 3)
                rec["facet_kernel_count_per_batch"] = k["count"] / a.steps
        # ordinal reads over a sample of the batch's queries (unpacking every bitmap of the batch takes minutes on the host)
        sample = min(16, a.batch)
        r = ix.search().query(queries[:sample]).limit(20).with_candidates().execute()
        reads = sum(int(per_doc[np.unpackbits(r.candidates[q].view(np.uint8), bitorder="little")[: a.docs].astype(bool)].sum()) for q in range(sample))
        rec["ordinal_reads_per_query"] = reads // sample
        rec["mean_candidates"] = float(np.mean(r.n_candidates))
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
