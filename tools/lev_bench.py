"""Term derivation alone on the benchmark's cfg 3 query batches: lev_match time, the (term, word) pairs the work items cover
against the full term x dictionary cross product, and work items per derivation wave.

The derivations are those of a keyword search of each batch (the same terms and waves as the hybrid benchmark's keyword stage),
timed with the per-kernel CUDA events of one lane.  Usage: python tools/lev_bench.py [--docs N] [--vocab V] [--repeat R]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_500_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--distinct-batches", type=int, default=4)
    ap.add_argument("--repeat", type=int, default=3, help="timed passes over the batches")
    args = ap.parse_args()

    import meilisearch_b200 as mb
    from corpus.pyindexgen import synthetic_image
    from meilisearch_b200.tokenizer import TokenBatch

    mb.load_library()
    img = synthetic_image(args.docs, args.vocab, seed=0xB200)
    batches = [TokenBatch(img.synthetic_queries(args.batch, seed=i)) for i in range(args.distinct_batches)]
    ix = mb.Index(img)
    os.environ["B200_SINGLE_LANE"] = "1"
    os.environ["B200_KERNEL_TIMERS"] = "1"
    for b in batches:  # warm-up
        ix.search().query(b).execute()
    ix.reset_stats()
    t = time.perf_counter()
    for _ in range(args.repeat):
        for b in batches:
            ix.search().query(b).execute()
    wall = time.perf_counter() - t
    st = ix.stats()
    n = args.repeat * len(batches)
    lev = st["kernels"]["lev_match"]
    waves = max(1, lev["count"])
    cross = st["lev_terms"] * img.n_words
    print(json.dumps({
        "batches": n, "n_words": img.n_words,
        "lev_match_ms_per_batch": lev["ms"] / n, "lev_match_ms_per_wave": lev["ms"] / waves, "waves_per_batch": waves / n,
        "terms_per_wave": st["lev_terms"] / waves, "work_items_per_wave": st["lev_items"] / waves,
        "pairs_per_wave": st["lev_pairs"] / waves, "cross_product_per_wave": cross / waves,
        "pairs_over_cross_product": st["lev_pairs"] / max(1, cross),
        "host_derive_ms_per_batch": st["host_ms"]["derive"] / n, "batch_wall_ms": 1e3 * wall / n,
    }))
    ix.close()


if __name__ == "__main__":
    main()
