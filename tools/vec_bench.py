"""Tiny driver for profiling the vector stage alone (1e6 x 768 fp16, B=1 and B=8)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import meilisearch_b200 as mb
from corpus.pyindexgen import IndexImage

img = IndexImage(1)
img.add_text(0, 0, "placeholder")
img.build()
ix = mb.Index(img)
rng = np.random.default_rng(0)
n, d = int(os.environ.get("VEC_N", "1000000")), 768
emb = rng.standard_normal((n, d), dtype=np.float32)
ix.set_embeddings(emb)
q = rng.standard_normal((8, d), dtype=np.float32)
if os.environ.get("VEC_GEMM_ONLY"):
    qq = rng.standard_normal((1024, d), dtype=np.float32)
    for i in range(4):
        ix.nns_by_vector(qq, 100)
    sys.exit(0)
for i in range(6):
    ix.nns_by_vector(q[:1], 100)
ix.reset_stats()
for i in range(10):
    ix.nns_by_vector(q[i % 8: i % 8 + 1], 100)
s = ix.stats()["kernels"]["vec_dist"]
print("B=1: %.3f ms/launch, %.1f GB/s" % (s["ms"] / s["count"], s["bytes"] / (s["ms"] * 1e-3) / 1e9))
ix.reset_stats()
for i in range(5):
    ix.nns_by_vector(q, 100)
s = ix.stats()["kernels"]["vec_dist"]
print("B=8: %.3f ms/launch, %.1f GB/s" % (s["ms"] / s["count"], s["bytes"] / (s["ms"] * 1e-3) / 1e9))

# batched stage: wgmma GEMM + fused top-k
for B in (128, 1024):
    qq = rng.standard_normal((B, d), dtype=np.float32)
    os.environ["B200_VEC_GEMM"] = "1"
    for i in range(3):
        ix.nns_by_vector(qq, 100)
    ix.reset_stats()
    for i in range(5):
        ix.nns_by_vector(qq, 100)
    s = ix.stats()["kernels"]["vec_gemm_topk"]
    ms = s["ms"] / s["count"]
    bp = (B + 63) // 64 * 64
    print("B=%d gemm+merge: %.3f ms/launch, %.1f TFLOP/s (padded %d), %.0f queries/s kernel-only" % (B, ms, 2.0 * bp * n * d / (ms * 1e-3) / 1e12, bp, B / (ms * 1e-3)))
