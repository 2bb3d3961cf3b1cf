"""Index images with facet databases for the Sort tests."""
import json
import os

from corpus.facets import FacetImage
from corpus.pyindexgen import IndexImage

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sort_goldens.json")


def load_sort_goldens():
    return json.load(open(GOLDEN))


def golden_images(g):
    """the index of sort.rs create_index(): every document's text field is empty; letter / rank / vague are sortable"""
    img = IndexImage(1)
    fac = FacetImage()
    for name in ("letter", "rank", "vague"):
        fac.fid(name)
    for d, doc in enumerate(g["docs"]):
        img.add_text(d, 0, "")
        for name in ("letter", "rank", "vague"):
            if name in doc:
                fac.add_json(d, name, doc[name])
    img.build()
    fac.build()
    return img, fac


def synthetic_images(n_docs, vocab=2000, seed=0xB200, facet_seed=0x50A7):
    img = IndexImage(1)
    img.add_synthetic(n_docs, vocab, seed=seed)
    img.build()
    fac = FacetImage().add_synthetic(n_docs, seed=facet_seed)
    fac.build()
    return img, fac
