"""GPU: the reference's filter known answers (tests/golden/filter_goldens.json) through b200_filter_batch and b200_search_batch."""
import numpy as np
import pytest

import meilisearch_b200 as mb
from tests.filter_fixtures import golden_images, golden_tree, load_filter_goldens

pytestmark = pytest.mark.gpu


def test_filter_goldens_on_the_device():
    g = load_filter_goldens()
    img, fac = golden_images(g)
    ix = mb.Index(img, facets=fac)
    ext = [d["id"] for d in g["docs"]]
    trees = [golden_tree(c["filter"]) for c in g["cases"]]
    unsupported = [c["name"].startswith("starts_with") for c in g["cases"]]
    out, status, _ = ix.filter_batch(trees)
    n = len(trees)
    r = ix.search().query([""] * n).limit(len(ext)).filter(trees).execute()
    for i, c in enumerate(g["cases"]):
        if unsupported[i]:
            assert status[i] == -4 and r.status[i] == -4, c["name"]
            continue
        assert status[i] == 0 and r.status[i] == 0, (c["name"], ix.last_error())
        bits = np.unpackbits(out[i].view(np.uint8), bitorder="little")[: img.n_docs]
        assert sorted(ext[d] for d in np.nonzero(bits)[0]) == c["ids"], c["name"]
        assert sorted(ext[d] for d in r.ids(i)) == c["ids"], c["name"]
        assert r.n_candidates[i] == len(c["ids"]), c["name"]
