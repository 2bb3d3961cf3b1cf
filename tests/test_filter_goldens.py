"""CPU: the filter specification (tests/filter_spec.py) against the reference's known answers (tests/golden/filter_goldens.json,
written by tests/golden/extract_filter_goldens.py): the `test_filter!` cases of crates/milli/tests/search/filters.rs."""
import pytest

from tests.filter_fixtures import geo_spec, golden_images, golden_tree, load_filter_goldens
from tests.filter_spec import FilterSpec, Unsupported


def test_filter_goldens_on_the_spec():
    g = load_filter_goldens()
    assert len(g["cases"]) == 49
    img, fac = golden_images(g)
    spec = FilterSpec(fac, range(img.n_docs), geo_spec(fac, img.n_docs))
    ext = [d["id"] for d in g["docs"]]
    for c in g["cases"]:
        tree = golden_tree(c["filter"])
        if c["name"].startswith("starts_with"):  # STARTS WITH is outside the implemented scope
            with pytest.raises(Unsupported):
                spec.evaluate(tree)
            continue
        assert sorted(ext[d] for d in spec.evaluate(tree)) == c["ids"], c["name"]
