"""Every degenerate-lens case of tests/lens_edges.py reaches the edge it is there for, computed on the host from the lens
oracle's own rays and trial counts, so that a case that stops reaching its edge fails without a GPU. The renders themselves
are compared on the GPU (tests/test_gpu_lens_edges.py)."""
import pytest

import lens_edges as LE

CASES = LE.cases()


@pytest.mark.parametrize("name", list(CASES))
def test_case_reaches_its_edge(name):
    sc, lens = CASES[name]
    LE.reach(name, sc, lens)


def test_the_deep_disk_seed_is_the_first_the_search_finds():
    assert LE.deep_seed_search(tries=64) == LE.DEEP_SEED


def test_the_64_bit_seed_changes_the_lens_render():
    """The oracle's lens render under SEED64 differs from its render under the low word alone."""
    import oracle_lens as OL
    sc, lens = CASES["u_1e3"]
    full = OL.render(sc, lens)["linear"]
    sc.seed = LE.SEED64 & 0xFFFFFFFF
    try:
        assert (LE.SEED64 >> 32) not in (0, LE.SEED64 & 0xFFFFFFFF)
        assert not (full.view("u4") == OL.render(sc, lens)["linear"].view("u4")).all()
    finally:
        sc.seed = LE.SEED64
