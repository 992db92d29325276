"""CPU half of test_gpu_kernel_paths.py: every case of the GPU file lands on the kernel and
branch it names (the host build runs the same selection code as the CUDA library), with the
task-row count K and free-column count nf of the tree size classes, and the host build of that
path agrees with the fp64 oracle.  Runs without a GPU, so a case that drifts off its branch is
caught before any device time is spent."""

import pytest

from tests import test_gpu_kernel_paths as g


@pytest.mark.parametrize("name", g.GENERAL)
def test_general_path_cases(name):
    g.host_side(g.general_case(name))


@pytest.mark.parametrize("nj", [n for n, _, _ in g.TREE_EXTRAS])
def test_tree_extras_boundary_cases(nj):
    g.host_side(g.tree_extras_case(nj))


@pytest.mark.parametrize("limits", [False, True], ids=["no-limits", "limits"])
@pytest.mark.parametrize("name", list(g.SIZE_CLASSES))
def test_tree_size_class_cases(name, limits):
    g.host_side(g.size_class_case(name, limits))


@pytest.mark.parametrize("lanes", [1, 2, 4, 8])
@pytest.mark.parametrize("name", list(g.CHAINS))
def test_sub_warp_chain_cases(name, lanes):
    g.chain_host_side(name, lanes)


def test_sub_warp_variants_cover_their_shapes():
    """L = 4 / 8 run the sub-warp kernel on <6, 1> only: the UR5 cases; the other chains check
    the fall-back to the default kernel."""
    takes = {name: g.coop_takes(4, g.CHAINS[name]()) for name in g.CHAINS}
    assert takes["ur5-reachable"] and not takes["nj6-two-frames"] and not takes["nj4-posture-only"]


@pytest.mark.parametrize("name", list(g.RECOMPUTE))
def test_recompute_cases_land_on_the_pdl_chain_kernel(name):
    g.recompute_dispatch(name)
