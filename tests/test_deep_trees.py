"""The request-tree join and the critical-path walk on deep, irregular trees (tests/deep_tree_util.py),
without a GPU.

The CPU build of the device steps (tests/emul/tw_emul_critical.cpp) runs levels 0 .. L - 1 as the kernels
do, the last of them walking everything below it through the kernels' own cp_tail_walk.  At every level
count L in 1 .. 64 its arrays must be the host reference's (traces.critical_paths_host), on spine-first and
spine-last trees, with int64 times and with float64 times divided by 3 and 7: a spine-last tree of 20
levels keeps up to 140 in-spans pending below level 1, more than a 64-entry stack holds.  The self times of
every request add up to its latency on trees of every call timing and service order; on sequential trees
every node is on the path and its self time has a closed form.  The host join (traces.assemble_host)
follows chains of thousands of levels and a deep tree under a long cycle."""
import numpy as np
import pytest

from deep_tree_util import ORDERS, TIMINGS, deep_trees
import emul_backend
from test_critical_path import check_invariant, check_same, compressed

LEVELS = range(1, 65)


def _sweep(g, levels=LEVELS):
    """Host reference with the invariant; the CPU step equal to it at every level count, int64 and
    float64 / 3, / 7."""
    from traceweaver_b200.traces import critical_paths_host
    hb, assign, in_caller = g["hb"], g["assign"], g["in_caller"]
    res = []
    for cf in (None, 3, 7):
        h = hb if cf is None else compressed(hb, cf)
        want = critical_paths_host(h, assign, in_caller, 0.0)
        check_invariant(want, h, exact=cf is None)
        for L in (0, *levels):
            got = emul_backend.critical_paths(h, assign, in_caller, want["root"], 0.0, levels=L)
            check_same(got, want, exact_sums=cf is None)
        res.append(want)
    return res[0]


@pytest.mark.parametrize("spine", ["first", "last"])
def test_tail_walk_gives_the_same_paths_at_every_level_count(spine):
    g = deep_trees(20, callees=8, spine=spine, requests=3, seed=5)
    res = _sweep(g)
    assert (res["on_path"] == 1).all()


@pytest.mark.parametrize("spine", ["first", "last"])
def test_tail_walk_on_every_call_timing(spine):
    for q, timing in enumerate(TIMINGS + ("mixed",)):
        _sweep(deep_trees(12, callees=5, spine=spine, timing=timing, requests=2, order=ORDERS[q % 3],
                          seed=10 + q))


@pytest.mark.parametrize("order", ORDERS)
def test_tail_walk_on_random_shapes(order):
    g = deep_trees(16, callees=8, random_shape=True, requests=12, timing="mixed", order=order, seed=21)
    assert (g["depth"] > 1).any() and (g["assign"] == -1).any()
    _sweep(g)


def test_tail_walk_below_level_1_of_a_deep_tree():
    # 600 levels of spine-last calls: the first level's threads walk all of it
    g = deep_trees(600, callees=3, spine="last", requests=2, seed=7)
    res = _sweep(g, levels=(1, 2, 33, 64))
    assert (res["on_path"] == 1).all()


@pytest.mark.parametrize("timing", TIMINGS + ("mixed",))
@pytest.mark.parametrize("order", ORDERS)
def test_self_times_add_up_on_generated_trees(timing, order):
    from traceweaver_b200.traces import critical_paths_host
    seed = 3 * (TIMINGS + ("mixed",)).index(timing) + ORDERS.index(order)
    g = deep_trees(40, callees=4, timing=timing, requests=5, random_shape=True, order=order, seed=seed)
    res = critical_paths_host(g["hb"], g["assign"], g["in_caller"], 0.0)
    check_invariant(res, g["hb"], exact=True)
    assert res["requests"][0] == len(g["roots"])


@pytest.mark.parametrize("callees", [1, 2, 8])
def test_sequential_spine_first_trees_have_the_closed_form(callees):
    from traceweaver_b200.traces import parents_host
    g = deep_trees(30, callees=callees, spine="first", timing="sequential", requests=3, order="shuffled",
                   seed=callees)
    hb = g["hb"]
    res = _sweep(g, levels=(1, 3, 64))
    assert (res["on_path"] == 1).all()
    # the calls are sequential and inside their caller, every server span inside its client span: a node's
    # self time is its length less its children's
    start = np.concatenate([hb.in_start, hb.out_start]).astype(np.int64)
    end = np.concatenate([hb.in_end, hb.out_end]).astype(np.int64)
    parent = parents_host(hb, g["assign"], g["in_caller"])
    child_len = np.zeros(len(start), np.int64)
    has = parent >= 0
    np.add.at(child_len, parent[has], (end - start)[has])
    assert np.array_equal(res["self_us"], (end - start - child_len).astype(np.float64))
    assert sorted(np.flatnonzero(res["culprit"] >= 0).tolist()) == sorted(g["roots"].tolist())


def test_equal_self_times_pick_the_smallest_node():
    g = deep_trees(50, callees=4, spine="last", requests=3, order="shuffled", const_times=True, seed=3)
    res = _sweep(g, levels=(1, 7, 64))
    on, self_us, root = res["on_path"] == 1, res["self_us"], res["root"]
    for r in g["roots"]:
        mine = np.flatnonzero(on & (root == r))
        top = mine[self_us[mine] == self_us[mine].max()]
        assert len(top) > 50                                 # every leaf in-span ties
        assert res["culprit"][r] == top.min()


@pytest.mark.parametrize("order", ORDERS)
def test_host_join_follows_deep_chains(order):
    from traceweaver_b200.traces import assemble_host
    g = deep_trees(2500, callees=1, requests=2, order=order, seed=4)
    parent, root, size = assemble_host(g["hb"], g["assign"], g["in_caller"])
    r0, r1 = g["roots"]
    assert (root >= 0).all() and size[r0] == size[r1] == 2 * 2500
    assert set(np.unique(root).tolist()) == {int(r0), int(r1)}


def test_host_join_puts_a_tree_under_a_cycle_in_no_request():
    from traceweaver_b200.traces import assemble_host
    g = cycle_trees(300)
    _, root, _ = assemble_host(g["hb"], g["assign"], g["in_caller"])
    assert (root[g["lost"]] == -1).all()
    assert (np.delete(root, g["lost"]) >= 0).all()


def cycle_trees(depth, seed=6):
    """Three spine-last requests of `depth` levels: request 0 closed into a cycle (its root's caller is its
    deepest spine call) and request 1 hanging under it (its root's caller is one of request 0's calls whose
    server span is not in the batch); request 2 is left whole.  lost: the nodes of requests 0 and 1."""
    from traceweaver_b200.traces import assemble_host
    g = deep_trees(depth, callees=4, spine="last", leaf_in_batch=False, requests=3, order="shuffled", seed=seed)
    _, root, _ = assemble_host(g["hb"], g["assign"], g["in_caller"])
    r0, r1, _ = g["roots"]
    lost = np.flatnonzero((root == r0) | (root == r1))
    in_caller = g["in_caller"].copy()
    in_caller[r0] = g["open_calls"][0][0]
    in_caller[r1] = g["open_calls"][0][len(g["open_calls"][0]) // 2]
    return dict(g, in_caller=in_caller, lost=lost)
