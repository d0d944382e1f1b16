"""The task graph of the selected inversion (csrc/covariance.cuh: sparse_selinv_kernel), restated in numpy from the
supernodal layout of tests/test_sparse_schur_plan.py and checked against b200_plan_sparse_selinv, for every test structure
under AMD and NESDIS.  No GPU needed.  This is the no-deadlock argument of the kernel: every block of Z_RR a supernode's task
reads lies in the panel of a supernode its counter waits on, each of those has a smaller ticket, and the counter the library
starts the task with is their number (0 for a root, which starts at once: there are no forward tasks in this launch)."""
import numpy as np
import pytest

from tests.test_sparse_schur_plan import STRUCTURES, Layout, camera_edges, eliminate, structure


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.mark.parametrize("ordering", ["amd", "nesdis"])
@pytest.mark.parametrize("name", STRUCTURES)
def test_selinv_task_graph(cs, name, ordering):
    ot = cs.NESDIS if ordering == "nesdis" else cs.AMD
    C, P, cam, pt = structure(name)
    perm, st = cs.plan_sparse_schur(C, P, cam, pt, ordering_type=ot)
    _, _, _, parent, below = eliminate(C, camera_edges(C, cam, pt), perm, structure=True)
    lay = Layout(parent, below)
    first, order, counter = cs.plan_sparse_selinv(C, P, cam, pt, ordering_type=ot)
    assert np.array_equal(first, lay.first) and st["supernodes"] == lay.ns
    ns = lay.ns
    assert sorted(order.tolist()) == list(range(ns))
    sn_of = np.repeat(np.arange(ns), lay.width)
    ticket = np.empty(ns, dtype=int)
    ticket[order[::-1]] = np.arange(ns)   # the selected inversion takes the factor's order in reverse
    rows = [set(r.tolist()) for r in lay.rows]
    for s in range(ns):
        below_s = lay.rows[s][lay.width[s]:]
        waits = set(sn_of[below_s].tolist())
        assert counter[s] == len(waits), (s, counter[s], waits)
        assert all(ticket[t] < ticket[s] for t in waits), s
        for i, a in enumerate(below_s):
            for b in below_s[:i + 1]:   # Z_RR entry (a, b), a >= b: in the panel of the supernode owning b, row a
                t = sn_of[b]
                assert t in waits and a in rows[t], (s, a, b)
    assert counter[[s for s in range(ns) if lay.R[s] == lay.width[s]]].sum() == 0
