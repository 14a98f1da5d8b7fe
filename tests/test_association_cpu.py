"""The obstacle association at its edges on the CPU (tests/assoc_cases.py): on every crafted case the oracle's orc_associate
equals the numpy restatement of the reference's rule with the K row slots, and the emulator's short-list association
(associate_stage, the device code of lists of at most 64 obstacles) equals the oracle.  This pins the rule that the GPU tests
hold the long-list association (dev_associate_list) to.  The resident-slot model of the long-list association is checked on
its own: without overflow it is a one-to-one relabelling of the selection."""
import numpy as np
import pytest

import assoc_cases as ac

GROUPS = ac.groups()
CASES = [(g, c) for g in GROUPS for c in g.cases]
IDS = [f"{g.name}-{c.name}" for g, c in CASES]


@pytest.mark.parametrize("gc", CASES, ids=IDS)
def test_oracle_equals_numpy_restatement(orc, gc):
    g, case = gc
    got = ac.oracle_selection(orc, g.cfg, case)
    want = ac.restated_selection(g.cfg, case.X, case.types, case.params, case.dt)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("gc", [gc for gc in CASES if gc[1].count <= ac.M_RES], ids=[i for i, gc in zip(IDS, CASES) if gc[1].count <= ac.M_RES])
def test_emulator_short_list_equals_oracle(orc, emu, gc):
    g, case = gc
    if g.cfg.k_max_obstacles_per_stage == 0:
        pytest.skip("K = 0: no row slots")
    np.testing.assert_array_equal(ac.emulator_selection(emu, g.cfg, case), ac.oracle_selection(orc, g.cfg, case))


def test_crafted_edges_are_reached(orc):
    """the hand-placed stages select what they were built for (read off the oracle: the GPU test compares with it)"""
    g = GROUPS[0]
    case = g.cases[0]
    sel = ac.oracle_selection(orc, g.cfg, case)
    row = lambda k: [int(v) for v in sel[:, k] if v >= 0]   # noqa: E731
    assert row(1) == [10, 12]                    # first of the duplicates, and the right one at the same distance
    assert row(2) == [31, 63]                    # across the chunk boundary
    assert row(3) == [5, 96]                     # one lane, two chunks
    assert row(4) == [0, 100]                    # the first entry beats the last
    assert row(5) == [200, 400]                  # mirrored pairs: the earlier index
    assert row(6) == [500, 700, 900, 541, 600]   # replacement of the FIRST farthest slot
    assert row(7) == [1103, 1100, 1101]          # forced just inside; == force_inclusion_dist and == cutoff_dist kept
    assert row(8) == [1201, 1200]                # the heading line is the right side
    for name, want in (("forced_K1", 1), ("forced_K5", 5), ("forced_K16", 16)):
        grp = next(x for x in GROUPS if x.cases[0].name == name)
        s = ac.oracle_selection(orc, grp.cfg, grp.cases[0])
        assert ((s[:, 1:-1] >= 0).sum(axis=0) == want).all(), name


def test_overflow_and_tie_cases_reach_their_edges(orc):
    """the overflow cases really fill the 64 resident slots and the others never do; the cases built on duplicates select an
    obstacle that has an exact twin in distance at some stage"""
    for g in GROUPS:
        for case in g.cases:
            sel = ac.oracle_selection(orc, g.cfg, case)
            _, gidx, dropped = ac.resident_model(sel)
            if "overflow" in case.tags:
                assert dropped > 0 and (gidx >= 0).all(), (g.name, case.name)
            else:
                assert dropped == 0, (g.name, case.name)
            if g.cfg.k_max_obstacles_per_stage and ({"tie_in_chunk", "footprint", "dynamic", "overflow"} & set(case.tags)):
                assert ac.has_exact_tie(g.cfg, case, sel), (g.name, case.name)


def test_resident_model_without_overflow_is_a_relabelling(orc):
    for g in GROUPS:
        for case in g.cases:
            sel = ac.oracle_selection(orc, g.cfg, case)
            slots, gidx, dropped = ac.resident_model(sel)
            if dropped:
                continue
            used = gidx[gidx >= 0]
            assert len(np.unique(used)) == len(used) == len(np.unique(sel[sel >= 0]))
            assert (gidx[len(used):] == -1).all()
            np.testing.assert_array_equal(np.where(slots >= 0, gidx[np.clip(slots, 0, None)], -1), sel)
            # first use order: the slots appear in increasing order along stages 1..N-2, slot order within a stage
            first = []
            for k in range(1, sel.shape[1] - 1):
                for s in slots[:, k]:
                    if s >= 0 and s not in first:
                        first.append(int(s))
            assert first == list(range(len(used)))


def test_resident_model_on_a_synthetic_overflow():
    """87 distinct selections over 2 slots per stage: 64 resident in first-use order, the rest dropped, repeats of resident
    ones kept"""
    N = 60
    sel = -np.ones((2, N), dtype=np.int64)
    nxt = 0
    for k in range(1, N - 1):
        sel[0, k] = nxt; nxt += 1
        sel[1, k] = nxt if k % 2 else 0   # every other stage a new one, else index 0 again
        nxt += k % 2
    slots, gidx, dropped = ac.resident_model(sel)
    # list indices appear in increasing order: the first 64 are resident, every later one is dropped
    assert len(np.unique(sel[sel >= 0])) > 64 and dropped == (sel >= 64).sum()
    assert (gidx == np.arange(64)).all()
    assert (slots[sel >= 64] == -1).all() and (slots[sel == 0] == 0).all()
