"""The mbarrier protocol of the tensor-core point kernel, checked on a discrete-event model (tools/tc_protocol_sim.py):
no deadlock, no parity wait that skipped or overran a phase, every MMA reads the ring contents it expects, no accumulator
overwritten while it is being drained -- under randomised operation latencies.  Broken variants must be caught."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import tc_protocol_sim as sim  # noqa: E402


@pytest.mark.parametrize("tiles", [1, 2, 5])
def test_kernel_protocol_is_sound_under_random_schedules(tiles):
    for seed in range(40):
        sim.simulate(tiles, seed)


def test_unskewed_epilogue_order_is_also_legal():
    for seed in range(10):
        sim.simulate(3, seed, "x3_after_final")


@pytest.mark.parametrize("mutation", ["no_xempty_wait", "no_wempty_wait", "no_acc_wait"])
def test_broken_protocols_are_detected(mutation):
    caught = 0
    for seed in range(10):
        try:
            sim.simulate(3, seed, mutation)
        except AssertionError:
            caught += 1
    assert caught == 10, (mutation, caught)


def test_dual_issuer_variant_is_sound():
    """The dual-issuer protocol variant (one MMA warp per N-block, producers owning fixed slots,
    every waiter observing every phase) -- the variant the round-2 plan builds on -- with 3 and 4 weight slots."""
    for prm in ({"issuers": 2, "NW": 3}, {"issuers": 2, "NW": 4, "split_wfull": 1}):
        for seed in range(15):
            sim.simulate(3, seed, params=prm)


def test_protocols_survive_heavy_jitter():
    """shipped protocol, the dual-issuer experiment (3 slots), and the round-2 candidate: two issuers with one "stage landed"
    barrier per (issuer, slot) and 4 weight slots"""
    for prm in ({}, {"issuers": 2}, {"issuers": 2, "NW": 4, "split_wfull": 1}, {"issuers": 2, "NW": 3, "split_wfull": 1}):
        for seed in range(12):
            sim.simulate(6, seed, params=dict(prm, jitter=0.9))


def test_observe_all_dual_issuer_with_four_slots_is_unsound():
    """Found by the model, not on the GPU: with 4 slots an issuer that merely *observes* the other's stages can fall two
    phases behind a slot's barrier -> the per-issuer barriers above are required."""
    bad = 0
    for seed in range(40):
        try:
            sim.simulate(8, seed, params={"issuers": 2, "NW": 4, "jitter": 0.9})
        except AssertionError:
            bad += 1
    assert bad >= 1


def test_issuer_that_skips_phases_aliases():
    """The bug of the first dual-issuer attempt: an issuer that waits only for its own stages sees a stale parity once the
    two issuers drift apart (needs strongly varying latencies to show up -- as it needed 1792 tiles x 74 pairs on the GPU)."""
    caught = 0
    for seed in range(20):
        try:
            sim.simulate(10, seed, "dual_skip_phases", {"issuers": 2, "jitter": 0.9})
        except AssertionError as e:
            assert "meant phase" in str(e) or "holds stage" in str(e) or "no progress" in str(e) or "deadlock" in str(e)
            caught += 1
    assert caught >= 5, caught


ROUND2 = {"x2_in_ring": 1, "NW": 4, "issuers": 2, "split_wfull": 1}


@pytest.mark.parametrize("tiles", [1, 2, 7])
def test_round2_candidate_protocol_is_sound(tiles):
    """fold1/conv1 output through the activation ring (frees its 16 KB slot), 4 weight slots, two issuers with per-issuer
    'stage landed' barriers -- the protocol DESIGN.md proposes for the next kernel revision."""
    for seed in range(15):
        sim.simulate(tiles, seed, params=ROUND2)
        sim.simulate(tiles, seed, params=dict(ROUND2, jitter=0.9))


def test_round2_candidate_is_faster_in_the_model():
    base = sum(sim.simulate(6, s) for s in range(5))
    cand = sum(sim.simulate(6, s, params=ROUND2) for s in range(5))
    assert cand < 0.93 * base, (cand, base)


def test_v2_static_maps_agree_with_the_issue_order():
    """point_tc.cu's stage_info() (stage -> image position, consuming issuer) and ring_seq() (activation slice -> ring
    position), restated here, against the MMA issue order and tc_pack_weights' kCyclePos -- incl. the last tile, which has no
    'next stream' entry."""
    FIRST_L0_POS, SPS = 57, 33
    kCyclePos = [[FIRST_L0_POS, 0, 8, 25], [24, 33, 41, 58]]
    SL, NNB = {0: 1, 1: 4, 2: 8, 3: 8}, {0: 1, 1: 2, 2: 2, 3: 1}

    def stage_info(g, tiles):
        if g == 0:
            return FIRST_L0_POS, 0
        cidx, last0 = g - 1, (tiles - 1) * 2 * SPS
        r = cidx % (2 * SPS)
        if cidx >= last0 and cidx - last0 >= FIRST_L0_POS:
            r = cidx - last0 + 1
        issuer = (r & 1) if r < 24 else (((r - 33) & 1) if 33 <= r < 57 else 0)
        return r, issuer

    for tiles in (1, 2, 3, 6):
        S = 2 * tiles

        def ring_seq(sn, kind, t):
            if kind == 2:
                return 0 if sn == 0 else 1 + 21 * (sn - 1) + 12
            base = 1 + 21 * sn
            return base + 12 + (1 if sn + 1 < S else 0) + t if kind == 5 else base + (0 if kind == 3 else 4) + t

        g = x = 0
        for grp in range(-1, S):
            for q in range(4):
                layer = (1, 2, 0, 3)[q]
                sn = grp + 1 if q == 2 else grp
                if sn < 0 or sn >= S:
                    continue
                for t in range(SL[layer]):
                    assert ring_seq(sn, 2 + layer, t) == x
                    x += 1
                    for nb in range(NNB[layer]):
                        img, issuer = stage_info(g, tiles)
                        assert img == kCyclePos[sn & 1][layer] + t * NNB[layer] + nb
                        assert issuer == (nb if NNB[layer] == 2 else 0)
                        g += 1
        assert g == 66 * tiles
