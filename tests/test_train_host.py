"""Host side of the training loop (cchess_zero_b200/train.py), no GPU: the mirror label table, the replay ring's deque order and
sampling, the policy_update arithmetic shared with cchess_main, and the record validation of ReplayBuffer.add."""
import random
from collections import deque

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)


def test_mirror_label_table_is_the_file_mirror_of_every_label():
    from cchess_zero_b200 import rules
    from cchess_zero_b200.train import mirror_labels
    m = mirror_labels()
    labels = rules.create_uci_labels()
    assert m.shape == (2086,) and m.dtype == np.int16
    assert np.array_equal(m[m], np.arange(2086))                         # an involution
    l2i = {v: i for i, v in enumerate(labels)}
    files = str.maketrans("abcdefghi", "ihgfedcba")
    assert [int(v) for v in m] == [l2i[s.translate(files)] for s in labels]
    assert int((m == np.arange(2086)).sum()) == 90                        # the moves along the centre file e map to themselves


@pytest.mark.parametrize("capacity", [1, 7, 64, 500])
def test_ring_order_is_deque_order(capacity):
    from cchess_zero_b200.train import RingIndex
    rs = np.random.RandomState(capacity)
    ring, dq = RingIndex(capacity), deque(maxlen=capacity)
    slot_id = np.full(capacity, -1, dtype=np.int64)
    next_id = 0
    for _ in range(60):
        k = int(rs.choice([0, 1, 3, capacity - 1, capacity, capacity + 5, rs.randint(0, 2 * capacity + 2)]))
        ids = np.arange(next_id, next_id + k)
        next_id += k
        first, slots = ring.add(k)
        slot_id[slots] = ids[first:]
        dq.extend(ids.tolist())
        assert len(ring) == len(dq)
        assert slot_id[ring.slots(np.arange(len(ring)))].tolist() == list(dq)
        if len(dq) > 1:
            k2 = int(rs.randint(1, len(dq)))
            seed = int(rs.randint(1 << 30))
            assert slot_id[ring.sample_rows(random.Random(seed), k2)].tolist() == random.Random(seed).sample(dq, k2)


def test_ring_rejects_empty_capacity():
    from cchess_zero_b200.train import RingIndex
    with pytest.raises(ValueError):
        RingIndex(0)


def _kl_reference(old_probs, new_probs):
    """The expression cchess_main.policy_update used before the helper existed."""
    with np.errstate(all="ignore"):
        kl_tmp = old_probs * (np.log((old_probs + 1e-10) / (new_probs + 1e-10)))
    return np.mean([np.sum(line[~(np.isnan(line) | np.isposinf(line))]) for line in kl_tmp])


def test_policy_kl_matches_the_policy_update_expression_and_keeps_minus_inf():
    from cchess_zero_b200.train import policy_kl
    rs = np.random.RandomState(0)
    for _ in range(20):
        old = (rs.randn(16, 2086) * 3).astype(np.float32)                 # logits: negative values are routine
        new = (old + rs.randn(16, 2086).astype(np.float32) * 0.1).astype(np.float32)
        a, b = policy_kl(old, new), _kl_reference(old, new)
        assert a.dtype == b.dtype and (a == b or (np.isnan(a) and np.isnan(b)))
    old = np.array([[1.0, 2.0, -1e-10, 0.5], [1.0, 1.0, 1.0, 1.0]], dtype=np.float32)
    new = np.array([[1.0, -1e-10, 0.5, -2.0], [1.0, 1.0, 1.0, 1.0]], dtype=np.float32)
    with np.errstate(all="ignore"):
        terms = old * np.log((old + 1e-10) / (new + 1e-10))
    assert np.isposinf(terms).any() and np.isnan(terms).any()            # both dropped ...
    assert np.isfinite(policy_kl(old, new))
    old2 = np.array([[-3e38, 0.0], [1.0, 1.0]], dtype=np.float32)       # a huge negative logit: the term overflows to -inf
    new2 = np.array([[-1e-5, 0.0], [1.0, 1.0]], dtype=np.float32)
    with np.errstate(all="ignore"):
        assert np.isneginf(old2 * np.log((old2 + 1e-10) / (new2 + 1e-10)))[0, 0]
    assert np.isneginf(policy_kl(old2, new2)) and np.isneginf(_kl_reference(old2, new2))   # ... and -inf is kept


@pytest.mark.parametrize("kl,mult,want", [
    (0.2, 1.0, 1.0 / 1.5),      # kl > 2 kl_targ: slow down
    (0.2, 0.1, 0.1),            # ... not below 0.1
    (0.001, 1.0, 1.5),          # kl < kl_targ / 2: speed up
    (0.001, 10.0, 10.0),        # ... not above 10
    (0.025, 2.0, 2.0),          # in between: unchanged
    (float("-inf"), 3.0, 4.5),  # a -inf KL counts as small
])
def test_next_lr_multiplier_covers_the_three_branches(kl, mult, want):
    from cchess_zero_b200.train import next_lr_multiplier
    kl_targ = 0.025
    ref = mult
    if kl > kl_targ * 2 and ref > 0.1:
        ref /= 1.5
    elif kl < kl_targ / 2 and ref < 10:
        ref *= 1.5
    assert next_lr_multiplier(kl, kl_targ, mult) == ref == pytest.approx(want)


def test_explained_variance_is_the_reference_expression():
    from cchess_zero_b200.train import explained_variance
    rs = np.random.RandomState(1)
    wb = np.expand_dims(rs.choice([-1.0, 0.0, 1.0], 32), 1)
    v = rs.uniform(-1, 1, (32, 1)).astype(np.float32)
    assert explained_variance(wb, v) == 1 - np.var(wb - v.flatten()) / np.var(wb)


def _records():
    """pack_records output for two small games built from state strings (what ReplayBuffer.add receives)."""
    from cchess_zero_b200 import rules
    from cchess_zero_b200.distributed import TupleBatch, pack_records
    from cchess_zero_b200.selfplay import GameRecord
    s0 = rules.START_STATE
    s1 = "RNBAKABNR/9/1C5C1/P1P1P1P1P/9/9/p1p1p1p1p/1c5c1/9/rnbakab1r"
    recs = [GameRecord.from_tuples([s0, s1], [np.array([3, 40, 7]), np.array([5])], [np.array([0.5, 0.25, 0.25]), np.array([1.0])],
                                   np.array([1.0, -1.0])),
            GameRecord.from_tuples([s1], [np.array([100, 2085])], [np.array([0.75, 0.25])], np.array([0.0]))]
    buf, n, _ = pack_records(recs)
    assert n == 3
    return TupleBatch(buf)


def test_validate_tuples_accepts_pack_records_output():
    from cchess_zero_b200.train import validate_tuples
    validate_tuples(_records())


@pytest.mark.parametrize("bad", ["piece", "n", "idx_low", "idx_high", "duplicate", "prob_nan", "prob_inf", "prob_f32_overflow", "z", "shape"])
def test_validate_tuples_rejects_malformed_records(bad):
    from cchess_zero_b200.train import validate_tuples
    tb = _records()
    if bad == "piece":
        tb.boards[1, 17] = 15
    elif bad == "n":
        tb.n[0] = 129
    elif bad == "idx_low":
        tb.idx[0, 1] = -1
    elif bad == "idx_high":
        tb.idx[2, 1] = 2086
    elif bad == "duplicate":
        tb.idx[0, 2] = tb.idx[0, 0]
    elif bad == "prob_nan":
        tb.prob[0, 0] = np.nan
    elif bad == "prob_inf":
        tb.prob[1, 0] = np.inf
    elif bad == "prob_f32_overflow":
        tb.prob[1, 0] = 1e300
    elif bad == "z":
        tb.z[2] = 0.5
    elif bad == "shape":
        tb.idx = tb.idx[:, :64]
    with pytest.raises(ValueError):
        validate_tuples(tb)


def test_validate_tuples_ignores_entries_beyond_n():
    from cchess_zero_b200.train import validate_tuples
    tb = _records()
    tb.idx[1, 5] = -7                       # padding beyond n is never read
    tb.prob[1, 5] = np.nan
    validate_tuples(tb)
