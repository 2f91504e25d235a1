"""Fused correlation + mutual-NN kernel vs the oracle / the reference's golden pairs."""
import numpy as np
import pytest
import torch

import fma_ref as FR
from conftest import golden
from oracle import outil_oracle as OO

pytestmark = pytest.mark.gpu


def gpu_match(rf, A, B, precision=0):
    i1, i2 = None, None
    rf.outil.corr_precision = precision
    try:
        i1, i2 = rf.outil.mutualMatching(torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda())
    finally:
        rf.outil.corr_precision = 0
    return i1.cpu().numpy(), i2.cpu().numpy()


def ambiguous(score, tol=2e-6):
    """Rows / columns whose top-2 gap is below fp32 accumulation noise (arg-max legitimately order dependent)."""
    s = np.sort(score, axis=1)
    rows = (s[:, -1] - s[:, -2]) < tol if score.shape[1] > 1 else np.zeros(score.shape[0], bool)
    s = np.sort(score, axis=0)
    cols = (s[-1] - s[-2]) < tol if score.shape[0] > 1 else np.zeros(score.shape[1], bool)
    return rows, cols


def check_exact(i1, i2, A, B):
    """Precision 0 is exact: the pairs are those of the fp32 FMA-chain restatement (tests/fma_ref.py), bit for bit.  A, B:
    (C, N) features as given to mutualMatching."""
    _, _, r1, r2 = FR.corr_keys(torch.from_numpy(np.ascontiguousarray(A.T)).cuda(), torch.from_numpy(np.ascontiguousarray(B.T)).cuda())
    assert np.array_equal(i1, r1) and np.array_equal(i2, r2), (len(i1), len(r1))


def check_same(i1, i2, o1, o2, score):
    if np.array_equal(i1, o1) and np.array_equal(i2, o2):
        return 0
    rows, cols = ambiguous(score)
    got, exp = set(zip(i1.tolist(), i2.tolist())), set(zip(o1.tolist(), o2.tolist()))
    bad = [(a, b) for (a, b) in got ^ exp if not (rows[a] or cols[b])]
    assert not bad, "unambiguous pairs differ: %s" % bad[:5]
    return len(got ^ exp)


def test_golden_pairs(rf):
    g = golden("mutual_matching")
    i1, i2 = gpu_match(rf, g["featA"], g["featB"])
    assert np.array_equal(i1, g["index1"]) and np.array_equal(i2, g["index2"])
    assert i1.dtype == np.int64 and np.all(np.diff(i1) > 0)


@pytest.mark.parametrize("C,NA,NB,seed", [(1024, 13065, 1200, 0), (1024, 2107, 300, 1), (64, 129, 127, 2), (16, 5, 3, 3),
                                           (256, 1, 1, 4), (1024, 300, 1200, 5), (36, 500, 260, 6)])
def test_random_features(rf, C, NA, NB, seed):
    rs = np.random.RandomState(seed)
    A = np.abs(rs.randn(C, NA)).astype(np.float32)
    B = np.abs(rs.randn(C, NB)).astype(np.float32)
    n = min(NA, NB) // 2
    B[:, :n] = A[:, rs.permutation(NA)[:n]] + 0.1 * np.abs(rs.randn(C, n)).astype(np.float32)
    A /= np.linalg.norm(A, axis=0, keepdims=True)
    B /= np.linalg.norm(B, axis=0, keepdims=True)
    if NB > 2:
        B[:, 1] = 0                              # masked target cell: never matches
    o1, o2, score = OO.mutualMatching(A, B, return_score=True)
    i1, i2 = gpu_match(rf, A, B)
    check_same(i1, i2, o1, o2, score)
    check_exact(i1, i2, A, B)
    if NB > 2:
        assert 1 not in i2
    assert len(i1) >= n // 2


def test_negative_scores_and_ties(rf):
    # signed features: (S*S > 0) keeps negative maxima too (utils/outil.py:41-42)
    rs = np.random.RandomState(9)
    A = rs.randn(32, 40).astype(np.float32)
    B = -A[:, :10].copy()
    B[:, 0] = A[:, 0]
    o1, o2, score = OO.mutualMatching(A, B, return_score=True)
    i1, i2 = gpu_match(rf, A, B)
    check_same(i1, i2, o1, o2, score)
    check_exact(i1, i2, A, B)
    # exact ties: first index wins on both sides (documented tie-break)
    A2 = np.zeros((4, 6), np.float32)
    A2[0] = 1
    B2 = np.zeros((4, 3), np.float32)
    B2[0] = 1
    i1, i2 = gpu_match(rf, A2, B2)
    assert i1.tolist() == [0] and i2.tolist() == [0]
