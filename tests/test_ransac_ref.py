"""The RANSAC restatement and certification of tests/ransac_ref.py against the oracle, and proof that the exact comparison of
tests/test_gpu_ransac_exact.py rejects subtly wrong kernels (CPU only)."""
import numpy as np
import pytest

import ransac_ref as R
from conftest import golden
from oracle import outil_oracle as OO
from oracle import synth

GOLDEN = ["ransac_m120", "ransac_m636", "ransac_grid", "ransac_remainder_only", "ransac_none", "ransac_lowinlier"]


def oracle_outcome(m1, m2, samples, tol):
    """(status, H, nbInlier, mask) of outil_oracle.RANSAC_from_samples in the kernel's status codes."""
    try:
        H, nb, inl, _ = OO.RANSAC_from_samples(m1, m2, samples, tol)
    except TypeError:
        return R.NO_MODEL, None, 0, None
    if H is None:
        return R.NONE, None, 0, None
    return R.OK, H, int(nb), inl


def fuzz_cases(n=30, seed=77):
    rs = np.random.RandomState(seed)
    for case in range(n):
        M = int(rs.choice([4, 5, 9, 40, 150, 636]))
        nbIter = int(rs.choice([1, 50, 99, 100, 101, 250, 700]))
        frac = float(rs.choice([0.0, 0.3, 0.6, 1.0]))
        tol = float(rs.choice([0.005, 0.05, 0.1]))
        m1, m2, _ = synth.make_matches(900 + case, M, frac, grid=(30, 40) if case % 2 else None)
        yield "fuzz%d" % case, m1, m2, synth.draw_samples(900 + case, M, nbIter), tol


def all_cases():
    for name in GOLDEN:
        g = golden(name)
        yield name, g["match1"], g["match2"], g["samples"], float(g["tol"])
    for name, build in R.BUILDERS.items():
        yield (name,) + build(R.lapack_provider)
    yield from fuzz_cases()


def test_given_lapack_H_is_the_oracle():
    """ransac_given_H with LAPACK's H: the oracle's status, H, nbInlier and mask on every golden case, every built case and
    a seeded fuzz; its per-hypothesis counts are the oracle's ScoreRANSAC."""
    seen = set()
    for name, m1, m2, s, tol in all_cases():
        r = R.ransac_given_H(m1, m2, s, tol, R.lapack_H(m1, m2, s))
        st, H, nb, inl = oracle_outcome(m1, m2, s, tol)
        seen.add(st)
        assert r["status"] == st, name
        if st == R.OK:
            assert np.array_equal(r["H"], H) and r["nbInlier"] == nb and np.array_equal(r["mask"], inl), name
        us = np.asarray(s)[r["rows"]]
        if len(us):
            assert np.array_equal(r["counts"], OO.ScoreRANSAC(m1, m2, tol, us)[1]), name
    assert seen == {R.OK, R.NONE, R.NO_MODEL}


def test_certified_bounds_hold_for_lapack_and_householder():
    """Every hypothesis' gated count under LAPACK's H and under the Householder recurrence (OO.householder_null_vector, the
    kernel's algorithm in fp64) lies in certify's [lo, hi]; the two DLTs' counts differ only where lo < hi."""
    tot = dict(hyp=0, uncertified=0, ambiguous=0, differ=0)
    for name, m1, m2, s, tol in all_cases():
        rows = R.unique_rows(s)
        if len(rows) == 0 or len(rows) > 1200:
            continue
        us = np.asarray(s)[rows]
        c = R.certify(m1, m2, s, tol)
        hl = R.ransac_given_H(m1, m2, s, tol, R.lapack_H(m1, m2, s))["counts"]
        Hh = np.array([OO.householder_null_vector(a) for a in OO.dlt_matrix(m1[us], m2[us])]).astype(np.float32)
        hh = R.ransac_given_H(m1, m2, s, tol, Hh.reshape(-1, 3, 3))["counts"]
        for cnt in (hl, hh):
            bad = (cnt < c["lo"]) | (cnt > c["hi"])
            assert not bad.any(), (name, np.nonzero(bad)[0][:5])
        assert (c["lo"] < c["hi"])[hl != hh].all(), name
        tot["hyp"] += len(rows)
        tot["uncertified"] += int((c["lo"] < c["hi"]).sum())
        tot["ambiguous"] += int(c["ambiguous"][c["tight"]].sum())
        tot["differ"] += int((hl != hh).sum())
    print(tot)
    assert tot["uncertified"] > 0 and tot["ambiguous"] > 0


def test_certify_decides_clear_matches():
    """On a well-conditioned quadrilateral the bounds are tight: exact inliers and far outliers are decided, the count
    bounds collapse to one value, and the det gate is decided both ways."""
    m1, m2, s, tol = R.tie_case(R.lapack_provider)
    c = R.certify(m1, m2, s, tol)
    assert c["tight"].all() and (c["lo"] == c["hi"]).all() and (c["gate"] == 1).all()
    m1, m2, s, tol = R.late_zero_case(R.lapack_provider)
    c = R.certify(m1, m2, s, tol)
    assert (c["gate"] == -1).sum() >= 100 and (c["gate"] == 1).sum() >= 200


def test_builders_reach_their_edges():
    lp = R.lapack_provider
    # boundary: errors exactly at, one ulp below and one ulp above tol under the case's own H, and FMA-sensitive matches
    m1, m2, s, tol = R.boundary_case(lp)
    H = R.lapack_H(m1, m2, s)[0]
    err = OO.Prediction(m1, m2, H[None])[0]
    t = np.float32(tol)
    for v in (t, np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1))):
        assert (err == v).sum() >= 3
    assert ((err < t) != (R.predict_fma(m1, m2, H[None])[0] < t)).sum() >= 3
    c = R.certify(m1, m2, s, tol)
    assert c["ambiguous"][0].sum() >= 18                    # every boundary match is undecided under the DLT bound
    # tie: equal counts, at least three distinct H bit patterns, the first order wins
    m1, m2, s, tol = R.tie_case(lp)
    r = R.ransac_given_H(m1, m2, s, tol, R.lapack_H(m1, m2, s))
    assert (r["counts"] == r["counts"][0]).all() and r["best"] == 0
    Hb = R.lapack_H(m1, m2, s).reshape(-1, 9).view(np.int32)
    assert len({h.tobytes() for h in Hb}) >= 3
    assert not np.array_equal(Hb[99], Hb[0]) and not np.array_equal(Hb[100], Hb[0])
    # late zero chunk: counts > 0 before it, a full chunk of zeros, status NONE; as a remainder it is not checked
    m1, m2, s, tol = R.late_zero_case(lp)
    r = R.ransac_given_H(m1, m2, s, tol, R.lapack_H(m1, m2, s))
    assert r["status"] == R.NONE and (r["counts"][:200] > 0).all() and (r["counts"][200:300] == 0).all()
    m1, m2, s, tol = R.late_zero_case(lp, remainder=True)
    r = R.ransac_given_H(m1, m2, s, tol, R.lapack_H(m1, m2, s))
    assert r["status"] == R.OK and (r["counts"][200:] == 0).all()
    # duplicates: 50 dropped rows shift the chunk boundary by 50 raw rows
    m1, m2, s, tol = R.duplicate_case(lp)
    assert len(R.unique_rows(s)) == 150 and R.unique_rows(s)[99] > 99
    # degenerate: collinear samples with an unbounded DLT
    m1, m2, s, tol = R.degenerate_case(lp)
    c = R.certify(m1, m2, s, tol)
    assert (~c["tight"]).sum() >= 20


# ------------------------------------------------------------------ mutations: wrong kernels the exact comparison rejects
class FMA(R.Rules):
    def errors(self, match1, match2, H):
        return R.predict_fma(match1, match2, H)


class LessEqual(R.Rules):
    def inliers(self, err, tol):
        return err <= np.float32(tol)


class LastArgmax(R.Rules):
    def pick(self, counts):
        return len(counts) - 1 - int(np.argmax(counts[::-1]))


class GreaterEqual(R.Rules):
    def better(self, a, b):
        return a >= b


class RawChunks(R.Rules):
    def chunks(self, rows, nbIter, chunk):
        cid = rows // chunk
        return [(np.nonzero(cid == c)[0], c < nbIter // chunk) for c in range(int(cid.max(initial=-1)) + 1)]


class CheckRemainder(R.Rules):
    def zero_check(self, full):
        return True


class NoGate(R.Rules):
    def gate(self, H):
        return np.ones(len(H), bool)


class GateGreaterEqual(R.Rules):
    def gate(self, H):
        return OO.det3(H) >= R.DET_MIN


MUTANTS = {"fma": FMA, "less_equal": LessEqual, "last_argmax": LastArgmax, "greater_equal_across": GreaterEqual,
           "raw_chunks": RawChunks, "check_remainder": CheckRemainder, "no_det_gate": NoGate}


def visible(r):
    """What the kernel returns: status, nbInlier, mask, H bits."""
    return (r["status"], r["nbInlier"], r["mask"].tobytes(), r["H"].view(np.int32).tobytes())


@pytest.fixture(scope="module")
def gpu_cases():
    """The GPU test's built and golden cases, built with LAPACK's H, and their restatements."""
    out = []
    for name, m1, m2, s, tol in all_cases():
        if name.startswith("fuzz"):
            continue
        H = R.lapack_H(m1, m2, s)
        out.append((name, m1, m2, s, tol, H, visible(R.ransac_given_H(m1, m2, s, tol, H))))
    return out


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_exact_comparison_rejects_mutant(gpu_cases, mutant):
    """The mutant changes the status, nbInlier, mask or H bits on at least one of the GPU test's cases: the GPU test would
    fail on a kernel that computed it."""
    caught = [name for name, m1, m2, s, tol, H, ref in gpu_cases
              if visible(R.ransac_given_H(m1, m2, s, tol, H, rules=MUTANTS[mutant]())) != ref]
    print("%s: caught by %s" % (mutant, caught))
    assert caught


def test_gate_mutant_equivalent_off_threshold(gpu_cases):
    """``>=`` in the det gate differs from ``>`` only at det3 == 1e-6 exactly, which no case reaches: the exact comparison
    cannot see it, and the dropped gate stands for the gate mutants."""
    for name, m1, m2, s, tol, H, ref in gpu_cases:
        assert not (OO.det3(H) == R.DET_MIN).any(), name
        assert visible(R.ransac_given_H(m1, m2, s, tol, H, rules=GateGreaterEqual())) == ref
