"""ransac_kernel bit for bit against the restatement of utils/outil.py:117-164 on the kernel's own DLT
(tests/ransac_ref.ransac_given_H fed with ``ops.homography_dlt``), and every disagreement with LAPACK's DLT inside the
certified count bounds (tests/ransac_ref.certify)."""
import numpy as np
import pytest
import torch

import ransac_ref as R
from conftest import golden
from oracle import synth

pytestmark = pytest.mark.gpu
f32 = np.float32
GOLDEN = ["ransac_m120", "ransac_m636", "ransac_grid", "ransac_remainder_only", "ransac_none", "ransac_lowinlier"]


def kernel_provider(rf):
    """H_of for the case builders: the kernel's DLT (dlt_kernel) of (N, 4, 3) sources and targets."""
    def H_of(X, Y):
        X, Y = np.ascontiguousarray(X, f32), np.ascontiguousarray(Y, f32)
        if len(X) == 0:
            return np.zeros((0, 3, 3), f32)
        return rf.ops.homography_dlt(torch.from_numpy(X).cuda(), torch.from_numpy(Y).cuda()).cpu().numpy()
    return H_of


def run_kernel(rf, m1, m2, raw, tol, M_dev=None, mode=None):
    Md = None if M_dev is None else torch.tensor([M_dev], dtype=torch.int32).cuda()
    H, nb, mask, st = rf.ops.ransac_homography(torch.from_numpy(m1).cuda(), torch.from_numpy(m2).cuda(),
                                               torch.from_numpy(np.ascontiguousarray(raw, np.int64)).cuda(), tol, 100, Md, mode)
    torch.cuda.synchronize()
    return dict(status=int(st.item()), H=H.cpu().numpy().reshape(3, 3), nbInlier=int(nb.item()),
                mask=mask.cpu().numpy().astype(bool))


def check_exact(rf, m1, m2, samples, tol, raw=None, M_dev=None, mode=None, what=""):
    """The kernel on (raw, M_dev, mode) returns what ransac_given_H returns on the index table ``samples`` (over the first
    M_dev matches) with the kernel's DLT of its unique rows: status, nbInlier, mask and H bits.  Returns the restatement."""
    M = len(m1) if M_dev is None else min(M_dev, len(m1))
    a1, a2 = m1[:M], m2[:M]
    us = np.asarray(samples).reshape(-1, 4)[R.unique_rows(samples)]
    exp = R.ransac_given_H(a1, a2, samples, tol, kernel_provider(rf)(a1[us], a2[us]))
    got = run_kernel(rf, m1, m2, samples if raw is None else raw, tol, M_dev, mode)
    assert got["status"] == exp["status"], (what, got["status"], exp["status"])
    assert got["nbInlier"] == exp["nbInlier"], what
    assert np.array_equal(got["mask"][:M], exp["mask"]) and not got["mask"][M:].any(), what
    assert np.array_equal(got["H"].view(np.int32), exp["H"].view(np.int32)), what
    return exp


def check_certified(m1, m2, samples, tol, exp, what=""):
    """The kernel's per-hypothesis counts (``exp``, the exact restatement) and LAPACK's lie in certify's bounds; counts that
    differ belong to uncertified hypotheses; when both choose the same hypothesis their masks differ only at ambiguous
    matches.  Returns (uncertified hypotheses, ambiguous matches of certified-DLT hypotheses, hypotheses whose counts
    differ, LAPACK's restatement)."""
    c = R.certify(m1, m2, samples, tol)
    lap = R.ransac_given_H(m1, m2, samples, tol, R.lapack_H(m1, m2, samples))
    for who, r in (("kernel", exp), ("lapack", lap)):
        bad = (r["counts"] < c["lo"]) | (r["counts"] > c["hi"])
        assert not bad.any(), "%s: %s count outside its certified bounds at hypotheses %s" % (what, who, np.nonzero(bad)[0][:5])
    differ = exp["counts"] != lap["counts"]
    assert (c["lo"] < c["hi"])[differ].all(), what
    if exp["best"] is not None and exp["best"] == lap["best"]:
        assert not (exp["mask"] != lap["mask"])[~c["ambiguous"][exp["best"]]].any(), what
    return int((c["lo"] < c["hi"]).sum()), int(c["ambiguous"][c["tight"]].sum()), int(differ.sum()), lap


def exact_and_certified(rf, m1, m2, samples, tol, what=""):
    exp = check_exact(rf, m1, m2, samples, tol, what=what)
    unc, amb, differ, lap = check_certified(m1, m2, samples, tol, exp, what)
    print("%s: status %d nbInlier %d (LAPACK %d %d); %d hypotheses, %d uncertified, %d ambiguous matches, %d counts differ"
          % (what, exp["status"], exp["nbInlier"], lap["status"], lap["nbInlier"], len(exp["counts"]), unc, amb, differ))
    return exp, lap, unc, amb


@pytest.mark.parametrize("name", sorted(R.BUILDERS))
def test_built_cases(rf, name):
    """The hand-built cases, constructed against the kernel's own DLT."""
    m1, m2, s, tol = R.BUILDERS[name](kernel_provider(rf))
    exp, lap, unc, amb = exact_and_certified(rf, m1, m2, s, tol, name)
    expect = {"late_zero": R.NONE}.get(name, R.OK)
    assert exp["status"] == expect
    if name == "boundary":
        assert amb > 0 and exp["best"] == 0
        t = f32(tol)
        err = R.OO.Prediction(m1, m2, exp["H"][None])[0]
        assert (err == t).any() and not exp["mask"][err == t].any()          # exactly tol is an outlier
    if name == "tie":
        assert (exp["counts"] == exp["counts"][0]).all() and exp["best"] == 0
    if name == "degenerate":
        assert unc > 0


@pytest.mark.parametrize("name", GOLDEN)
def test_golden_cases_exact(rf, name):
    g = golden(name)
    exact_and_certified(rf, g["match1"], g["match2"], g["samples"], float(g["tol"]), name)


@pytest.mark.parametrize("case", range(24))
def test_fuzz_grid_and_continuous(rf, case):
    rs = np.random.RandomState(4000 + case)
    M = int(rs.choice([4, 6, 37, 200, 636, 1500]))
    nbIter = int(rs.choice([1, 99, 100, 101, 777, 2500]))
    frac = float(rs.choice([0.0, 0.2, 0.6, 0.95]))
    tol = float(rs.choice([0.005, 0.02, 0.05, 0.1]))
    m1, m2, _ = synth.make_matches(4000 + case, M, frac, grid=(30, 40) if case % 2 else None)
    exact_and_certified(rf, m1, m2, synth.draw_samples(4000 + case, M, nbIter), tol, "fuzz%d" % case)


def launch_sizes(sms):
    """nbIter around the launcher's switches: G = 128 from 256 #SM, the grid-stride loop beyond 128 #SM (G = 32) and 512
    #SM (G = 128); 2 groups per CTA below 256 #SM and about 2.1 above 1100 #SM."""
    return [128 * sms, 128 * sms + 1, 256 * sms - 1, 256 * sms, 512 * sms, 512 * sms + 1, 1100 * sms + 37]


def test_launch_sizes_straddle_the_switches(rf):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = launch_sizes(sms)
    for i, n in enumerate(sizes):
        G = 128 if n >= 256 * sms else 32
        groups = (n + G - 1) // G
        print("nbIter %d: G %d, %d groups on %d CTAs" % (n, G, groups, min(groups, 4 * sms)))
        m1, m2, _ = synth.make_matches(300 + i, 48, 0.5)
        s = synth.draw_samples(300 + i, 48, n)
        exp = check_exact(rf, m1, m2, s, 0.05, what="nbIter %d" % n)
        check_certified(m1, m2, s, 0.05, exp, "nbIter %d" % n)
    assert any(-(-n // 32) > 4 * sms for n in sizes if n < 256 * sms)
    assert any(-(-n // 128) > 4 * sms for n in sizes if n >= 256 * sms)


def test_sample_modes_equal_their_index_tables(rf):
    """SAMPLES_MOD (raw % M, M from the device) and SAMPLES_PHILOX64 (high word % M) against the reduced index table."""
    ops = rf.ops
    m1, m2, _ = synth.make_matches(17, 300, 0.6)
    raw = synth.draw_samples(17, 2 ** 31 - 1, 3000)
    for Md in (300, 211):
        red = raw % Md
        check_exact(rf, m1, m2, red, 0.05, raw=raw, M_dev=Md, mode=ops.SAMPLES_MOD, what="mod %d" % Md)
        check_exact(rf, m1[:Md].copy(), m2[:Md].copy(), red, 0.05, mode=ops.SAMPLES_INDEX, what="index %d" % Md)
    words = np.random.RandomState(18).randint(-2 ** 63, 2 ** 63 - 1, (3000, 4), dtype=np.int64)
    red = ((words.view(np.uint64) >> np.uint64(32)) % np.uint64(300)).astype(np.int64)
    check_exact(rf, m1, m2, red, 0.05, raw=words, mode=ops.SAMPLES_PHILOX64, what="philox")
    check_exact(rf, m1, m2, red, 0.05, mode=ops.SAMPLES_INDEX, what="philox reduced")


def test_too_few_device_matches(rf):
    """M_dev < 4 with M_host >= 4: status TOO_FEW, zero outputs over all M_host matches."""
    m1, m2, _ = synth.make_matches(19, 50, 0.6)
    raw = synth.draw_samples(19, 2 ** 31 - 1, 300)
    for Md in (0, 1, 3):
        got = run_kernel(rf, m1, m2, raw, 0.05, Md)
        assert got["status"] == R.TOO_FEW and got["nbInlier"] == 0 and not got["mask"].any() and not got["H"].any()
    check_exact(rf, m1, m2, raw % 4, 0.05, raw=raw, M_dev=4, what="M_dev 4")


def test_zero_and_one_iteration(rf):
    m1, m2, _ = synth.make_matches(20, 60, 0.6)
    got = run_kernel(rf, m1, m2, np.zeros((0, 4), np.int64), 0.05)
    assert got["status"] == R.NO_MODEL and got["nbInlier"] == 0 and not got["mask"].any()
    assert R.ransac_given_H(m1, m2, np.zeros((0, 4), np.int64), 0.05, np.zeros((0, 3, 3), f32))["status"] == R.NO_MODEL
    for row in ([[0, 1, 2, 3]], [[5, 9, 33, 41]], [[7, 7, 1, 2]]):
        exact_and_certified(rf, m1, m2, np.array(row, np.int64), 0.05, "one row %s" % row)
