"""Host parts of the graphed evalYFCC pair (``pipeline.align_pair_yfcc_graph`` / ``GraphedYfccAligner``): the select record's
layout, the orientation classes, the slot chain against the eager path's draw-and-rewind sequence, and the C ABI export.  No GPU."""
import ctypes

import numpy as np
import pytest
import torch


def eager_draws(rot_counts, loop_counts, alive, nbPoint=4):
    """The eager path's draw sequence (``align_pair_yfcc``): rotations draw in order when they have nbPoint matches; the loop
    calls ``getCoarse`` until a call draws nothing (None before ``torch.randint``, the generator rewound) or a hypothesis dies.
    Returns, per call the eager path makes, the index of the table it draws (None: no draw)."""
    drawn, out = 0, []
    for m in rot_counts:
        out.append(drawn if m >= nbPoint else None)
        drawn += m >= nbPoint
    for m, a in zip(loop_counts, alive):
        if m < nbPoint:
            out.append(None)
            break
        out.append(drawn)
        drawn += 1
        if not a:
            break
    return out


def test_record_layout_matches_the_header(rf):
    from conftest import ROOT
    import os
    hdr = open(os.path.join(ROOT, "include", "ransacflow_b200.h")).read()
    Y = rf.yfcc_graph
    for name, v in (("WINNER", Y.REC_WINNER), ("SCORES", Y.REC_SCORES), ("DRAWN", Y.REC_DRAWN), ("ERROR", Y.REC_ERROR),
                    ("CLASS", Y.REC_CLASS), ("WORDS", Y.REC_WORDS)):
        assert "#define RF_YFCC_REC_%s %d" % (name, v) in hdr, name


def test_unpack_record(rf):
    rec = np.array([2, 7, 0, 9, 9, 3, 0, 0], dtype=np.int32)
    assert rf.yfcc_graph.unpack_record(rec) == (2, [7, 0, 9, 9], 3, False, 0)
    rec = np.array([3, 0, 1, 2, 5, 4, 1, 1], dtype=np.int32)
    assert rf.yfcc_graph.unpack_record(rec) == (3, [0, 1, 2, 5], 4, True, 1)
    with pytest.raises(TypeError):
        rf.yfcc_graph._raise_on_error(rec)
    rf.yfcc_graph._raise_on_error(np.zeros(8, dtype=np.int32))


def test_result_dict(rf):
    """A select record and two loop records (the second dead) give align_pair_yfcc's keys, the angle and the scores."""
    f8 = (1, 2, 3, 4)
    n8 = int(np.prod(f8))
    rows = [np.concatenate([[a, 0, 40 + k, 20 + k], np.arange(9) + 10 * k, np.full(n8, k + 0.5), np.full(2 * n8, k + 0.25)])
            for k, a in enumerate((1, 0))]
    host = np.concatenate(rows).astype(np.float32)
    rec = np.array([1, 3, 8, 8, 0, 3, 0, 1], dtype=np.int32)
    out = rf.yfcc_graph._result(rec, host, None, (24, 32), f8, 1)
    assert out["angle"] == 90 and out["nbInlierRot"] == [3, 8, 8, 0]
    assert out["H"].shape == (1, 3, 3) and out["H"].dtype == np.float32 and np.array_equal(out["H"][0].reshape(-1), np.arange(9))
    assert out["flowDown8"].shape == (1, 2, 3, 4) and out["matchDown8"].shape == (1, 2, 3, 4) and out["nbMatch"] == [40]
    assert out["It_bg"].shape == (24, 32) and out["It_bg"].dtype == bool and out["It_bg"].all()
    bg = np.zeros(24 * 32, dtype=np.float32)
    bg[5] = 1
    out = rf.yfcc_graph._result(rec, host, bg, (24, 32), f8, 1)
    assert out["It_bg"].sum() == 1 and out["It_bg"][0, 5]


def test_orientation_classes(rf):
    C = rf.yfcc_graph.orientation_classes
    assert C([(128, 96), (96, 128), (128, 96), (96, 128)]) == {0: [0, 2], 1: [1, 3]}
    assert C([(96, 96)] * 4) == {0: [0, 1, 2, 3], 1: [0, 1, 2, 3]}
    # the rotated targets' sizes come from the resize of the rotated original, which is the transposed size
    c = type("C", (), {"resize_mode": "min", "strideNet": 16})()
    ts = rf.CoarseAlignB._target_size
    for w, h, minSize in ((640, 480, 480), (1024, 683, 480), (500, 500, 96), (128, 96, 96), (97, 131, 96)):
        sizes = [ts(c, w, h, minSize) if k % 2 == 0 else ts(c, h, w, minSize) for k in range(4)]
        cl = C(sizes)
        assert sizes[1] == sizes[0][::-1]
        assert cl[0] == ([0, 1, 2, 3] if sizes[0] == sizes[1] else [0, 2])
        assert cl[1] == ([0, 1, 2, 3] if sizes[0] == sizes[1] else [1, 3])


@pytest.mark.parametrize("seed", range(40))
def test_slot_chain_reads_the_eager_draws(rf, seed):
    """Random match counts (many below 4) and alive flags: every call the eager path makes that draws reads, through the slot
    chain, the table the eager path draws for it; the chain never reads past T = 4 + maxCoarse + 1 tables."""
    rs = np.random.RandomState(seed)
    maxCoarse = int(rs.randint(0, 11))
    rot = rs.choice([0, 2, 3, 4, 5, 50], size=4).tolist()
    loop = rs.choice([0, 3, 4, 9, 100], size=maxCoarse + 1).tolist()
    alive = (rs.rand(maxCoarse + 1) < 0.7).tolist()
    chain = rf.yfcc_graph.slot_chain(rot + loop)
    want = eager_draws(rot, loop, alive)
    assert len(chain) == 4 + maxCoarse + 1 and max(chain) <= 4 + maxCoarse
    for i, t in enumerate(want):
        if t is not None:
            assert chain[i] == t, (i, chain, want)
    # the rotations that draw are pipeline.rotation_draws'
    assert [k for k in range(4) if want[k] is not None] == rf.pipeline.rotation_draws(rot)


def test_entry_points_are_exported(rf):
    lib = ctypes.CDLL(rf._lib.LIB_PATH)
    for s in ("rf_ransac_homography_drawn", "rf_yfcc_rotation_select", "rf_select_copy"):
        assert hasattr(lib, s) and s in rf._lib.SIGNATURES


def test_entry_points_refuse_host_tensors(rf):
    z = torch.zeros((8, 3))
    i = torch.zeros(1, dtype=torch.int32)
    Y = rf.yfcc_graph
    with pytest.raises(rf._lib.RFError):
        Y.ransac_homography_drawn(z, z, torch.zeros((2, 10, 4), dtype=torch.int64), i, i.clone(), 0.05, i, rf.ops.SAMPLES_MOD)
    with pytest.raises(rf._lib.RFError):
        Y.rotation_select([i] * 4, [i] * 4, [torch.zeros(3, dtype=torch.uint8)] * 4)
    with pytest.raises(rf._lib.RFError):
        Y.select_copy([z, None], i, z.clone())


def test_graph_aligner_needs_segnet_weights(rf):
    c = type("C", (), {"segNet": None})()
    with pytest.raises(NotImplementedError):
        rf.pipeline.GraphedYfccAligner(c, {}, segNet=True)
