"""Pin bookkeeping of the layer programs (program.py): a graphed aligner's record pins the compiled entries its CUDA graphs point
into, an entry goes with its last pin, an entry nobody pinned stays, and a recording scope collects the entries that
``LayerProgram.run`` uses inside it.  Programs compiled on the CPU; the library call is stubbed out, so no kernel runs."""
import types

import torch

from oracle import synth


def program(rf):
    fe = rf.model.FeatureExtractor()
    fe.load_state_dict(synth.feature_extractor_state(0))
    fe.eval()
    return fe._fold_build(False)


def key(h, w):
    return (((h, w),), "cpu", 0)


def test_an_entry_goes_with_its_last_pin(rf):
    P = program(rf)
    a, b, c = key(32, 48), key(16, 24), key(8, 8)
    for k in (a, b, c):
        P._compiled[k] = P._compile(list(k[0]), torch.device("cpu"))
    P.pin(a)                                 # two records' graphs point into a, one into c
    P.pin(a)
    P.pin(c)
    P.unpin(a)
    assert a in P._compiled
    P.unpin(c)
    assert c not in P._compiled and a in P._compiled
    P.unpin(a)
    assert a not in P._compiled
    assert b in P._compiled                  # used eagerly only: never pinned, never deleted
    assert P._pins == {}


def test_recording_collects_what_run_uses_inside_the_scope(rf, monkeypatch):
    prog = rf.program
    monkeypatch.setattr(prog, "need_cuda", lambda *t: None)
    monkeypatch.setattr(prog, "lib", types.SimpleNamespace(rf_run_layers=lambda *a: 0))
    monkeypatch.setattr(prog, "stream", lambda: None)
    P, Q = program(rf), program(rf)

    def run(p, h, w):
        p.run(rf.ops.Ragged(torch.zeros(h * w, 3), [(h, w)]), 0)

    run(P, 32, 48)                           # before the scope
    with prog.recording() as used:
        run(P, 32, 48)
        run(Q, 16, 24)
        with prog.recording() as inner:
            run(P, 8, 8)
    run(P, 24, 24)                           # after it
    run(Q, 40, 40)
    assert used == {(P, key(32, 48)), (Q, key(16, 24)), (P, key(8, 8))}
    assert inner == {(P, key(8, 8))}
    assert set(P._compiled) == {key(32, 48), key(8, 8), key(24, 24)} and set(Q._compiled) == {key(16, 24), key(40, 40)}
    assert P._pins == {} and Q._pins == {}   # recording pins nothing
