"""Launch accounting: pnb_launch_count and the profile (pnb_profile_read) see the same launches.  With profiling on,
every call's profile records add up to the launches it added to the count, less the ones the profile leaves out (a
session call's state launch when its residency changed, and the gather of its g/r into list order); a training-record
call's two stage_in launches are two records.  State operations and the trainer add their launches to the count and
nothing to the profile."""
import numpy as np
import pytest

from percepnet_b200.synth import synth_pairs
from percepnet_b200.weights import synth_state_dict
from test_gpu_lifecycle import _engine, _signal
from test_gpu_parity import api  # noqa: F401
from test_gpu_train import moderate_records, trainer

pytestmark = pytest.mark.gpu

HOP = 480


def _counted(e, call):
    """Runs call() on e with profiling on: (launches it added, {class: profile records}, its result)."""
    e.profile(True)
    e.profile_read()
    n0 = e.launches
    out = call()
    prof = {k: n for k, (_, n) in e.profile_read().items()}
    return e.launches - n0, prof, out


def _moved(e, before):
    """1 when a session call changed the pool's residency (it then issued the state launch), else 0."""
    return int(e.session_stats() != before)


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_profile_records_match_launch_count(api, model0, mode):
    """Slot, network, score and split calls on a slot engine, session and ragged calls on a pool: each call's profile
    records equal its launches, but for the state launch and the g/r gather of a session call."""
    S, F = 16, 4
    e = _engine(api, model0, S, mode, Fm=F)
    x = _signal(S, 3, 11)
    rng = np.random.RandomState(5)
    slides = 0
    for k in range(10):  # ten calls cross a history slide (every eighth call at most)
        xk = np.ascontiguousarray(x[:, (k % 6) * F * HOP:(k % 6 + 1) * F * HOP])
        n, prof, _ = _counted(e, lambda: e.process(xk, want_gr=True))
        assert n == sum(prof.values()), (k, n, prof)
        assert n in (e.launches_per_call(F), e.launches_per_call(F) + 1), (k, n)
        slides += prof.get("slide_history_kernel", 0)
    assert slides >= 1
    feats = rng.rand(S, F, 70).astype(np.float32)
    n, prof, _ = _counted(e, lambda: e.compute_rnn(feats))
    assert n == sum(prof.values()) == e.launches_per_call(F) - 3 + 2, prof
    rec = rng.rand(S, F, 138).astype(np.float32)
    for want_gr in (False, True):
        n, prof, _ = _counted(e, lambda: e.score_records(rec, want_gr=want_gr))
        assert n == sum(prof.values()), (want_gr, n, prof)
    n, prof, feat = _counted(e, lambda: e.analyze(np.ascontiguousarray(x[:, :F * HOP])))
    assert n == sum(prof.values()) == 3, prof
    gr = rng.rand(S, F, 68).astype(np.float32)
    n, prof, _ = _counted(e, lambda: e.synthesize(gr))
    assert n == sum(prof.values()) and n in (2, 3), prof
    e.check()
    e.close()

    p = _engine(api, model0, S, mode, Fm=F)
    p.reserve_sessions(48)
    moves = []
    for k, ids in enumerate([np.arange(8), np.arange(4, 16), np.arange(20, 36), np.arange(20, 36)]):
        ids = ids.astype(np.int32)
        xs = np.ascontiguousarray(x[:len(ids), :F * HOP])
        before = p.session_stats()
        n, prof, _ = _counted(p, lambda: p.process_sessions(ids, xs))
        moves.append(_moved(p, before))
        assert n == sum(prof.values()) + moves[-1], (k, n, prof)
    assert moves[2] == 1 and moves[3] == 0, moves  # the third list parks residents; its repeat moves nothing
    ids = np.array([3, 30, 7, 25, 40], np.int32)
    hops = np.array([F, 1, 2, F, 3], np.int32)
    xs = np.ascontiguousarray(x[:len(ids), :F * HOP])
    before = p.session_stats()
    n, prof, _ = _counted(p, lambda: p.process_sessions(ids, xs, want_gr=True, hops=hops))
    assert n == sum(prof.values()) + _moved(p, before) + 1, (n, prof)   # + the g/r gather
    assert prof.get("slide_history_kernel", 0) >= 1, prof                 # the fix-up of the short sessions
    p.check()
    p.close()


@pytest.mark.parametrize("audio", [False, True], ids=["records", "audio"])
def test_training_record_call_profiles_each_stage_in(api, audio):
    """A training-record call stages speech and noisy in two launches: two stage_in_kernel records, and as many
    records in all as launches."""
    N, F = 3, 8
    e = api.Engine(2 * N, F, None, api.TRAIN_DATA | (api.TRAIN_AUDIO if audio else 0))
    clean, noisy = synth_pairs(N, 3 * F, seed=31)
    for k in range(3):
        c, m = (np.ascontiguousarray(a[:, k * F * HOP:(k + 1) * F * HOP]) for a in (clean, noisy))
        n, prof, _ = _counted(e, lambda: e.train_audio(c, m) if audio else e.train_records(c, m))
        assert prof["stage_in_kernel"] == 2, prof
        assert n == sum(prof.values()), (k, n, prof)
        # two stage_in, analysis, labels, the resynthesis of an audio engine, and the occasional history slide
        # (pnb_launches_per_call of a training-data engine counts the enhancement schedule instead)
        assert n in (4 + audio, 5 + audio), (k, n)
    e.wait()
    e.close()


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_state_operations_are_counted_not_profiled(api, model0, mode):
    """A reset adds one launch, an import two, and neither adds a profile record."""
    import torch
    S = 16
    e = _engine(api, model0, S, mode, Fm=4)
    e.process(np.ascontiguousarray(_signal(S, 1, 3)[:, :4 * HOP]))
    blobs = e.export_states([1, 2], None)
    torch.cuda.synchronize()
    for name, op, want in (("reset", lambda: e.reset_streams([0, 5]), 1),
                           ("import", lambda: e.import_states([7, 8], blobs), 2)):
        n, prof, _ = _counted(e, op)
        assert (n, prof) == (want, {}), name
    e.check()
    e.close()


def test_trainer_is_counted_not_profiled(api):
    """train_grad adds train_grad_launches (pnb_launches_per_call), Adam one launch, accumulate one and finish two;
    none of them adds a profile record."""
    B, T = 4, 20
    e = trainer(synth_state_dict(1), B, T)
    rec = moderate_records(B, T, 77)
    for name, op, want in (("grad", lambda: e.train_grad(rec), e.launches_per_call(T)),
                           ("adam", lambda: e.train_adam(1e-3, 1), 1),
                           ("grad", lambda: e.train_grad(rec), e.launches_per_call(T)),
                           ("accumulate", e.train_accumulate, 1),
                           ("finish", e.train_finish, 2)):
        n, prof, _ = _counted(e, op)
        assert (n, prof) == (want, {}), name
    assert e.launches_per_call(T) == 118
    e.wait()
    e.close()
