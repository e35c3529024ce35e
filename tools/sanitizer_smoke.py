#!/usr/bin/env python
"""Small run of every kernel for compute-sanitizer (memcheck / racecheck / synccheck / initcheck):

    compute-sanitizer --tool racecheck python tools/sanitizer_smoke.py

Exercises the fp32 path, the tensor path (one CTA pair's worth of streams), the post-filter, the int16 entry,
the pipelined host entry, the training-data generator (records alone and with its audio), the persistent fp32 GRU chain (both block sizes), submitted
calls on the chain's anti-diagonal unit order, state export / import, a session-pool schedule (parks, unparks,
relocations, fresh starts, session export / import / reset), ragged session calls (sessions that stop early, across the
history slide and the fp32 network's 32-hop chunk), network-only calls on features and on records (both network modes),
the pitch-only kernel on tiny batches and the network trainer (ten windows, more than a recurrence CTA's eight warps,
on an active range, a call shorter than max_frames_per_call, ragged frames, then one Adam step, then two micro-batches
accumulated, exported, imported and finished before a second step); prints a checksum per leg."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from percepnet_b200 import api  # noqa: E402
from percepnet_b200.synth import synth_pairs, synth_pcm, to_int16  # noqa: E402
from percepnet_b200.weights import pack_state_dict, synth_model, synth_state_dict  # noqa: E402


def main():
    legs = sys.argv[1:] or ["fp32", "tensor", "train", "fp32chain", "submit", "sessions", "ragged", "rnn", "pitch", "trainnet"]
    m = synth_model(0)
    if "fp32" in legs:
        x = synth_pcm(5, 4, seed=3)
        e = api.Engine(5, 2, m, api.NN_FP32 | api.POSTFILTER | api.KEEP_TAPS)
        o1, gr = e.process(x[:, :960], want_gr=True)
        o2 = e.process(to_int16(x[:, 960:]))[0]
        print("fp32", float(np.abs(o1).sum()), int(np.abs(o2.astype(np.int64)).sum()), float(gr.sum()))
        e.close()
    if "tensor" in legs:
        S = 300
        x = synth_pcm(S, 3, seed=4)
        e = api.Engine(S, 2, m, api.NN_TENSOR)
        o1, gr = e.process(x[:, :960], want_gr=True)
        o2, _ = e.process(x[:, 960:], want_gr=True)
        print("tensor", float(np.abs(o1).sum()), float(np.abs(o2).sum()), float(gr.sum()))
        e.close()
    if "fp32chain" in legs:  # the persistent fp32 GRU chain: 128-stream blocks (partial last block) and 16-stream blocks
        for S, F in ((130, 5), (5, 3)):
            x = synth_pcm(S, 2 * F, seed=6)
            e = api.Engine(S, F, m, api.NN_FP32)
            o1 = e.process(x[:, :F * 480])[0]
            o2 = e.process(x[:, F * 480:])[0]
            blob = e.get_state(S - 1)
            e.set_state(0, blob)
            print("fp32chain", S, float(np.abs(o1).sum()), float(np.abs(o2).sum()), len(blob))
            e.close()
    if "submit" in legs:     # pipelined host calls in flight together, anti-diagonal unit order (few streams)
        S, F = 300, 6
        x = synth_pcm(S, 3 * F, seed=8)
        e = api.Engine(S, F, m, api.NN_TENSOR | api.CONV_WIDE)
        outs = [np.empty((S, F * 480), np.float32) for _ in range(3)]
        for k in range(3):
            e.submit(np.ascontiguousarray(x[:, k * F * 480:(k + 1) * F * 480]), outs[k])
        e.wait()
        print("submit", [float(np.abs(o).sum()) for o in outs])
        e.close()
    if "sessions" in legs:   # session pool on both network modes: every kind of move, list sizes across a row tile
        for flags in (api.NN_FP32, api.NN_TENSOR):
            S, N, F = 130, 400, 2
            e = api.Engine(S, F, m, flags)
            e.reserve_sessions(N)
            rng = np.random.RandomState(13)
            x = synth_pcm(S, F, seed=14)
            sums = []
            for c, k in enumerate((129, 130, 1, 128, 130, 64)):
                ids = rng.choice(N if c > 2 else 200, size=k, replace=False).astype(np.int32)
                if c == 3:
                    e.reset_sessions(ids[:3])
                    blobs = e.export_sessions(ids[3:9], None)
                    e.import_sessions(ids[9:15], blobs)
                o, gr = e.process_sessions(ids, x[:k], want_gr=True)
                sums.append(float(np.abs(o).sum()) + float(gr.sum()))
            e.wait()
            print("sessions", flags, sums, e.session_stats())
            e.close()
    if "ragged" in legs:     # ragged session calls on both network modes; max_frames 33 crosses the fp32 32-hop chunk
        for flags in (api.NN_FP32, api.NN_TENSOR):
            S, N, F = 130, 300, 33
            e = api.Engine(S, F, m, flags)
            e.reserve_sessions(N)
            rng = np.random.RandomState(15)
            x = synth_pcm(S, F, seed=16)
            sums = []
            for c, k in enumerate((129, 130, 1, 128, 130, 64)):
                ids = rng.choice(N, size=k, replace=False).astype(np.int32)
                hops = rng.randint(1, F + 1, size=k).astype(np.int32)
                w = int(hops.max())
                o, gr = e.process_sessions(ids, np.ascontiguousarray(x[:k, :w * 480]), want_gr=True, hops=hops)
                sums.append(float(np.abs(o).sum()) + float(gr.sum()))
            e.wait()
            print("ragged", flags, sums)
            e.close()
    if "rnn" in legs:        # network-only calls on both network modes: features, then records, on an active range
        for flags in (api.NN_FP32, api.NN_TENSOR):
            S, F = 130, 3
            e = api.Engine(S, F, m, flags | api.KEEP_TAPS)
            e.process(synth_pcm(S, F, seed=17))
            f = np.ascontiguousarray(e.read_tap("features", F).transpose(1, 0, 2))
            e.set_active(129)
            g1 = e.compute_rnn(f[:129])
            rec = np.zeros((129, F, 138), np.float32)
            rec[:, :, :68], rec[:, :, 68:70] = f[:129, :, :68] / np.float32(30), f[:129, :, 68:]
            g2 = e.compute_rnn(rec)
            print("rnn", flags, float(g1.sum()), float(g2.sum()))
            e.close()
    if "pitch" in legs:
        buf = synth_pcm(40, 4, seed=12)[:, :1728].copy()
        r = api.pitch_only(buf, np.zeros(40, np.int32), np.zeros(40, np.float32))
        print("pitch", [float(np.asarray(a, np.float64).sum()) for a in r])
    if "train" in legs:
        c, n = synth_pairs(6, 5, seed=9)
        e = api.Engine(12, 3, None, api.TRAIN_DATA)
        r1 = e.train_records(c[:, :3 * 480], n[:, :3 * 480])
        r2 = e.train_records(c[:, 3 * 480:], n[:, 3 * 480:])
        print("train", float(r1.sum()), float(r2.sum()))
        e.close()
        c, n = synth_pairs(6, 10, seed=9)        # output frame t carries input frame t - 6: ten frames, audible audio
        e = api.Engine(12, 5, None, api.TRAIN_DATA | api.TRAIN_AUDIO)   # with the resynthesis of the noisy rows
        r3, a3 = e.train_audio(c[:, :5 * 480], n[:, :5 * 480])
        r4, a4 = e.train_audio(c[:, 5 * 480:], n[:, 5 * 480:])
        print("train_audio", float(r3.sum()), float(r4.sum()), int(np.abs(a3.astype(np.int64)).sum()),
              int(np.abs(a4.astype(np.int64)).sum()))
        e.close()
    if "trainnet" in legs:   # 12 slots, 10 active, F = 6 of Fmax 8, windows ending after 1 to 6 hops
        rng = np.random.RandomState(18)
        rec = rng.rand(10, 6, 138).astype(np.float32)
        rec[..., :68] *= np.float32(0.05)
        e = api.Engine(12, 8, pack_state_dict(synth_state_dict(0)), api.TRAIN_NETWORK)
        e.set_active(10)
        sums = e.train_grad(rec, [3, 6, 1, 6, 2, 5, 4, 6, 1, 6])
        e.train_adam(1e-3, 1)
        e.wait()
        print("trainnet", float(sums.sum()), float(np.abs(e.train_export("gradient").astype(np.float64)).sum()),
              float(e.train_export("weights").astype(np.float64).sum()))
        # two micro-batches accumulated, the accumulator through the host and back, finished, one more Adam step
        e.train_grad(rec, [6] * 10)
        e.train_accumulate()
        e.train_grad(rec, [1, 2, 3, 4, 5, 6, 5, 4, 3, 2])
        e.train_accumulate()
        e.train_import("accum", e.train_export("accum"))
        e.train_finish()
        e.train_adam(1e-3, 2)
        e.wait()
        print("trainaccum", float(np.abs(e.train_export("gradient").astype(np.float64)).sum()),
              float(e.train_export("weights").astype(np.float64).sum()))
        e.close()


if __name__ == "__main__":
    main()
