"""Pins the CPU restatement of train()'s TEST block (tests/train_audio_oracle.py, composed from the oracle's stage
functions: test_input.pcm / test_output.pcm, src/denoise.cpp:722-728, 742-759) to the compiled, unmodified reference,
BIT FOR BIT, together with the records.
Where the reference library has been built (oracle/_ref) its train() runs live, and the files it leaves beside its
output are compared directly; the outputs must also hash to tests/golden/train_audio_digests.json, which
PNB_RECORD_REFERENCE=1 rewrites from the live reference instead.  CPU only."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from train_audio_oracle import train_audio
from util import digest

DIGESTS = os.path.join(GOLDEN, "train_audio_digests.json")


class AudioRef:
    """`check(key, speech_file, noisy_file, count, got)`: got = (records, test_input, test_output) of the oracle."""

    def __init__(self, tmp):
        from oracle import ffi
        ffi.build()
        self.tmp = tmp
        self.ref = ffi.Reference() if ffi.Reference.available() else None
        self.record = os.environ.get("PNB_RECORD_REFERENCE") == "1"
        if self.record and self.ref is None:
            raise RuntimeError("PNB_RECORD_REFERENCE=1 needs the compiled reference (oracle/_ref)")
        self.table = {} if self.record else json.load(open(DIGESTS))

    def live(self, speech, noisy, count):
        """train() on the two int16 arrays written as files; its record file and the TEST audio it wrote beside it."""
        fc, fn, fo = (str(self.tmp / nm) for nm in ("speech.pcm", "noisy.pcm", "out.f32"))
        speech.tofile(fc)
        noisy.tofile(fn)
        assert self.ref.train_files(fc, fn, count, fo) == 0
        return (np.fromfile(fo, np.float32).reshape(count, 138), np.fromfile(str(self.tmp / "test_input.pcm"), np.int16),
                np.fromfile(str(self.tmp / "test_output.pcm"), np.int16))

    def __call__(self, key, speech, noisy, count, got):
        if self.ref is not None:
            want = self.live(speech, noisy, count)
            assert np.array_equal(got[0].view(np.int32), want[0].view(np.int32)), (key, "records")
            assert np.array_equal(got[1], want[1]), (key, "test_input")
            assert np.array_equal(got[2], want[2]), (key, "test_output", np.abs(got[2].astype(np.int32) - want[2]).max())
            if self.record:
                self.table[key] = digest(*want)
                return
        assert key in self.table, f"no stored reference digest for {key}"
        assert digest(*got) == self.table[key], key


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    rc = AudioRef(tmp_path_factory.mktemp("train_audio"))
    yield rc
    if rc.record:
        with open(DIGESTS, "w") as f:
            json.dump(rc.table, f, indent=0, sort_keys=True)
            f.write("\n")


def test_pairs_at_several_snrs(oracle, ref):
    """Speech-like pairs from clean to -5 dB: the comb branch (pitch_filter) runs on most frames, and the records are
    those of pn_oracle_train_records."""
    from percepnet_b200.synth import synth_pairs
    n = 40
    clean, noisy = synth_pairs(5, n, seed=91)
    for k in range(5):
        got = train_audio(oracle, clean[k], noisy[k])
        assert np.array_equal(got[0].view(np.int32), oracle.train_records(clean[k], noisy[k]).view(np.int32))
        assert np.array_equal(got[1], noisy[k])               # the clamp of test_input.pcm is a no-op on int16
        assert np.any(got[2] != 0)
        ref(f"snr/{k}", clean[k], noisy[k], n, got)


def test_file_shorter_than_count(oracle, ref):
    """train() re-reads a file from its start at EOF; the restatement is fed read_cyclic_frames' view of the files."""
    from percepnet_b200.gen_features import read_cyclic_frames
    from percepnet_b200.synth import synth_pairs
    clean, noisy = synth_pairs(1, 12, seed=92)
    c, n, count = clean[0][:9 * 480 + 100], noisy[0][:12 * 480], 30
    tmp = ref.tmp
    c.tofile(str(tmp / "wc")), n.tofile(str(tmp / "wn"))
    got = train_audio(oracle, read_cyclic_frames(str(tmp / "wc"), count), read_cyclic_frames(str(tmp / "wn"), count))
    ref("wrap", c, n, count, got)


def test_silent_noisy_file(oracle, ref):
    """An all-zero noisy file: every frame silent (no pitch_filter), and the resynthesis is silence; then a noisy file
    with a silent stretch in the middle."""
    from percepnet_b200.synth import synth_pairs
    n = 24
    clean, noisy = synth_pairs(1, n, seed=93)
    z = np.zeros_like(noisy[0])
    got = train_audio(oracle, clean[0], z)
    assert not np.any(got[2])
    ref("silent", clean[0], z, n, got)
    gap = noisy[0].copy()
    gap[6 * 480:16 * 480] = 0
    ref("gap", clean[0], gap, n, train_audio(oracle, clean[0], gap))


def test_clamped_resynthesis(oracle, ref):
    """A pair loud enough that the resynthesis leaves the int16 range: the clamp to [-32768, 32767] is hit."""
    n = 24
    t = np.arange(n * 480) / 48000.0
    sq = np.sign(np.sin(2 * np.pi * 150 * t)) + 0.6 * np.sign(np.sin(2 * np.pi * 450 * t + 1))
    loud = np.clip(np.rint(sq * 32767), -32768, 32767).astype(np.int16)
    got = train_audio(oracle, loud, loud)
    assert np.any(got[2] == 32767) and np.any(got[2] == -32768), (got[2].min(), got[2].max())
    ref("clamp", loud, loud, n, got)
