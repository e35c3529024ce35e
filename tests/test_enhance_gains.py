"""The batch CLI's --gains input (percepnet_b200.enhance): a gains file that does not hold n_frames x 68 floats for its
input is refused before any engine is created, so these checks need no GPU."""
import numpy as np
import pytest

FRAME = 480


@pytest.fixture
def no_engine(monkeypatch):
    from percepnet_b200 import api

    def refuse(*a, **k):
        raise AssertionError("an engine was created")
    monkeypatch.setattr(api, "Engine", refuse)
    monkeypatch.setattr(api, "BlobModel", refuse)


def _files(tmp_path, frames, gain_rows, extra_bytes=0):
    pin, gains = str(tmp_path / f"in{frames}.pcm"), str(tmp_path / f"g{frames}_{gain_rows}.f32")
    np.zeros(frames * FRAME + 100, "<i2").tofile(pin)   # a trailing partial frame is not a frame
    with open(gains, "wb") as f:
        f.write(np.zeros((gain_rows, 68), "<f4").tobytes() + b"\0" * extra_bytes)
    return pin, gains


@pytest.mark.parametrize("rows,extra", [(4, 0), (6, 0), (5, 4), (0, 0)], ids=["short", "long", "ragged", "empty"])
def test_gains_file_of_the_wrong_length_is_refused(tmp_path, capsys, no_engine, rows, extra):
    from percepnet_b200 import enhance
    pin, gains = _files(tmp_path, 5, rows, extra)
    out = tmp_path / "out.pcm"
    assert enhance.main(["--gains", gains, pin, str(out)]) == 2
    assert "5 frames" in capsys.readouterr().err
    assert not out.exists()


def test_list_mode_checks_every_gains_file_first(tmp_path, capsys, no_engine):
    """One bad gains file in a list stops the whole list before any job runs, the network jobs included."""
    from percepnet_b200 import enhance
    good_in, good_gains = _files(tmp_path, 3, 3)
    bad_in, bad_gains = _files(tmp_path, 7, 6)
    (tmp_path / "jobs.txt").write_text(f"{good_in} {tmp_path / 'a.pcm'} {good_gains}\n{good_in} {tmp_path / 'n.pcm'}\n"
                                       f"{bad_in} {tmp_path / 'b.pcm'} {bad_gains}\n")
    assert enhance.main(["--list", str(tmp_path / "jobs.txt"), "--seed", "0"]) == 2
    assert bad_gains in capsys.readouterr().err
    assert not any((tmp_path / n).exists() for n in ("a.pcm", "n.pcm", "b.pcm"))


def test_gains_is_single_file_only(tmp_path, no_engine):
    from percepnet_b200 import enhance
    pin, gains = _files(tmp_path, 2, 2)
    assert enhance.main(["--gains", gains, "--list", str(tmp_path / "jobs.txt")]) == 1
    assert enhance.main(["--gains", gains, "--gr", str(tmp_path / "gr.f32"), pin, str(tmp_path / "o.pcm")]) == 1
