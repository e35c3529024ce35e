"""Every refusal of the engine's entry points.  Each bad argument, alone and together with others where the order of the
checks decides which one is reported, gives a fixed return code and pnb_last_error() text, and every entry point of a
family refuses alike.  A refused call enqueues nothing and changes nothing: each engine's launch count stays, and its
next valid slot, session, ragged, training-record, training-audio and network call gives the bits of a twin engine that
saw no refusal.  So do the synthesis of an engine whose analysis was pending during the refusals and the call after it."""
import ctypes

import numpy as np
import pytest

from test_gpu_host_staging import _pairs
from test_gpu_lifecycle import HOP, _signal
from test_gpu_parity import api  # noqa: F401

pytestmark = pytest.mark.gpu

MODES = ["fp32", "tensor"]
S, FMAX, ACTIVE, CAP = 16, 4, 12, 24   # slots, max_frames, the slot engine's active range, the session pool
ROW = FMAX * HOP
SZ = 63804                             # pnb_state_size()
IDS = [3, 20, 0, 7, 11, 5]             # a valid session list (ids >= S: more sessions than slots)
HOPS = [4, 2, 4, 1, 3, 4]
SLOTS = [2, 0, 11]                     # a valid slot list, inside the active range
PEND = 3                               # hops of the analysis the pending engine waits to synthesise

SLOT = ["pnb_process_host_f32", "pnb_process_host_i16", "pnb_submit_host_f32", "pnb_submit_host_i16",
        "pnb_process_device_f32", "pnb_process_device_i16", "pnb_submit_device_f32", "pnb_submit_device_i16"]
SESSION = ["pnb_process_sessions_host_f32", "pnb_process_sessions_host_i16", "pnb_process_sessions_device_f32",
           "pnb_process_sessions_device_i16"]
RAGGED = ["pnb_process_sessions_ragged_host_f32", "pnb_process_sessions_ragged_host_i16",
          "pnb_process_sessions_ragged_device_f32", "pnb_process_sessions_ragged_device_i16"]
TRAIN = ["pnb_train_records_host", "pnb_submit_train_records", "pnb_train_records_device"]
AUDIO = ["pnb_train_audio_host", "pnb_train_audio_device"]
NETWORK = ["pnb_compute_rnn_host", "pnb_compute_rnn_device"]
SCORE = ["pnb_score_records_host", "pnb_score_records_device"]
STATES = ["pnb_reset_streams", "pnb_export_states", "pnb_import_states"]
ONE_STATE = ["pnb_get_state", "pnb_set_state"]
SESSION_STATES = ["pnb_reset_sessions", "pnb_export_sessions", "pnb_import_sessions"]

# family: (entry points, engine, valid arguments, {case: the arguments it changes}).  "e" names the engine: slot (an
# enhancement engine with active range ACTIVE), pend (one like it, with a synthesis pending), ses (one in session mode),
# trn (PNB_TRAIN_DATA), aud (PNB_TRAIN_DATA | PNB_TRAIN_AUDIO), net (PNB_NETWORK_ONLY), or None for NULL.
FAMILIES = {
    "slot": (SLOT, "slot", {"F": FMAX}, {
        "engine NULL": {"e": None},
        "training engine": {"e": "trn"},
        "F 0": {"F": 0},
        "F max+1": {"F": FMAX + 1},
        "in NULL": {"in": None},
        "out NULL": {"out": None},
        "in_stride short": {"in_stride": ROW - 1},
        "out_stride short": {"out_stride": ROW - 1},
        "session mode": {"e": "ses"},
        "network-only engine": {"e": "net"},
        "training engine, F 0": {"e": "trn", "F": 0},
        "F 0, in NULL": {"F": 0, "in": None},
        "out NULL, in_stride short": {"out": None, "in_stride": ROW - 1},
        "session mode, F max+1": {"e": "ses", "F": FMAX + 1},
        "session mode, out_stride short": {"e": "ses", "out_stride": ROW - 1},
    }),
    "session": (SESSION, "ses", {"F": FMAX, "ids": IDS}, {
        "engine NULL": {"e": None},
        "training engine": {"e": "trn"},
        "no pool": {"e": "slot"},
        "F 0": {"F": 0},
        "F max+1": {"F": FMAX + 1},
        "in NULL": {"in": None},
        "out NULL": {"out": None},
        "in_stride short": {"in_stride": ROW - 1},
        "out_stride short": {"out_stride": ROW - 1},
        "ids NULL": {"ids": None, "n": len(IDS)},
        "n 0": {"n": 0},
        "n slots+1": {"ids": list(range(S + 1))},
        "ids[i] -1": {"ids": [3, 20, -1, 7]},
        "ids[i] capacity": {"ids": [3, CAP, 0]},
        "ids listed twice": {"ids": [3, 20, 0, 20, 5]},
        "training engine, F 0": {"e": "trn", "F": 0},
        "no pool, F 0": {"e": "slot", "F": 0},
        "no pool, ids NULL": {"e": "slot", "ids": None, "n": len(IDS)},
        "F 0, ids NULL": {"F": 0, "ids": None, "n": len(IDS)},
        "ids listed twice, in NULL": {"ids": [3, 3], "in": None},
        "ids NULL, n 0": {"ids": None, "n": 0},
        "n slots+1, ids[i] capacity": {"ids": list(range(S)) + [CAP]},
        "ids listed twice, ids[i] capacity": {"ids": [3, 3, CAP]},
        "n 0, in_stride short": {"n": 0, "in_stride": ROW - 1},
    }),
    "ragged": (RAGGED, "ses", {"ids": IDS, "hops": HOPS}, {
        "engine NULL": {"e": None},
        "training engine": {"e": "trn"},
        "no pool": {"e": "slot"},
        "in NULL": {"in": None},
        "out NULL": {"out": None},
        "in_stride short": {"in_stride": ROW - 1},
        "out_stride short": {"out_stride": ROW - 1},
        "stride short for max(hops)": {"hops": [2, 1, 2, 2, 1, 2], "out_stride": 2 * HOP - 1},
        "ids NULL": {"ids": None, "n": len(IDS)},
        "n 0": {"n": 0},
        "n slots+1": {"ids": list(range(S + 1)), "hops": [1] * (S + 1)},
        "ids[i] -1": {"ids": [3, 20, -1, 7]},
        "ids[i] capacity": {"ids": [3, CAP, 0]},
        "ids listed twice": {"ids": [3, 20, 0, 20, 5]},
        "hops NULL": {"hops": None},
        "hops[i] 0": {"hops": [4, 2, 0, 1, 3, 4]},
        "hops[i] max+1": {"hops": [4, 2, 4, FMAX + 1, 3, 4]},
        "training engine, hops NULL": {"e": "trn", "hops": None},
        "no pool, ids NULL": {"e": "slot", "ids": None, "n": len(IDS)},
        "ids listed twice, hops NULL": {"ids": [3, 20, 3], "hops": None},
        "hops NULL, in NULL": {"hops": None, "in": None},
        "hops[i] max+1, then 0": {"ids": [3, 20, 0], "hops": [4, FMAX + 1, 0]},
        "hops[i] 0, in NULL": {"hops": [0, 2, 4, 1, 3, 4], "in": None},
        "in NULL, in_stride short": {"in": None, "in_stride": ROW - 1},
    }),
    "train": (TRAIN, "trn", {"F": FMAX}, {
        "engine NULL": {"e": None},
        "enhancement engine": {"e": "slot"},
        "session engine": {"e": "ses"},
        "audio engine": {"e": "aud"},
        "network-only engine": {"e": "net"},
        "F 0": {"F": 0},
        "F max+1": {"F": FMAX + 1},
        "speech NULL": {"speech": None},
        "noisy NULL": {"noisy": None},
        "records NULL": {"records": None},
        "speech_stride short": {"speech_stride": ROW - 1},
        "noisy_stride short": {"noisy_stride": ROW - 1},
        "records_stride short": {"records_stride": FMAX * 138 - 1},
        "enhancement engine, F 0": {"e": "slot", "F": 0},
        "F 0, speech NULL": {"F": 0, "speech": None},
        "records NULL, speech_stride short": {"records": None, "speech_stride": ROW - 1},
        "records_stride short, noisy_stride short": {"records_stride": FMAX * 138 - 1, "noisy_stride": ROW - 1},
        "audio engine, F 0": {"e": "aud", "F": 0},
    }),
    "audio": (AUDIO, "aud", {"F": FMAX}, {
        "engine NULL": {"e": None},
        "enhancement engine": {"e": "slot"},
        "records engine": {"e": "trn"},
        "F 0": {"F": 0},
        "F max+1": {"F": FMAX + 1},
        "speech NULL": {"speech": None},
        "noisy NULL": {"noisy": None},
        "records NULL": {"records": None},
        "audio NULL": {"audio": None},
        "speech_stride short": {"speech_stride": ROW - 1},
        "noisy_stride short": {"noisy_stride": ROW - 1},
        "records_stride short": {"records_stride": FMAX * 138 - 1},
        "audio_stride short": {"audio_stride": ROW - 1},
        "records engine, F 0": {"e": "trn", "F": 0},
        "records engine, records_stride short": {"e": "trn", "records_stride": FMAX * 138 - 1},
        "records_stride short, audio_stride short": {"records_stride": FMAX * 138 - 1, "audio_stride": ROW - 1},
    }),
    "network": (NETWORK, "net", {"F": FMAX, "in_stride": FMAX * 70}, {
        "training engine": {"e": "trn"},
        "F 0": {"F": 0},
        "in NULL": {"in": None},
        "gr NULL": {"gr": None},
        "in_stride short": {"in_stride": FMAX * 70 - 1},
        "in_stride short, records": {"format": 1, "in_stride": FMAX * 138 - 1},
        "gr_stride short": {"gr_stride": FMAX * 68 - 1},
        "format 2": {"format": 2},
        "session mode": {"e": "ses"},
        "format 2, in_stride short": {"format": 2, "in_stride": FMAX * 70 - 1},
        "session mode, format 2": {"e": "ses", "format": 2},
    }),
    "score": (SCORE, "net", {"F": FMAX}, {
        "sums NULL": {"sums": None},
        "rec_stride short": {"records_stride": FMAX * 138 - 1},
        "gr_stride short": {"gr_stride": FMAX * 68 - 1},
        "frames[i] -1": {"frames": [FMAX] * 5 + [-1] + [FMAX] * (S - 6)},
        "frames[i] F+1": {"frames": [FMAX] * 2 + [FMAX + 1] + [FMAX] * (S - 3)},
        "training engine": {"e": "trn"},
        "session mode": {"e": "ses"},
        "session mode, frames[i] -1": {"e": "ses", "frames": [FMAX] * 5 + [-1] + [FMAX] * (S - 6)},
    }),
    "states": (STATES, "slot", {"ids": SLOTS}, {
        "engine NULL": {"e": None},
        "session mode": {"e": "ses"},
        "n -1": {"n": -1},
        "streams NULL": {"ids": None, "n": len(SLOTS)},
        "blobs NULL": {"blobs": None},
        "blob_stride short": {"stride": SZ - 4},
        "blobs unaligned": {"blobs": 2},
        "blob_stride unaligned": {"stride": SZ + 2},
        "n slots+1": {"ids": list(range(S + 1))},
        "streams[i] -1": {"ids": [2, -1]},
        "streams[i] slots": {"ids": [2, S]},
        "streams[i] inactive": {"ids": [2, ACTIVE]},
        "streams listed twice": {"ids": [2, 0, 2]},
        "streams listed twice, then slots": {"ids": [2, 2, S]},
        "session mode, n -1": {"e": "ses", "n": -1},
        "n -1, streams NULL": {"n": -1, "ids": None},
        "streams NULL, blobs NULL": {"ids": None, "n": len(SLOTS), "blobs": None},
        "blobs NULL, streams listed twice": {"blobs": None, "ids": [2, 2]},
        "blob_stride short, n slots+1": {"stride": SZ - 4, "ids": list(range(S + 1))},
        "streams[i] inactive, then slots": {"ids": [2, ACTIVE, S]},
        "pending": {"e": "pend"},
        "pending, n -1": {"e": "pend", "n": -1},
        "pending, streams NULL": {"e": "pend", "ids": None, "n": len(SLOTS)},
        "pending, blobs NULL": {"e": "pend", "blobs": None},
        "pending, stream slots": {"e": "pend", "ids": [2, S]},
    }),
    "one state": (ONE_STATE, "slot", {"slot": 2}, {
        "engine NULL": {"e": None},
        "buffer NULL": {"buf": None},
        "session mode": {"e": "ses"},
        "stream -1": {"slot": -1},
        "stream slots": {"slot": S},
        "stream inactive": {"slot": ACTIVE},
        "bytes short": {"bytes": SZ - 1},
        "session mode, buffer NULL": {"e": "ses", "buf": None},
        "session mode, stream slots": {"e": "ses", "slot": S},
        "stream slots, bytes short": {"slot": S, "bytes": SZ - 1},
        "pending": {"e": "pend"},
        "pending, buffer NULL": {"e": "pend", "buf": None},
        "pending, stream slots": {"e": "pend", "slot": S},
        "pending, bytes short": {"e": "pend", "bytes": SZ - 1},
    }),
    "active": (["pnb_set_active_streams"], "slot", {"n": ACTIVE}, {
        "engine NULL": {"e": None},
        "training engine": {"e": "trn"},
        "session mode": {"e": "ses"},
        "n 0": {"n": 0},
        "n slots+1": {"n": S + 1},
        "training engine, n 0": {"e": "trn", "n": 0},
        "session mode, n 0": {"e": "ses", "n": 0},
        "pending": {"e": "pend"},
        "pending, n 0": {"e": "pend", "n": 0},
        "pending, n slots+1": {"e": "pend", "n": S + 1},
    }),
    "reserve": (["pnb_sessions_reserve"], "slot", {"n": CAP}, {
        "engine NULL": {"e": None},
        "training engine": {"e": "trn"},
        "n 0": {"n": 0},
        "training engine, n 0": {"e": "trn", "n": 0},
        "pending": {"e": "pend"},
        "pending, n 0": {"e": "pend", "n": 0},
    }),
    "session states": (SESSION_STATES, "ses", {"ids": IDS}, {
        "engine NULL": {"e": None},
        "no pool": {"e": "slot"},
        "no pool, n 0": {"e": "slot", "n": 0},
        "ids NULL": {"ids": None, "n": len(IDS)},
        "n -1": {"n": -1},
        "n capacity+1": {"ids": list(range(CAP + 1))},
        "ids[i] -1": {"ids": [3, -1]},
        "ids[i] capacity": {"ids": [3, CAP]},
        "ids listed twice": {"ids": [3, 20, 0, 20]},
        "blobs NULL": {"blobs": None},
        "blob_stride short": {"stride": SZ - 4},
        "blobs unaligned": {"blobs": 2},
        "blob_stride unaligned": {"stride": SZ + 2},
        "no pool, blobs NULL": {"e": "slot", "blobs": None},
        "blobs NULL, ids NULL": {"blobs": None, "ids": None, "n": len(IDS)},
        "ids NULL, n -1": {"ids": None, "n": -1},
        "ids listed twice, ids[i] capacity": {"ids": [20, 20, CAP]},
    }),
}
BLOB_CASE_KEYS = ("blobs", "stride")   # arguments pnb_reset_streams / pnb_reset_sessions do not take

SESSION_MODE = "engine is in session mode (pnb_sessions_reserve): slots are the pool's; use the *_sessions entry points"
TRAINING_ENGINE = "engine was created with PNB_TRAIN_DATA: use pnb_train_records_* / pnb_submit_train_records"
NO_POOL = "no session pool: call pnb_sessions_reserve first"
NETWORK_ENGINE = "engine was created with PNB_NETWORK_ONLY: use pnb_compute_rnn_* / pnb_score_records_*"
AUDIO_ENGINE = "engine was created with PNB_TRAIN_AUDIO: use pnb_train_audio_*, so that its audio has no gaps"
NOT_AUDIO = "engine was not created with PNB_TRAIN_AUDIO"
STRIDE = "row stride smaller than n_frames*480"
PENDING = (f"a synthesis is pending (pnb_analyze_* of {PEND} hops): call pnb_synthesize_* with the same n_frames, "
           "or pnb_reset")
# (family, case): (return code, pnb_last_error()); -1 is PNB_ERR_ARG.
EXPECTED = {
    ("slot", "engine NULL"): (-1, "engine is NULL"),
    ("slot", "training engine"): (-1, TRAINING_ENGINE),
    ("slot", "F 0"): (-1, "n_frames 0 outside [1, 4]"),
    ("slot", "F max+1"): (-1, "n_frames 5 outside [1, 4]"),
    ("slot", "in NULL"): (-1, "input/output pointer is NULL"),
    ("slot", "out NULL"): (-1, "input/output pointer is NULL"),
    ("slot", "in_stride short"): (-1, STRIDE),
    ("slot", "out_stride short"): (-1, STRIDE),
    ("slot", "session mode"): (-1, SESSION_MODE),
    ("slot", "network-only engine"): (-1, NETWORK_ENGINE),
    ("slot", "training engine, F 0"): (-1, TRAINING_ENGINE),
    ("slot", "F 0, in NULL"): (-1, "n_frames 0 outside [1, 4]"),
    ("slot", "out NULL, in_stride short"): (-1, "input/output pointer is NULL"),
    ("slot", "session mode, F max+1"): (-1, "n_frames 5 outside [1, 4]"),
    ("slot", "session mode, out_stride short"): (-1, STRIDE),
    ("session", "engine NULL"): (-1, "engine is NULL"),
    ("session", "training engine"): (-1, TRAINING_ENGINE),
    ("session", "no pool"): (-1, NO_POOL),
    ("session", "F 0"): (-1, "n_frames 0 outside [1, 4]"),
    ("session", "F max+1"): (-1, "n_frames 5 outside [1, 4]"),
    ("session", "in NULL"): (-1, "input/output pointer is NULL"),
    ("session", "out NULL"): (-1, "input/output pointer is NULL"),
    ("session", "in_stride short"): (-1, STRIDE),
    ("session", "out_stride short"): (-1, STRIDE),
    ("session", "ids NULL"): (-1, "ids is NULL"),
    ("session", "n 0"): (-1, "n = 0 sessions outside [1, 16]"),
    ("session", "n slots+1"): (-1, "n = 17 sessions outside [1, 16]"),
    ("session", "ids[i] -1"): (-1, "ids[2] = -1 outside [0, 24)"),
    ("session", "ids[i] capacity"): (-1, "ids[1] = 24 outside [0, 24)"),
    ("session", "ids listed twice"): (-1, "ids[3] = 20 listed twice"),
    ("session", "training engine, F 0"): (-1, TRAINING_ENGINE),
    ("session", "no pool, F 0"): (-1, "n_frames 0 outside [1, 4]"),
    ("session", "no pool, ids NULL"): (-1, NO_POOL),
    ("session", "F 0, ids NULL"): (-1, "n_frames 0 outside [1, 4]"),
    ("session", "ids listed twice, in NULL"): (-1, "input/output pointer is NULL"),
    ("session", "ids NULL, n 0"): (-1, "ids is NULL"),
    ("session", "n slots+1, ids[i] capacity"): (-1, "n = 17 sessions outside [1, 16]"),
    ("session", "ids listed twice, ids[i] capacity"): (-1, "ids[2] = 24 outside [0, 24)"),
    ("session", "n 0, in_stride short"): (-1, STRIDE),
    ("ragged", "engine NULL"): (-1, "engine is NULL"),
    ("ragged", "training engine"): (-1, NO_POOL),
    ("ragged", "no pool"): (-1, NO_POOL),
    ("ragged", "in NULL"): (-1, "input/output pointer is NULL"),
    ("ragged", "out NULL"): (-1, "input/output pointer is NULL"),
    ("ragged", "in_stride short"): (-1, STRIDE),
    ("ragged", "out_stride short"): (-1, STRIDE),
    ("ragged", "stride short for max(hops)"): (-1, STRIDE),
    ("ragged", "ids NULL"): (-1, "ids is NULL"),
    ("ragged", "n 0"): (-1, "n = 0 sessions outside [1, 16]"),
    ("ragged", "n slots+1"): (-1, "n = 17 sessions outside [1, 16]"),
    ("ragged", "ids[i] -1"): (-1, "ids[2] = -1 outside [0, 24)"),
    ("ragged", "ids[i] capacity"): (-1, "ids[1] = 24 outside [0, 24)"),
    ("ragged", "ids listed twice"): (-1, "ids[3] = 20 listed twice"),
    ("ragged", "hops NULL"): (-1, "hops is NULL"),
    ("ragged", "hops[i] 0"): (-1, "hops[2] = 0 outside [1, 4]"),
    ("ragged", "hops[i] max+1"): (-1, "hops[3] = 5 outside [1, 4]"),
    ("ragged", "training engine, hops NULL"): (-1, NO_POOL),
    ("ragged", "no pool, ids NULL"): (-1, NO_POOL),
    ("ragged", "ids listed twice, hops NULL"): (-1, "ids[2] = 3 listed twice"),
    ("ragged", "hops NULL, in NULL"): (-1, "hops is NULL"),
    ("ragged", "hops[i] max+1, then 0"): (-1, "hops[1] = 5 outside [1, 4]"),
    ("ragged", "hops[i] 0, in NULL"): (-1, "hops[0] = 0 outside [1, 4]"),
    ("ragged", "in NULL, in_stride short"): (-1, "input/output pointer is NULL"),
    ("train", "engine NULL"): (-1, "engine is NULL"),
    ("train", "enhancement engine"): (-1, "engine was not created with PNB_TRAIN_DATA"),
    ("train", "session engine"): (-1, "engine was not created with PNB_TRAIN_DATA"),
    ("train", "audio engine"): (-1, AUDIO_ENGINE),
    ("train", "network-only engine"): (-1, NETWORK_ENGINE),
    ("train", "F 0"): (-1, "n_frames 0 outside [1, 4]"),
    ("train", "F max+1"): (-1, "n_frames 5 outside [1, 4]"),
    ("train", "speech NULL"): (-1, "speech/noisy/records pointer is NULL"),
    ("train", "noisy NULL"): (-1, "speech/noisy/records pointer is NULL"),
    ("train", "records NULL"): (-1, "speech/noisy/records pointer is NULL"),
    ("train", "speech_stride short"): (-1, STRIDE),
    ("train", "noisy_stride short"): (-1, STRIDE),
    ("train", "records_stride short"): (-1, "records_stride smaller than n_frames*138"),
    ("train", "enhancement engine, F 0"): (-1, "engine was not created with PNB_TRAIN_DATA"),
    ("train", "F 0, speech NULL"): (-1, "n_frames 0 outside [1, 4]"),
    ("train", "records NULL, speech_stride short"): (-1, "speech/noisy/records pointer is NULL"),
    ("train", "records_stride short, noisy_stride short"): (-1, STRIDE),
    ("train", "audio engine, F 0"): (-1, "n_frames 0 outside [1, 4]"),
    ("audio", "engine NULL"): (-1, "engine is NULL"),
    ("audio", "enhancement engine"): (-1, "engine was not created with PNB_TRAIN_DATA"),
    ("audio", "records engine"): (-1, NOT_AUDIO),
    ("audio", "F 0"): (-1, "n_frames 0 outside [1, 4]"),
    ("audio", "F max+1"): (-1, "n_frames 5 outside [1, 4]"),
    ("audio", "speech NULL"): (-1, "speech/noisy/records pointer is NULL"),
    ("audio", "noisy NULL"): (-1, "speech/noisy/records pointer is NULL"),
    ("audio", "records NULL"): (-1, "speech/noisy/records pointer is NULL"),
    ("audio", "audio NULL"): (-1, "speech/noisy/records pointer is NULL"),
    ("audio", "speech_stride short"): (-1, STRIDE),
    ("audio", "noisy_stride short"): (-1, STRIDE),
    ("audio", "records_stride short"): (-1, "records_stride smaller than n_frames*138"),
    ("audio", "audio_stride short"): (-1, "audio_stride smaller than n_frames*480"),
    ("audio", "records engine, F 0"): (-1, "n_frames 0 outside [1, 4]"),
    ("audio", "records engine, records_stride short"): (-1, NOT_AUDIO),
    ("audio", "records_stride short, audio_stride short"): (-1, "records_stride smaller than n_frames*138"),
    ("network", "training engine"): (-1, TRAINING_ENGINE),
    ("network", "F 0"): (-1, "n_frames 0 outside [1, 4]"),
    ("network", "in NULL"): (-1, "input/output pointer is NULL"),
    ("network", "gr NULL"): (-1, "input/output pointer is NULL"),
    ("network", "in_stride short"): (-1, "row stride smaller than n_frames*70"),
    ("network", "in_stride short, records"): (-1, "row stride smaller than n_frames*138"),
    ("network", "gr_stride short"): (-1, "row stride smaller than n_frames*68"),
    ("network", "format 2"): (-1, "format 2 is neither PNB_RNN_FEATURES (0) nor PNB_RNN_RECORDS (1)"),
    ("network", "session mode"): (-1, SESSION_MODE),
    ("network", "format 2, in_stride short"): (-1, "row stride smaller than n_frames*70"),
    ("network", "session mode, format 2"): (-1, "format 2 is neither PNB_RNN_FEATURES (0) nor PNB_RNN_RECORDS (1)"),
    ("score", "sums NULL"): (-1, "input/output pointer is NULL"),
    ("score", "rec_stride short"): (-1, "row stride smaller than n_frames*138"),
    ("score", "gr_stride short"): (-1, "row stride smaller than n_frames*68"),
    ("score", "frames[i] -1"): (-1, "frames[5] = -1 outside [0, 4]"),
    ("score", "frames[i] F+1"): (-1, "frames[2] = 5 outside [0, 4]"),
    ("score", "training engine"): (-1, TRAINING_ENGINE),
    ("score", "session mode"): (-1, SESSION_MODE),
    ("score", "session mode, frames[i] -1"): (-1, SESSION_MODE),
    ("states", "engine NULL"): (-1, "engine is NULL"),
    ("states", "session mode"): (-1, SESSION_MODE),
    ("states", "n -1"): (-1, "n = -1 is negative"),
    ("states", "streams NULL"): (-1, "streams is NULL"),
    ("states", "blobs NULL"): (-1, "d_blobs is NULL"),
    ("states", "blob_stride short"): (-1, "blob_stride 63800 below pnb_state_size() = 63804"),
    ("states", "blobs unaligned"): (-1, "d_blobs and blob_stride must be multiples of 4 bytes"),
    ("states", "blob_stride unaligned"): (-1, "d_blobs and blob_stride must be multiples of 4 bytes"),
    ("states", "n slots+1"): (-1, "n = 17 streams, the engine has 16"),
    ("states", "streams[i] -1"): (-1, "streams[1] = -1 outside [0, 16)"),
    ("states", "streams[i] slots"): (-1, "streams[1] = 16 outside [0, 16)"),
    ("states", "streams[i] inactive"): (-1, "streams[1] = 12 outside the active range [0, 12)"),
    ("states", "streams listed twice"): (-1, "streams[2] = 2 listed twice"),
    ("states", "streams listed twice, then slots"): (-1, "streams[2] = 16 outside [0, 16)"),
    ("states", "session mode, n -1"): (-1, SESSION_MODE),
    ("states", "n -1, streams NULL"): (-1, "n = -1 is negative"),
    ("states", "streams NULL, blobs NULL"): (-1, "streams is NULL"),
    ("states", "blobs NULL, streams listed twice"): (-1, "d_blobs is NULL"),
    ("states", "blob_stride short, n slots+1"): (-1, "blob_stride 63800 below pnb_state_size() = 63804"),
    ("states", "streams[i] inactive, then slots"): (-1, "streams[1] = 12 outside the active range [0, 12)"),
    ("states", "pending"): (-1, PENDING),
    ("states", "pending, n -1"): (-1, PENDING),
    ("states", "pending, streams NULL"): (-1, PENDING),
    ("states", "pending, blobs NULL"): (-1, PENDING),
    ("states", "pending, stream slots"): (-1, PENDING),
    ("one state", "engine NULL"): (-1, "NULL argument"),
    ("one state", "buffer NULL"): (-1, "NULL argument"),
    ("one state", "session mode"): (-1, SESSION_MODE),
    ("one state", "stream -1"): (-1, "stream[0] = -1 outside [0, 16)"),
    ("one state", "stream slots"): (-1, "stream[0] = 16 outside [0, 16)"),
    ("one state", "stream inactive"): (-1, "stream[0] = 12 outside the active range [0, 12)"),
    ("one state", "bytes short"): (-1, "state buffer of 63803 bytes, need pnb_state_size() = 63804"),
    ("one state", "session mode, buffer NULL"): (-1, "NULL argument"),
    ("one state", "session mode, stream slots"): (-1, SESSION_MODE),
    ("one state", "stream slots, bytes short"): (-1, "stream[0] = 16 outside [0, 16)"),
    ("one state", "pending"): (-1, PENDING),
    ("one state", "pending, buffer NULL"): (-1, "NULL argument"),
    ("one state", "pending, stream slots"): (-1, PENDING),
    ("one state", "pending, bytes short"): (-1, PENDING),
    ("active", "engine NULL"): (-1, "engine is NULL"),
    ("active", "training engine"): (-1, "PNB_TRAIN_DATA engines always advance all their streams"),
    ("active", "session mode"): (-1, SESSION_MODE),
    ("active", "n 0"): (-1, "active streams 0 outside [1, 16]"),
    ("active", "n slots+1"): (-1, "active streams 17 outside [1, 16]"),
    ("active", "training engine, n 0"): (-1, "PNB_TRAIN_DATA engines always advance all their streams"),
    ("active", "session mode, n 0"): (-1, SESSION_MODE),
    ("active", "pending"): (-1, PENDING),
    ("active", "pending, n 0"): (-1, PENDING),
    ("active", "pending, n slots+1"): (-1, PENDING),
    ("reserve", "engine NULL"): (-1, "engine is NULL"),
    ("reserve", "training engine"): (-1, "PNB_TRAIN_DATA engines have no session pool"),
    ("reserve", "n 0"): (-1, "n_sessions = 0, need >= 1"),
    ("reserve", "training engine, n 0"): (-1, "PNB_TRAIN_DATA engines have no session pool"),
    ("reserve", "pending"): (-1, PENDING),
    ("reserve", "pending, n 0"): (-1, PENDING),
    ("session states", "engine NULL"): (-1, "engine is NULL"),
    ("session states", "no pool"): (-1, NO_POOL),
    ("session states", "no pool, n 0"): (-1, NO_POOL),
    ("session states", "ids NULL"): (-1, "ids is NULL"),
    ("session states", "n -1"): (-1, "n = -1 sessions outside [1, 24]"),
    ("session states", "n capacity+1"): (-1, "n = 25 sessions outside [1, 24]"),
    ("session states", "ids[i] -1"): (-1, "ids[1] = -1 outside [0, 24)"),
    ("session states", "ids[i] capacity"): (-1, "ids[1] = 24 outside [0, 24)"),
    ("session states", "ids listed twice"): (-1, "ids[3] = 20 listed twice"),
    ("session states", "blobs NULL"): (-1, "d_blobs is NULL"),
    ("session states", "blob_stride short"): (-1, "blob_stride 63800 below pnb_state_size() = 63804"),
    ("session states", "blobs unaligned"): (-1, "d_blobs and blob_stride must be multiples of 4 bytes"),
    ("session states", "blob_stride unaligned"): (-1, "d_blobs and blob_stride must be multiples of 4 bytes"),
    ("session states", "no pool, blobs NULL"): (-1, "d_blobs is NULL"),
    ("session states", "blobs NULL, ids NULL"): (-1, "d_blobs is NULL"),
    ("session states", "ids NULL, n -1"): (-1, "ids is NULL"),
    ("session states", "ids listed twice, ids[i] capacity"): (-1, "ids[2] = 24 outside [0, 24)"),
    ("one state", "set_state: not a blob"): (-1, "not a pnb_get_state blob (magic/version)"),
}


def _ints(v, keep):
    if v is None:
        return None
    a = np.ascontiguousarray(np.asarray(v, np.int32))
    keep.append(a)
    return a.ctypes.data


def _call(L, name, a, keep):
    """Entry point `name` with the argument set a (engine handle, host or device buffers, lists as Python lists)."""
    f = getattr(L, name)
    ids = _ints(a.get("ids"), keep)
    n = a["n"] if "n" in a else len(a.get("ids") or [])
    if name in SLOT + SESSION + RAGGED:
        head = [a["e"]]
        if name in RAGGED:
            head += [ids, _ints(a.get("hops"), keep), n]
        elif name in SESSION:
            head += [ids, n]
        args = head + [a["in"], a["in_stride"], a["out"], a["out_stride"]]
        args += [] if name in RAGGED else [a["F"]]
        args += [] if name.startswith("pnb_submit") else [None]
        args += [a["stream"]] if "device" in name else []
        return f(*args)
    tail = [a["stream"]] if name.endswith("device") else []
    if name in TRAIN + AUDIO:
        args = [a["e"], a["speech"], a["speech_stride"], a["noisy"], a["noisy_stride"], a["F"], a["records"],
                a["records_stride"]]
        args += [a["audio"], a["audio_stride"]] if name in AUDIO else []
        return f(*args, *tail)
    if name in NETWORK:
        return f(a["e"], a["format"], a["in"], a["in_stride"], a["F"], a["gr"], a["gr_stride"], *tail)
    if name in SCORE:
        return f(a["e"], a["records"], a["records_stride"], a["F"], _ints(a.get("frames"), keep), a["sums"], a["gr"],
                 a["gr_stride"], *tail)
    if name in STATES + SESSION_STATES:
        if "reset" in name:
            return f(a["e"], ids, n, a["stream"])
        return f(a["e"], ids, n, a["blobs"], a["stride"], a["stream"])
    if name in ONE_STATE:
        return f(a["e"], a["slot"], a["buf"], a["bytes"])
    if name == "pnb_set_active_streams":
        return f(a["e"], a["n"], a["stream"])
    return f(a["e"], a["n"])


class _Buffers:
    """Host and device buffers big enough for every valid call of the table."""

    def __init__(self):
        import torch
        self.h32, self.h16 = np.zeros((S, ROW), np.float32), np.zeros((S, ROW), np.int16)
        self.d32 = torch.zeros((2, S, ROW), dtype=torch.float32, device="cuda")
        self.d16 = torch.zeros((2, S, ROW), dtype=torch.int16, device="cuda")
        self.hsp, self.hrec = np.zeros((S // 2, ROW), np.int16), np.zeros((S, FMAX * 138), np.float32)
        self.dsp = torch.zeros((3, S // 2, ROW), dtype=torch.int16, device="cuda")
        self.drec = torch.zeros((S, FMAX * 138), device="cuda")
        self.hsums, self.dsums = np.zeros((S, 4)), torch.zeros((S, 4), dtype=torch.float64, device="cuda")
        self.blobs = torch.zeros(((CAP + 1) * (SZ + 4),), dtype=torch.uint8, device="cuda")
        self.state = ctypes.create_string_buffer(SZ)   # zeros: not a pnb_get_state blob
        self.stream = torch.cuda.current_stream().cuda_stream

    def valid(self, name):
        """The arguments of a valid call of `name`, buffers only."""
        a = {"stream": self.stream, "blobs": self.blobs.data_ptr(), "stride": SZ, "buf": self.state, "bytes": SZ}
        if "host" in name or "submit_host" in name or name == "pnb_submit_train_records":
            h = self.h16 if name.endswith("i16") else self.h32
            a.update({"in": h.ctypes.data, "out": h.ctypes.data, "gr": h.ctypes.data, "speech": self.hsp.ctypes.data,
                      "noisy": self.hsp.ctypes.data, "records": self.hrec.ctypes.data, "audio": self.hsp.ctypes.data,
                      "sums": self.hsums.ctypes.data})
        else:
            d = self.d16 if name.endswith("i16") else self.d32
            a.update({"in": d[0].data_ptr(), "out": d[1].data_ptr(), "gr": d[1].data_ptr(),
                      "speech": self.dsp[0].data_ptr(), "noisy": self.dsp[1].data_ptr(), "records": self.drec.data_ptr(),
                      "audio": self.dsp[2].data_ptr(), "sums": self.dsums.data_ptr()})
        a.update({"in_stride": ROW, "out_stride": ROW, "speech_stride": ROW, "noisy_stride": ROW,
                  "records_stride": FMAX * 138, "audio_stride": ROW, "gr_stride": FMAX * 68, "format": 0})
        return a


def _refusals(L, engines, bufs):
    """{(family, case): (rc, message)} of every entry point of every family; raises if two entry points of one family
    answer a case differently."""
    got = {}
    for fam, (names, eng, valid, cases) in FAMILIES.items():
        for case, change in cases.items():
            for name in names:
                if "reset" in name and any(k in change for k in BLOB_CASE_KEYS):
                    continue
                a = {**bufs.valid(name), **valid, "e": eng, **change}
                if "blobs" in change and change["blobs"] is not None:
                    a["blobs"] = bufs.blobs.data_ptr() + change["blobs"]
                a["e"] = None if a["e"] is None else engines[a["e"]].h
                keep = []
                rc = _call(L, name, a, keep)
                r = (rc, L.pnb_last_error().decode())
                prev = got.setdefault((fam, case), r)
                assert prev == r, (fam, case, name, prev, r)
    # the magic check of pnb_set_state: the only host-side blob check
    a = {**bufs.valid("pnb_set_state"), "slot": 2, "e": engines["slot"].h}
    rc = _call(L, "pnb_set_state", a, [])
    got[("one state", "set_state: not a blob")] = (rc, L.pnb_last_error().decode())
    return got


def _engines(api, model, mode):
    flags = api.NN_FP32 if mode == "fp32" else api.NN_TENSOR
    slot, pend, ses = (api.Engine(S, FMAX, model, flags) for _ in range(3))
    slot.set_active(ACTIVE)
    pend.set_active(ACTIVE)
    ses.reserve_sessions(CAP)
    return {"slot": slot, "pend": pend, "ses": ses, "trn": api.Engine(S, FMAX, None, api.TRAIN_DATA),
            "aud": api.Engine(S, FMAX, None, api.TRAIN_DATA | api.TRAIN_AUDIO),
            "net": api.Engine(S, FMAX, model, flags | api.NETWORK_ONLY)}


@pytest.mark.parametrize("mode", MODES)
def test_refusals(api, model0, mode):
    """Every case of FAMILIES gives its EXPECTED code and text on every entry point of its family, enqueues nothing, and
    leaves each engine to continue like its twin."""
    import torch
    x = _signal(S, 2, 43)
    speech, noisy = _pairs(S // 2, 2 * FMAX, 7)
    rec = np.random.RandomState(44).rand(S, 2 * FMAX, 138).astype(np.float32)   # labels in [0, 1)
    engines, twins = _engines(api, model0, mode), _engines(api, model0, mode)
    for es in (engines, twins):   # one valid call of each kind before the refusals
        es["slot"].process(np.ascontiguousarray(x[:ACTIVE, :ROW]))
        es["pend"].process(np.ascontiguousarray(x[:ACTIVE, :ROW]))
        es["pend"].analyze(np.ascontiguousarray(x[:ACTIVE, ROW:ROW + PEND * HOP]))
        es["ses"].process_sessions(IDS, np.ascontiguousarray(x[:len(IDS), :ROW]))
        es["trn"].train_records(np.ascontiguousarray(speech[:, :ROW]), np.ascontiguousarray(noisy[:, :ROW]))
        es["aud"].train_audio(np.ascontiguousarray(speech[:, :ROW]), np.ascontiguousarray(noisy[:, :ROW]))
        es["net"].compute_rnn(np.ascontiguousarray(rec[:, :FMAX, :70]))
    bufs = _Buffers()
    torch.cuda.synchronize()
    launches = {k: e.launches for k, e in engines.items()}

    got = _refusals(engines["slot"].L, engines, bufs)
    torch.cuda.synchronize()
    assert {k: e.launches for k, e in engines.items()} == launches
    assert set(got) == set(EXPECTED)
    for key, want in EXPECTED.items():
        assert got[key] == want, key

    nxt = np.ascontiguousarray(x[:, ROW:2 * ROW])
    (a, ga), (b, gb) = (es["slot"].process(nxt[:ACTIVE], want_gr=True) for es in (engines, twins))
    assert np.array_equal(a, b) and np.array_equal(ga, gb) and np.abs(a).max() > 0
    gr = np.random.RandomState(45).rand(ACTIVE, PEND, 68).astype(np.float32)
    a, b = (es["pend"].synthesize(gr) for es in (engines, twins))
    assert np.array_equal(a, b) and np.abs(a).max() > 0
    after = np.ascontiguousarray(x[:ACTIVE, ROW + PEND * HOP:2 * ROW + PEND * HOP])
    (a, ga), (b, gb) = (es["pend"].process(after, want_gr=True) for es in (engines, twins))
    assert np.array_equal(a, b) and np.array_equal(ga, gb) and np.abs(a).max() > 0
    ids = [5, 20, 9, 3]                 # three resident, one fresh
    (a, ga), (b, gb) = (es["ses"].process_sessions(ids, nxt[:4, :2 * HOP], want_gr=True) for es in (engines, twins))
    assert np.array_equal(a, b) and np.array_equal(ga, gb) and np.abs(a).max() > 0
    ids, hops = [0, 9, 11, 20], [1, 4, 2, 4]   # two parked by the last call, two resident
    (a, ga), (b, gb) = (es["ses"].process_sessions(ids, nxt[4:8], want_gr=True, hops=hops) for es in (engines, twins))
    assert np.array_equal(a, b) and np.array_equal(ga, gb) and np.abs(a).max() > 0
    s, y = np.ascontiguousarray(speech[:, ROW:]), np.ascontiguousarray(noisy[:, ROW:])
    ra, rb = (es["trn"].train_records(s, y) for es in (engines, twins))
    assert np.array_equal(ra.view(np.int32), rb.view(np.int32))
    (ra, aa), (rb, ab) = (es["aud"].train_audio(s, y) for es in (engines, twins))
    assert np.array_equal(ra.view(np.int32), rb.view(np.int32)) and np.array_equal(aa, ab) and np.abs(aa).max() > 0
    (sa, ga), (sb, gb) = (es["net"].score_records(rec[:, FMAX:], want_gr=True) for es in (engines, twins))
    assert np.array_equal(sa, sb) and np.array_equal(ga, gb) and np.abs(ga).max() > 0
    for es in (engines, twins):
        for e in es.values():
            e.check()
            e.close()
