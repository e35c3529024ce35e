import hashlib

import numpy as np


def digest(*arrays):
    """SHA-256 over the shapes and bits of the arrays (floats as float32 with -0 folded into +0, integers as int64):
    equal digests <=> same_bits / array_equal on every array."""
    h = hashlib.sha256()
    for a in arrays:
        a = np.asarray(a)
        if a.dtype.kind == "f":
            a = np.ascontiguousarray(a, np.float32)
            a = np.where(a == 0, np.float32(0), a)
        else:
            a = np.ascontiguousarray(a, np.int64)
        h.update(repr(a.shape).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def first_hop_major(sm):
    """Fewest active streams whose GRU chain walks its units in hop-major order on a device with `sm` SMs.
    tc_gru_chain (pnb_nn_tc.cu) picks anti-diagonal order while ceil(n / 128) * (512 / 64) < sm, so the first
    hop-major size starts the row tile that brings the count to ceil(sm / 8) (132 SMs: 2 049, 114 SMs: 1 793)."""
    return 128 * (-(-sm // 8) - 1) + 1


def device_first_hop_major():
    """first_hop_major of cuda:0."""
    import torch
    return first_hop_major(torch.cuda.get_device_properties(0).multi_processor_count)


def crowd(n_streams, n_frames, seed, n_base=32):
    """[n_streams, n_frames*480] float32 of distinct rows made cheaply: n_base synthetic streams, each row one of them
    at its own level and shifted by its own whole number of hops."""
    from percepnet_b200.synth import synth_pcm
    base = synth_pcm(n_base, n_frames, seed=seed)
    rng = np.random.RandomState(seed)
    rows = rng.randint(0, n_base, n_streams)
    level = (0.25 + rng.rand(n_streams)).astype(np.float32)
    shift = rng.randint(0, n_frames, n_streams) * 480
    out = np.empty((n_streams, base.shape[1]), np.float32)
    for i in range(n_streams):
        out[i] = np.roll(base[rows[i]], shift[i]) * level[i]
    return out


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def same_bits(a, b):
    """float arrays equal bit for bit (distinguishes nothing but +-0, which compare equal by value)."""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((bits(a) == bits(b)) | ((a == 0) & (b == 0))))


def edge_signals(n_frames=24, scale=1.0):
    """Edge-case single-stream inputs the reference never tests itself (SURVEY.md 8c(3))."""
    T = n_frames * 480
    t = np.arange(T) / 48000.0
    rng = np.random.RandomState(11)
    sig = {}
    sig["zeros"] = np.zeros(T, np.float32)
    imp = np.zeros(T, np.float32); imp[2000] = 0.9
    sig["impulse"] = imp
    sig["sine62"] = (0.8 * np.sin(2 * np.pi * 62.5 * t)).astype(np.float32)    # period 768 = PITCH_MAX_PERIOD
    sig["sine800"] = (0.8 * np.sin(2 * np.pi * 800.0 * t)).astype(np.float32)   # period 60  = PITCH_MIN_PERIOD
    h = np.zeros(T)
    for k, a in ((1, 0.3), (2, 1.0), (3, 0.2), (4, 0.8), (6, 0.5)):            # octave-ambiguous stack (doubling logic)
        h += a * np.sin(2 * np.pi * 110.0 * k * t + 0.3 * k)
    sig["octave"] = (0.25 * h / np.abs(h).max()).astype(np.float32)
    sig["noise"] = (0.1 * rng.randn(T)).astype(np.float32)
    sig["fullscale_sq"] = np.sign(np.sin(2 * np.pi * 150.0 * t)).astype(np.float32) * 0.999
    sw = np.sin(2 * np.pi * (80.0 * t + 160.0 * t * t))                        # chirp 80 -> 400 Hz/s
    sig["chirp"] = (0.5 * sw).astype(np.float32)
    return {k: (v * np.float32(scale)).astype(np.float32) for k, v in sig.items()}


def random_mixtures(n_streams, n_frames, seed=2025, max_log_amp=0.0):
    """Seeded random streams: harmonic stacks + noise + DC + exact-silence gaps + clicks at log-uniform amplitudes
    in [1e-4, 10**max_log_amp] (the same family the CPU property test draws from)."""
    T = n_frames * 480
    t = np.arange(T) / 48000.0
    out = np.empty((n_streams, T), np.float32)
    for s in range(n_streams):
        rng = np.random.RandomState(seed + s)
        f0, noise, dc = 55.0 + 845.0 * rng.rand(), rng.rand(), 0.4 * rng.rand() - 0.2
        x = np.zeros(T)
        for h in range(1, 9):
            x += rng.rand() * np.sin(2 * np.pi * f0 * h * t + rng.rand() * 6.28) / h
        x = x / (np.abs(x).max() + 1e-9) * (1 - noise) + noise * rng.randn(T) * 0.3 + dc
        gap = rng.randint(0, 9)
        if gap:
            g0 = rng.randint(0, n_frames - gap + 1) * 480
            x[g0:g0 + gap * 480] = 0.0
        if rng.rand() < 0.5:
            x[rng.randint(0, T)] += 3.0
        out[s] = (x * 10.0 ** (-4.0 + (4.0 + max_log_amp) * rng.rand())).astype(np.float32)
    return out
