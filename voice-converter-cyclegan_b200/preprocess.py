"""Feature-side helpers of the reference's `preprocess.py` that sit directly either side of the hot path (SURVEY.md 8f).

The numpy functions here keep the reference's names (including its spelling) and argument meaning so `train.py` /
`convert.py` callers can switch imports:

  coded_sps_normalization_fit_transoform / _transoform / _inverse_transoform   preprocess.py:106-133
  coded_sp_padding, wav_padding                                                preprocess.py:135-158
  logf0_statistics, pitch_conversion                                           preprocess.py:161-175
  transpose_in_list                                                            preprocess.py:63-68
  sample_train_data                                                            preprocess.py:207-238
  counter_sample_plan, sample_train_data_counter                               the same contract, host twin of the device sampler

WORLD analysis / synthesis (`world_decompose`, `world_encode_spectral_envelop`, ... preprocess.py:6-104) is CPU audio
code in pyworld + librosa and is NOT rebuilt: the wrappers below forward to pyworld when it is importable and raise a
clear ImportError otherwise (neither package exists in this image).
"""
from __future__ import annotations

import numpy as np


# --------------------------------------------------------------------------------------------- WORLD (gated on pyworld)
def _pyworld():
    try:
        import pyworld
        return pyworld
    except ImportError as e:                                   # pragma: no cover - pyworld is absent in this image
        raise ImportError("WORLD analysis/synthesis needs the `pyworld` package (CPU audio code, outside the GPU hot path); "
                          "feed pre-extracted MCEP matrices instead (see cgvc.convert / cgvc.train)") from e


def world_decompose(wav, fs, frame_period=5.0):
    """f0 (harvest, 71..800 Hz), time axis, spectral envelope (cheaptrick), aperiodicity (d4c) -- preprocess.py:17-25."""
    pw = _pyworld()
    wav = np.asarray(wav, dtype=np.float64)
    f0, timeaxis = pw.harvest(wav, fs, frame_period=frame_period, f0_floor=71.0, f0_ceil=800.0)
    return f0, timeaxis, pw.cheaptrick(wav, f0, timeaxis, fs), pw.d4c(wav, f0, timeaxis, fs)


def world_encode_spectral_envelop(sp, fs, dim=24):
    return _pyworld().code_spectral_envelope(sp, fs, dim)


def world_decode_spectral_envelop(coded_sp, fs):
    pw = _pyworld()
    return pw.decode_spectral_envelope(coded_sp, fs, pw.get_cheaptrick_fft_size(fs))


def world_speech_synthesis(f0, decoded_sp, ap, fs, frame_period):
    return _pyworld().synthesize(f0, decoded_sp, ap, fs, frame_period).astype(np.float32)


def world_encode_data(wavs, fs, frame_period=5.0, coded_dim=24):
    cols = ([], [], [], [], [])
    for wav in wavs:
        f0, timeaxis, sp, ap = world_decompose(wav, fs, frame_period)
        for c, v in zip(cols, (f0, timeaxis, sp, ap, world_encode_spectral_envelop(sp, fs, coded_dim))):
            c.append(v)
    return cols


# --------------------------------------------------------------------------------------------- numpy feature helpers
def transpose_in_list(lst):
    return [np.asarray(a).T for a in lst]


def _fit(coded_sps):
    cat = np.concatenate(coded_sps, axis=1)
    return np.mean(cat, axis=1, keepdims=True), np.std(cat, axis=1, keepdims=True)


def coded_sps_normalization_fit_transoform(coded_sps):
    """Per-coefficient z-normalisation over all frames of all utterances ([24, frames] each).
    Returns (normalised list, mean [24,1], std [24,1])."""
    mean, std = _fit(coded_sps)
    return [(c - mean) / std for c in coded_sps], mean, std


def coded_sps_normalization_transoform(coded_sps, coded_sps_mean, coded_sps_std):
    return [(c - coded_sps_mean) / coded_sps_std for c in coded_sps]


def coded_sps_normalization_inverse_transoform(normalized_coded_sps, coded_sps_mean, coded_sps_std):
    return [c * coded_sps_std + coded_sps_mean for c in normalized_coded_sps]


def _split_pad(total):
    left = total // 2
    return left, total - left


def coded_sp_padding(coded_sp, multiple=4):
    """Zero-pad the frame axis of a [features, frames] matrix to a multiple of `multiple`, the smaller half in front."""
    frames = coded_sp.shape[1]
    left, right = _split_pad(-frames % multiple)
    return np.pad(coded_sp, ((0, 0), (left, right)), 'constant', constant_values=0)


def wav_padding(wav, sr, frame_period, multiple=4):
    """Pad a waveform so that WORLD yields a frame count that is a multiple of `multiple` (generator needs T % 4 == 0)."""
    assert wav.ndim == 1
    n = len(wav)
    hop = sr * frame_period / 1000
    padded = int((np.ceil((np.floor(n / hop) + 1) / multiple + 1) * multiple - 1) * hop)
    left, right = _split_pad(padded - n)
    return np.pad(wav, (left, right), 'constant', constant_values=0)


def logf0_statistics(f0s):
    """Mean / std of log f0 over voiced frames (unvoiced frames have f0 == 0 and are masked out)."""
    logs = np.ma.log(np.concatenate(f0s))
    return logs.mean(), logs.std()


def pitch_conversion(f0, mean_log_src, std_log_src, mean_log_target, std_log_target):
    """Log-Gaussian normalised pitch transformation; unvoiced frames (f0 == 0) map to 0 (exp(-inf))."""
    with np.errstate(divide='ignore'):
        z = (np.log(f0) - mean_log_src) / std_log_src
    return np.exp(z * std_log_target + mean_log_target)


def sample_train_data(dataset_A, dataset_B, n_frames=128, rng=np.random):
    """One epoch's training pairs: both utterance index lists shuffled independently (global numpy RNG, seeded by the
    caller like train.py:13, unless `rng` is given), truncated to the shorter list, one uniform random `n_frames` crop per
    utterance.  Returns two arrays [num_samples, features, n_frames]."""
    num = min(len(dataset_A), len(dataset_B))
    order_A = np.arange(len(dataset_A)); order_B = np.arange(len(dataset_B))
    rng.shuffle(order_A); rng.shuffle(order_B)
    crops_A, crops_B = [], []
    for ia, ib in zip(order_A[:num], order_B[:num]):
        for utt, sink in ((dataset_A[ia], crops_A), (dataset_B[ib], crops_B)):     # A's crop is drawn before B's
            total = utt.shape[1]
            assert total >= n_frames
            s = rng.randint(total - n_frames + 1)
            sink.append(utt[:, s:s + n_frames])
    return np.array(crops_A), np.array(crops_B)


# ---- the same sampling contract from a counter-based generator: the host twin of the device sampler (cgvc_sample_plan in
#      include/cgvc.h, kernels in csrc/simt_kernels.cu), which draws an epoch's pairing and crops in HBM so that a training step
#      needs no host -> device copy.  Same distribution as sample_train_data (two independent uniform shuffles truncated to the
#      shorter list, one uniform crop per utterance); the random stream is keyed by (seed, epoch) instead of numpy's global state.
_M64 = (1 << 64) - 1


def _mix64(x):
    """splitmix64 finaliser on uint64 numpy arrays (wrap-around arithmetic)."""
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def _sample_key(seed, epoch, stream, idx):
    base = (int(seed) ^ ((int(epoch) << 20) & _M64) ^ ((int(stream) << 60) & _M64)) & _M64
    with np.errstate(over="ignore"):
        return _mix64(_mix64(np.array([base], dtype=np.uint64))[0] + np.asarray(idx, dtype=np.uint64))


def counter_sample_plan(lens_A, lens_B, seed, epoch, n_frames=128):
    """(utt_A, start_A, utt_B, start_B), each int array [min(len(lens_A), len(lens_B))]: the epoch's pairs in order.
    Utterances of a side are taken in ascending key order (ties by index); start = key' mod (frames - n_frames + 1)."""
    num = min(len(lens_A), len(lens_B))
    out = []
    for side, lens in ((0, np.asarray(lens_A, dtype=np.int64)), (1, np.asarray(lens_B, dtype=np.int64))):
        idx = np.arange(len(lens))
        order = np.lexsort((idx, _sample_key(seed, epoch, side, idx)))[:num]
        assert (lens[order] >= n_frames).all(), "every sampled utterance must hold an %d-frame crop (preprocess.py:217)" % n_frames
        start = (_sample_key(seed, epoch, side + 2, order) % (lens[order] - n_frames + 1).astype(np.uint64)).astype(np.int64)
        out += [order.astype(np.int64), start]
    return tuple(out)


def sample_train_data_counter(dataset_A, dataset_B, seed, epoch, n_frames=128):
    """sample_train_data with the counter-based generator: what the device sampler returns, computed on the host."""
    ua, sa, ub, sb = counter_sample_plan([d.shape[1] for d in dataset_A], [d.shape[1] for d in dataset_B], seed, epoch, n_frames)
    return (np.array([dataset_A[u][:, s:s + n_frames] for u, s in zip(ua, sa)]),
            np.array([dataset_B[u][:, s:s + n_frames] for u, s in zip(ub, sb)]))
