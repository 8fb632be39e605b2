"""Conversion driver: the caller of `CycleGAN.test` in the reference (`convert.py:8-59` of /root/reference) on the native engine.

`conversion(model_dir, model_name, data_dir, conversion_direction, output_dir)` keeps the reference's signature.  For each
utterance it does what convert.py:33-59 does around the generator call:

    f0' = pitch_conversion(f0)                      log-Gaussian pitch transformation with the stored logf0 statistics
    x   = (coded_sp.T - mean_src) / std_src         z-normalise the [24, T] MCEP matrix with the stored MCEP statistics
    y   = model.test([x], direction)[0]             generator forward on the H100 engine (T % 4 == 0)
    coded_sp' = (y * std_tgt + mean_tgt).T

What differs, and why:
  * WORLD analysis / synthesis and wav IO are CPU audio code in pyworld / librosa (absent from this image, SURVEY.md 8f-4).
    `.wav` inputs are handled only when pyworld and soundfile/librosa import; otherwise the driver works on FEATURE files:
    one `.npz` per utterance holding `f0` [T], `coded_sp` [T, 24] and optionally `ap`, as `world_decompose` +
    `world_encode_spectral_envelop` produce them.  The output is an `.npz` with `f0`, `coded_sp` (converted) and `ap`.
  * utterances are BATCHED: all utterances are padded to T % 4 == 0 (edge frames replicated, cropped off again after the
    generator) and go through `model.test_packed` in chunks of any lengths bounded by an utterance count and a frame budget
    (convolutions and instance norm stay within each utterance, so batching does not change any result); models without
    `test_packed` get groups of equal padded length through `model.test`.  The engine is sized once for the whole job.

    python -m cgvc.convert --model_dir ./model/sf1_tm1 --model_name sf1_tm1.ckpt --data_dir ./features/SF1 --conversion_direction A2B
"""
from __future__ import annotations

import argparse
import os
from collections import defaultdict

import numpy as np

from .preprocess import pitch_conversion

NUM_FEATURES = 24            # convert.py:10
SAMPLING_RATE = 16000        # convert.py:11
FRAME_PERIOD = 5.0           # convert.py:12


def load_normalization(model_dir):
    """mcep_normalization.npz / logf0s_normalization.npz written next to the checkpoint by train.py:56-57."""
    mcep = np.load(os.path.join(model_dir, 'mcep_normalization.npz'))
    stats = {k: mcep[k] for k in ('mean_A', 'std_A', 'mean_B', 'std_B')}
    p = os.path.join(model_dir, 'logf0s_normalization.npz')
    logf0 = None
    if os.path.exists(p):
        z = np.load(p)
        logf0 = {k: z[k] for k in ('mean_A', 'std_A', 'mean_B', 'std_B')}
    return stats, logf0


def _sides(direction):
    if direction == 'A2B':
        return 'A', 'B'
    if direction == 'B2A':
        return 'B', 'A'
    raise Exception('Conversion direction must be specified.')       # model.py:135


def _pad_frames(c, multiple=4):
    """[24, T] -> ([24, T'], left): T' = T rounded up to `multiple`, split like preprocess.coded_sp_padding (smaller half in front) but
    by REPLICATING the edge frames: the reference pads the waveform with silence before analysis (convert.py:41, wav_padding), which
    yields silence-like MCEP frames -- a raw zero vector in the MCEP domain is not one -- and only the feature matrix is available here."""
    T = c.shape[1]
    diff = -T % multiple
    left = diff // 2
    return np.pad(c, ((0, 0), (left, diff - left)), mode='edge'), left


def plan_groups(lengths, max_group=256, frame_budget=65536):
    """Batches of utterance indices with equal padded length, longest first; a batch holds at most `max_group` utterances and
    about `frame_budget` frames, so the engine's workspace is sized by a frame budget and not by (most utterances) x (longest)."""
    groups = defaultdict(list)
    for i, n in enumerate(lengths):
        groups[n].append(i)
    plan = []
    for frames in sorted(groups, reverse=True):
        idx = groups[frames]
        chunk = max(1, min(max_group, frame_budget // frames))
        for s in range(0, len(idx), chunk):
            plan.append((frames, idx[s:s + chunk]))
    return plan


def plan_chunks(lengths, max_group=256, frame_budget=65536):
    """Consecutive runs of utterance indices for packed generator calls (`model.test_packed`): a chunk holds at most `max_group`
    utterances and `frame_budget` frames; an utterance longer than the budget gets a chunk of its own."""
    plan, cur, frames = [], [], 0
    for i, n in enumerate(lengths):
        if cur and (len(cur) == max_group or frames + n > frame_budget):
            plan.append(cur)
            cur, frames = [], 0
        cur.append(i)
        frames += n
    if cur:
        plan.append(cur)
    return plan


def _special_norm_length(T):
    """Whether the engine's forward of one T-frame utterance runs an instance norm through a kernel specialised for its positions per
    sample: the fused GEMM epilogues (32, 64 or 128) or the streaming one-pass kernels (32, 48, 64, 96, 128 or 384), at the T, T/2 or
    T/4 level.  `model.test` then sums the statistics in another order than `model.test_packed`, which moves results by about 1e-5,
    so conversion keeps such utterances on the length-grouped path; for every other length the two paths agree bit for bit."""
    return any(T % d == 0 and T // d in (32, 48, 64, 96, 128, 384) for d in (1, 2, 4))


def convert_features(model, coded_sps, direction, mcep_stats, max_group=256, frame_budget=65536):
    """Convert a list of MCEP matrices (each [T_i, 24], time-major like pyworld returns them).

    Returns a list of converted [T_i, 24] float64 matrices: every utterance is padded to T % 4 == 0 for the generator's two
    stride-2 stages (edge frames replicated) and the converted frames of the padding are cropped off again, so the result lines up
    with the utterance's f0 / aperiodicity tracks frame for frame.
    """
    src, tgt = _sides(direction)
    mean_s, std_s = mcep_stats['mean_' + src], mcep_stats['std_' + src]
    mean_t, std_t = mcep_stats['mean_' + tgt], mcep_stats['std_' + tgt]
    padded, lefts = [], []
    for c in coded_sps:
        x, left = _pad_frames(np.asarray(c, dtype=np.float64).T, 4)          # [24, T']
        padded.append(x); lefts.append(left)
    out = [None] * len(padded)

    def crop(i, y):
        T = np.asarray(coded_sps[i]).shape[0]
        conv = (y.astype(np.float64) * std_t + mean_t).T                     # [T', 24]
        out[i] = np.ascontiguousarray(conv[lefts[i]:lefts[i] + T])

    grouped = list(range(len(padded)))
    if hasattr(model, "test_packed"):
        # utterances of any lengths share one generator call: a few large GEMMs instead of one small call per length
        packed = [i for i in grouped if not (hasattr(model, "test") and _special_norm_length(padded[i].shape[1]))]
        grouped = sorted(set(grouped) - set(packed))
        lengths = [padded[i].shape[1] for i in packed]
        chunks = [[packed[j] for j in ch] for ch in plan_chunks(lengths, max_group, frame_budget)]
        if chunks and hasattr(model, "_ensure_capacity"):
            # one size for the whole job: the engine takes a chunk when n <= max_batch and its frames <= max_batch * max_frames
            batch = max(len(ch) for ch in chunks)
            frames = max(sum(padded[i].shape[1] for i in ch) for ch in chunks)
            model._ensure_capacity(batch, max(16, -(-frames // (4 * batch)) * 4))
        for part in chunks:
            ys = model.test_packed([(padded[i] - mean_s) / std_s for i in part], direction)
            for i, y in zip(part, ys):
                crop(i, y)
        if not grouped:
            return out
    plan = [(f, [grouped[j] for j in part]) for f, part in plan_groups([padded[i].shape[1] for i in grouped], max_group, frame_budget)]
    if plan and hasattr(model, "_ensure_capacity"):
        # size the engine once for the whole job (its workspace is re-planned, never re-allocated, per call)
        model._ensure_capacity(max(len(part) for _, part in plan), max(frames for frames, _ in plan))
    for frames, part in plan:
        x = np.stack([(padded[i] - mean_s) / std_s for i in part])           # [n, 24, T']
        y = model.test(inputs=x, direction=direction)
        for j, i in enumerate(part):
            crop(i, y[j])
    return out


def convert_f0(f0, direction, logf0_stats):
    src, tgt = _sides(direction)
    return pitch_conversion(f0=f0, mean_log_src=logf0_stats['mean_' + src], std_log_src=logf0_stats['std_' + src],
                            mean_log_target=logf0_stats['mean_' + tgt], std_log_target=logf0_stats['std_' + tgt])


def _load_wav(path):
    try:
        import soundfile as sf
        wav, sr = sf.read(path, dtype='float64', always_2d=False)
        if wav.ndim > 1:
            wav = wav.mean(axis=1)
        if sr != SAMPLING_RATE:
            raise ValueError("%s: expected %d Hz audio" % (path, SAMPLING_RATE))
        return wav
    except ImportError:
        import librosa
        return librosa.load(path, sr=SAMPLING_RATE, mono=True)[0]


def convert_directory(model, data_dir, conversion_direction, output_dir, mcep_stats, logf0_stats):
    """Convert every utterance of `data_dir` with an already loaded model (convert.py:33-59; also the body of train.py:119-155, the
    validation conversions during training): `.npz` feature files (f0, coded_sp [T,24], optional ap) -> `.npz` with the converted
    coded_sp / f0, `.wav` files through WORLD when pyworld is available.  Returns the paths written."""
    from . import preprocess as pp

    _sides(conversion_direction)
    os.makedirs(output_dir, exist_ok=True)
    names, f0s, coded, aps, is_wav = [], [], [], [], []
    for file in sorted(os.listdir(data_dir)):
        path = os.path.join(data_dir, file)
        if file.endswith('.npz'):
            z = np.load(path)
            f0s.append(z['f0']); coded.append(z['coded_sp']); aps.append(z['ap'] if 'ap' in z else None); is_wav.append(False)
        elif file.endswith('.wav'):
            wav = pp.wav_padding(wav=_load_wav(path), sr=SAMPLING_RATE, frame_period=FRAME_PERIOD, multiple=4)
            f0, _, sp, ap = pp.world_decompose(wav=wav, fs=SAMPLING_RATE, frame_period=FRAME_PERIOD)
            f0s.append(f0); coded.append(pp.world_encode_spectral_envelop(sp=sp, fs=SAMPLING_RATE, dim=NUM_FEATURES)); aps.append(ap); is_wav.append(True)
        else:
            continue
        names.append(file)
    converted = convert_features(model, coded, conversion_direction, mcep_stats)
    written = []
    for name, f0, sp_c, ap, wav_in in zip(names, f0s, converted, aps, is_wav):
        f0_c = convert_f0(f0, conversion_direction, logf0_stats) if logf0_stats is not None else f0
        if wav_in:
            decoded = pp.world_decode_spectral_envelop(coded_sp=sp_c, fs=SAMPLING_RATE)
            wav_out = pp.world_speech_synthesis(f0=f0_c, decoded_sp=decoded, ap=ap, fs=SAMPLING_RATE, frame_period=FRAME_PERIOD)
            import soundfile as sf
            out = os.path.join(output_dir, os.path.basename(name))
            sf.write(out, wav_out, SAMPLING_RATE)
        else:
            out = os.path.join(output_dir, os.path.basename(name))
            blob = {'f0': f0_c, 'coded_sp': sp_c}
            if ap is not None:
                blob['ap'] = ap
            np.savez(out, **blob)
        written.append(out)
    return written


def conversion(model_dir, model_name, data_dir, conversion_direction, output_dir, precision='bf16x3'):
    from .model import CycleGAN

    _sides(conversion_direction)
    model = CycleGAN(num_features=NUM_FEATURES, mode='test', precision=precision)
    model.load(filepath=os.path.join(model_dir, model_name))
    mcep_stats, logf0_stats = load_normalization(model_dir)
    return convert_directory(model, data_dir, conversion_direction, output_dir, mcep_stats, logf0_stats)


def main():
    p = argparse.ArgumentParser(description='Convert voices using a trained CycleGAN model (native H100 engine).')
    p.add_argument('--model_dir', type=str, default='./model/sf1_tm1')
    p.add_argument('--model_name', type=str, default='sf1_tm1.ckpt')
    p.add_argument('--data_dir', type=str, default='./data/evaluation_all/SF1')
    p.add_argument('--conversion_direction', type=str, default='A2B')
    p.add_argument('--output_dir', type=str, default='./converted_voices')
    p.add_argument('--precision', type=str, default='bf16x3')
    a = p.parse_args()
    conversion(a.model_dir, a.model_name, a.data_dir, a.conversion_direction, a.output_dir, a.precision)


if __name__ == '__main__':
    main()
