"""Training driver: the step loop of the reference's `train.py` (train.py:78-118 of /root/reference) on the native engine.

Scope (SURVEY.md 8f-1): the epoch / iteration loop, the lambda_identity and learning-rate schedule (train.py:96-102),
the random pairing + 128-frame crop sampler (`preprocess.py:207-238`), per-epoch checkpoints (train.py:113), the
normalisation side files, and the conversion of the validation utterances every 50th epoch (train.py:119-155; on feature files,
or on wavs when pyworld is installed).  OUT of scope: WORLD analysis / synthesis and wav IO (`preprocess.py:6-105`, CPU audio code;
pyworld / librosa are not available here) -- this driver starts from MCEP matrices that were already extracted:
`--train_A_dir` / `--train_B_dir` hold one `.npy` per utterance, shaped [24, frames] (what `world_encode_data` +
`transpose_in_list` produce), or `--synthetic N` draws N random utterances per speaker.

    python -m cgvc.train --synthetic 64 --epochs 2 --batch_size 8
"""
from __future__ import annotations

import argparse
import glob
import os
import time

import numpy as np

from .preprocess import coded_sps_normalization_fit_transoform, sample_train_data      # noqa: F401  (the host sampler stays the tested contract)

# hyper-parameters of train.py:15-26
NUM_MCEP = 24
N_FRAMES = 128
LAMBDA_CYCLE = 10
LAMBDA_IDENTITY = 5
GENERATOR_LR = 0.0002
DISCRIMINATOR_LR = 0.0001
LR_DECAY_START = 200000
IDENTITY_OFF_AFTER = 10000
VALIDATION_INTERVAL = 50      # train.py:120,138: validation utterances are converted every 50th epoch


def schedule(num_iterations, generator_lr=GENERATOR_LR, discriminator_lr=DISCRIMINATOR_LR):
    """(lambda_identity, generator_lr, discriminator_lr) for iteration `num_iterations`, replaying train.py:96-102:
    lambda_identity drops to 0 after 10k iterations; both learning rates decay linearly (by lr0/200000 per iteration)
    once past 200k iterations, floored at 0."""
    lam_id = 0 if num_iterations > IDENTITY_OFF_AFTER else LAMBDA_IDENTITY
    k = max(0, num_iterations - LR_DECAY_START)
    return lam_id, max(0.0, generator_lr - k * GENERATOR_LR / 200000), max(0.0, discriminator_lr - k * DISCRIMINATOR_LR / 200000)


def fit_normalization(coded_sps):
    """`coded_sps_normalization_fit_transoform` (preprocess.py:106-116): per-coefficient mean / std over all frames."""
    return coded_sps_normalization_fit_transoform(coded_sps)


class DeviceDataset:
    """Both speakers' normalised MCEP corpora resident in HBM, with the epoch sampler on the device (SURVEY.md 8f-1).

    Upload once; `plan(epoch)` draws the epoch's pairing and crops (cgvc_sample_plan, the counter-based twin of
    preprocess.sample_train_data); `minibatch(i)` gathers pairs [i*batch, (i+1)*batch) into two [batch, 24, n_frames] device
    tensors (cgvc_gather_minibatch) that go straight into CycleGAN.train_async -- no host array is touched per step."""

    def __init__(self, model, dataset_A, dataset_B, batch, n_frames=N_FRAMES, seed=0):
        import torch
        self.model, self.batch, self.n_frames, self.seed = model, int(batch), int(n_frames), int(seed)
        dev = model.device
        self.n = [len(dataset_A), len(dataset_B)]
        self.num_pairs = min(self.n)
        self.lens = [[int(d.shape[1]) for d in ds] for ds in (dataset_A, dataset_B)]
        self.corpus, self.offsets = [], []
        for ds, lens in zip((dataset_A, dataset_B), self.lens):
            flat = np.concatenate([np.ascontiguousarray(d, dtype=np.float32).reshape(-1) for d in ds])     # utterance u: [24][len_u]
            self.corpus.append(torch.from_numpy(flat).to(dev))
            self.offsets.append(torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)).to(dev))
        self.plan_dev = torch.zeros(4 * self.num_pairs, dtype=torch.int32, device=dev)
        self.err_dev = torch.zeros(1, dtype=torch.int32, device=dev)
        nf = model.num_features
        self.A = torch.empty(self.batch, nf, self.n_frames, dtype=torch.float32, device=dev)
        self.B = torch.empty(self.batch, nf, self.n_frames, dtype=torch.float32, device=dev)
        self.epoch = None

    def iterations_per_epoch(self):
        return self.num_pairs // self.batch                        # the epoch's tail is dropped, like train.py:94

    def plan(self, epoch):
        m = self.model
        m._chk(m._lib.cgvc_sample_plan(m._handle, self.offsets[0].data_ptr(), self.n[0], self.offsets[1].data_ptr(), self.n[1],
                                       self.seed, int(epoch), self.n_frames, self.plan_dev.data_ptr(), self.err_dev.data_ptr(), m._stream()))
        self.epoch = int(epoch)
        err = int(self.err_dev.item())                             # once per epoch (the reference asserts per utterance, preprocess.py:217)
        if err:
            raise AssertionError("utterance %d of speaker %s is shorter than the %d-frame crop" % ((err & ~(1 << 30)) - 1, "B" if err >> 30 else "A", self.n_frames))

    def plan_host(self):
        """The drawn plan as four int arrays (utt_A, start_A, utt_B, start_B) -- for tests / logging."""
        p = self.plan_dev.cpu().numpy().reshape(4, self.num_pairs)
        return p[0], p[1], p[2], p[3]

    def minibatch(self, i):
        m = self.model
        m._chk(m._lib.cgvc_gather_minibatch(m._handle, self.corpus[0].data_ptr(), self.offsets[0].data_ptr(), self.corpus[1].data_ptr(),
                                            self.offsets[1].data_ptr(), self.plan_dev.data_ptr(), self.num_pairs, int(i) * self.batch, self.batch,
                                            self.n_frames, self.A.data_ptr(), self.B.data_ptr(), m._stream()))
        return self.A, self.B


def load_mcep_dir(path, with_f0=False):
    """MCEP matrices [24, frames] of one speaker: `.npy` files, or the `.npz` feature files `cgvc.convert` reads
    (`coded_sp` [frames, 24] time-major as pyworld returns it, plus `f0`).  with_f0: also return the list of f0 tracks
    (None when no file carries one)."""
    files = sorted(glob.glob(os.path.join(path, "*.npy")) + glob.glob(os.path.join(path, "*.npz")))
    if not files:
        raise FileNotFoundError("no .npy / .npz MCEP features under %s (wav preprocessing with WORLD is out of scope of this driver)" % path)
    mceps, f0s = [], []
    for f in files:
        if f.endswith(".npz"):
            z = np.load(f)
            mceps.append(np.asarray(z["coded_sp"], dtype=np.float64).T)
            if "f0" in z:
                f0s.append(np.asarray(z["f0"], dtype=np.float64))
        else:
            mceps.append(np.load(f).astype(np.float64))
    if with_f0:
        return mceps, (f0s if len(f0s) == len(mceps) else None)
    return mceps


def synthetic_speaker(n_utt, seed):
    rs = np.random.RandomState(seed)
    return [np.cumsum(rs.randn(NUM_MCEP, rs.randint(N_FRAMES, 4 * N_FRAMES)), axis=1) * 0.1 + rs.randn(NUM_MCEP, 1) for _ in range(n_utt)]


def validation_conversions(model, epoch, validation_A_dir, validation_B_dir, output_dir, mcep_stats, logf0_stats, interval=VALIDATION_INTERVAL,
                           test_model=None):
    """train.py:119-155: every 50th epoch the validation utterances of both speakers are converted with the current weights
    (A -> B into `output_dir/converted_A`, B -> A into `output_dir/converted_B`).  The training engine is sized for 128-frame crops at the
    training batch; whole utterances go through a forward-only model (`test_model`, any object with set_params / test) that receives a
    copy of the current weights, so the training workspace is never re-planned for utterance-length inputs.  Returns the paths written."""
    from .convert import convert_directory
    if epoch % interval != 0 or (validation_A_dir is None and validation_B_dir is None):
        return []
    if test_model is not None and test_model is not model:
        test_model.set_params(model.get_params())
    m = test_model if test_model is not None else model
    written = []
    if validation_A_dir is not None:
        print('Generating Validation Data B from A...')                                   # train.py:121
        written += convert_directory(m, validation_A_dir, 'A2B', os.path.join(output_dir, 'converted_A'), mcep_stats, logf0_stats)
    if validation_B_dir is not None:
        print('Generating Validation Data A from B...')                                   # train.py:139
        written += convert_directory(m, validation_B_dir, 'B2A', os.path.join(output_dir, 'converted_B'), mcep_stats, logf0_stats)
    return written


def loss_scale_log(model, loss_scale):
    """The loss-scaler part of the periodic log line (empty in static mode): the state train() / fetch_losses() read last."""
    ls = model.last_loss_scale if loss_scale != 'static' else None
    if not ls:
        return ''
    if 'scale_G' in ls:                                           # loss_scale_per_network: both scales, the underflow fractions
        frac = lambda tag: ls['ufl_grad_' + tag] / ls['groups_' + tag] if ls['groups_' + tag] else 0.0
        return (', Loss Scale (G / D): {:g} / {:g}, Skipped Steps: {:d}, Saturated Groups (gradient G / D, activation): {:d} / {:d}, '
                '{:d}, Underflow Fraction (G / D): {:.2e} / {:.2e}{}').format(
            ls['scale_G'], ls['scale_D'], ls['skipped'], ls['sat_grad_G'], ls['sat_grad_D'], ls['sat_act'], frac('G'), frac('D'),
            ', Non-finite Gradients' if ls['nonfinite'] else '')
    return ', Loss Scale: {:g}, Skipped Steps: {:d}, Saturated Groups (gradient / activation): {:d} / {:d}{}'.format(
        ls['scale'], ls['skipped'], ls['sat_grad'], ls['sat_act'], ', Non-finite Gradients' if ls['nonfinite'] else '')


def train(train_A_dir, train_B_dir, model_dir, model_name, random_seed, num_epochs, mini_batch_size, synthetic=0,
          precision="bf16x3", log_every=50, device_data=True, validation_A_dir=None, validation_B_dir=None, output_dir='./validation_output',
          tensorboard_log_dir='./log', loss_scale='static', deterministic=False, loss_scale_per_network=False):
    """The reference's training loop (train.py:78-118).  device_data=True (default): the normalised corpus is uploaded once and the
    epoch sampler runs on the device (DeviceDataset), so no step copies anything host -> device and the losses are read back only
    when they are printed; device_data=False feeds host minibatches from the numpy sampler through CycleGAN.train(), like the
    reference's feed_dict.  loss_scale: 'static', 'monitor' or 'dynamic' (CycleGAN); when not static the log line also reports the
    loss scale, the skipped steps and the last step's saturated F16F8 plane groups; loss_scale_per_network: a scale each for the
    generators and the discriminators (CycleGAN), logged with each network's fraction of gradient groups below the fp16 lower edge.  deterministic: bit-reproducible steps
    (CycleGAN), so that a rerun of the same seed writes the same checkpoints."""
    from .model import CycleGAN
    np.random.seed(random_seed)                                   # train.py:13
    f0_A = f0_B = None
    if synthetic:
        A, B = synthetic_speaker(synthetic, 1), synthetic_speaker(synthetic, 2)
    else:
        A, f0_A = load_mcep_dir(train_A_dir, with_f0=True)
        B, f0_B = load_mcep_dir(train_B_dir, with_f0=True)
    A_norm, A_mean, A_std = fit_normalization(A)
    B_norm, B_mean, B_std = fit_normalization(B)
    os.makedirs(model_dir, exist_ok=True)
    np.savez(os.path.join(model_dir, 'mcep_normalization.npz'), mean_A=A_mean, std_A=A_std, mean_B=B_mean, std_B=B_std)   # train.py:57
    logf0_stats = None
    if f0_A is not None and f0_B is not None:                     # train.py:47-48,56: log-f0 statistics for convert.py's pitch conversion
        from .preprocess import logf0_statistics
        (mA, sA), (mB, sB) = logf0_statistics(f0_A), logf0_statistics(f0_B)
        np.savez(os.path.join(model_dir, 'logf0s_normalization.npz'), mean_A=mA, std_A=sA, mean_B=mB, std_B=sB)
        logf0_stats = {'mean_A': mA, 'std_A': sA, 'mean_B': mB, 'std_B': sB}
    mcep_stats = {'mean_A': A_mean, 'std_A': A_std, 'mean_B': B_mean, 'std_B': B_std}
    model = CycleGAN(num_features=NUM_MCEP, max_batch=mini_batch_size, max_frames=N_FRAMES, precision=precision, seed=random_seed,
                     log_dir=tensorboard_log_dir, loss_scale=loss_scale, deterministic=deterministic,
                     loss_scale_per_network=loss_scale_per_network)
    test_model = None
    data = DeviceDataset(model, A_norm, B_norm, mini_batch_size, N_FRAMES, seed=random_seed) if device_data else None
    g_loss = d_loss = float("nan")
    for epoch in range(num_epochs):
        t0 = time.time()
        if data is not None:
            data.plan(epoch)
            n_samples = data.num_pairs
        else:
            data_A, data_B = sample_train_data(A_norm, B_norm, n_frames=N_FRAMES)
            n_samples = data_A.shape[0]
        n_iter = n_samples // mini_batch_size                     # the epoch's tail is dropped, like train.py:94
        for i in range(n_iter):
            num_iterations = n_iter * epoch + i
            lam_id, lr_g, lr_d = schedule(num_iterations)
            log = i % log_every == 0
            if data is not None:
                a_dev, b_dev = data.minibatch(i)
                model.train_async(a_dev, b_dev, LAMBDA_CYCLE, lam_id, lr_g, lr_d)
                if log or i == n_iter - 1:
                    g_loss, d_loss = model.fetch_losses()
            else:
                s, e = i * mini_batch_size, (i + 1) * mini_batch_size
                g_loss, d_loss = model.train(input_A=data_A[s:e], input_B=data_B[s:e], lambda_cycle=LAMBDA_CYCLE, lambda_identity=lam_id,
                                             generator_learning_rate=lr_g, discriminator_learning_rate=lr_d)
            if log:
                print('Iteration: {:07d}, Generator Learning Rate: {:.7f}, Discriminator Learning Rate: {:.7f}, Generator Loss : {:.3f}, '
                      'Discriminator Loss : {:.3f}'.format(num_iterations, lr_g, lr_d, g_loss, d_loss) + loss_scale_log(model, loss_scale))
        model.save(directory=model_dir, filename=model_name)      # train.py:113
        if (validation_A_dir is not None or validation_B_dir is not None) and epoch % VALIDATION_INTERVAL == 0:      # train.py:119-155
            if test_model is None:
                test_model = CycleGAN(num_features=NUM_MCEP, mode='test', precision=precision, log_dir=tensorboard_log_dir,
                                      deterministic=deterministic)
            validation_conversions(model, epoch, validation_A_dir, validation_B_dir, output_dir, mcep_stats, logf0_stats, test_model=test_model)
        dt = time.time() - t0
        print('Epoch %d: %d iterations, time elapsed %02d:%02d:%02d' % (epoch, n_iter, dt // 3600, dt % 3600 // 60, dt % 60))
    return model, g_loss, d_loss


def main():
    p = argparse.ArgumentParser(description='Train CycleGAN model on pre-extracted MCEP features (native H100 engine).')
    p.add_argument('--train_A_dir', type=str, default='./data/mcep/SF1')
    p.add_argument('--train_B_dir', type=str, default='./data/mcep/TM1')
    p.add_argument('--model_dir', type=str, default='./model/sf1_tm1')
    p.add_argument('--model_name', type=str, default='sf1_tm1.ckpt')
    p.add_argument('--random_seed', type=int, default=0)
    p.add_argument('--epochs', type=int, default=5000)            # train.py:15
    p.add_argument('--batch_size', type=int, default=1)           # train.py:16
    p.add_argument('--validation_A_dir', type=str, default='none', help='feature (.npz) or wav directory converted A -> B every 50th epoch; none: off')
    p.add_argument('--validation_B_dir', type=str, default='none')
    p.add_argument('--output_dir', type=str, default='./validation_output')           # train.py:171
    p.add_argument('--tensorboard_log_dir', type=str, default='./log')                # train.py:172
    p.add_argument('--synthetic', type=int, default=0, help='use N random utterances per speaker instead of the data directories')
    p.add_argument('--precision', type=str, default='bf16x3')
    p.add_argument('--loss_scale', type=str, default='static', choices=['static', 'monitor', 'dynamic'],
                   help='F16F8 gradient-plane loss scale: static (fixed), monitor (fixed, saturation counted and logged) or dynamic '
                        '(saturated or non-finite steps skipped, scale adapted)')
    p.add_argument('--host_data', action='store_true', help='feed host minibatches from the numpy sampler every step (the reference\'s feed) '
                                                             'instead of the device-resident corpus + device sampler')
    p.add_argument('--deterministic', action='store_true', help='bit-reproducible train steps (fixed-order gradient and loss reductions)')
    p.add_argument('--loss_scale_per_network', action='store_true',
                   help='with --loss_scale monitor or dynamic (F16F8): a loss scale each for the generators and the discriminators')
    a = p.parse_args()
    none = lambda v: None if v in ('None', 'none') else v                                # train.py:191-192
    train(a.train_A_dir, a.train_B_dir, a.model_dir, a.model_name, a.random_seed, a.epochs, a.batch_size, a.synthetic, a.precision,
          device_data=not a.host_data, validation_A_dir=none(a.validation_A_dir), validation_B_dir=none(a.validation_B_dir),
          output_dir=a.output_dir, tensorboard_log_dir=a.tensorboard_log_dir, loss_scale=a.loss_scale, deterministic=a.deterministic,
          loss_scale_per_network=a.loss_scale_per_network)


if __name__ == '__main__':
    main()
