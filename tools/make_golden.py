#!/usr/bin/env python
"""Generate tests/golden/* from the REFERENCE implementation (run in the build container only).

Imports the reference's own modules from $CMGAN_REFERENCE/src (a checkout of the original CMGAN repository) (generator.py, conformer.py,
utils.py, discriminator.py with a stub ``pesq`` module) and the shipped checkpoint, runs them
on CPU fp32 with fixed seeds and stores inputs + outputs as small .npz fixtures.  The glue of
train.py / evaluation.py cannot be imported (module-level argparse, missing torchaudio/natsort,
pre-2.0 torch.stft API) so the few lines between load and save are replayed here with
``return_complex=True`` / ``view_as_complex`` exactly as SURVEY.md section 8c describes.

Nothing in here is used at test time: tests read only the .npz/.wav files this script wrote.
"""
import os
import sys
import types

import numpy as np
import torch

REF = os.path.join(os.environ.get("CMGAN_REFERENCE", "CMGAN"), "src")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")


def import_reference():
    sys.path.insert(0, REF)
    if "pesq" not in sys.modules:
        stub = types.ModuleType("pesq")
        stub.pesq = lambda *a, **k: 0.0
        sys.modules["pesq"] = stub
    from models.generator import TSCNet, DilatedDenseNet  # noqa
    from models.conformer import ConformerBlock  # noqa
    from models.discriminator import Discriminator  # noqa
    import utils as ref_utils  # noqa
    return TSCNet, DilatedDenseNet, ConformerBlock, Discriminator, ref_utils


def ref_stft(x):
    return torch.view_as_real(torch.stft(x, 400, 100, window=torch.hamming_window(400), onesided=True, return_complex=True))


def ref_istft(spec):
    return torch.istft(torch.view_as_complex(spec.contiguous()), 400, 100, window=torch.hamming_window(400), onesided=True)


def ref_enhance(model, noisy, ref_utils, cut_len=None):
    """evaluation.py:21-53 replayed with the torch>=2 complex API."""
    c = torch.sqrt(noisy.size(-1) / torch.sum((noisy ** 2.0), dim=-1))
    noisy = torch.transpose(noisy, 0, 1)
    noisy = torch.transpose(noisy * c, 0, 1)
    length = noisy.size(-1)
    frame_num = int(np.ceil(length / 100))
    padded_len = frame_num * 100
    padding_len = padded_len - length
    noisy = torch.cat([noisy, noisy[:, :padding_len]], dim=-1)
    if cut_len is not None and padded_len > cut_len:
        batch_size = int(np.ceil(padded_len / cut_len))
        while 100 % batch_size != 0:
            batch_size += 1
        noisy = torch.reshape(noisy, (batch_size, -1))
    noisy_spec = ref_stft(noisy)
    noisy_spec = ref_utils.power_compress(noisy_spec).permute(0, 1, 3, 2)
    est_real, est_imag = model(noisy_spec)
    est_real, est_imag = est_real.permute(0, 1, 3, 2), est_imag.permute(0, 1, 3, 2)
    est_spec_uncompress = ref_utils.power_uncompress(est_real, est_imag).squeeze(1)
    est_audio = ref_istft(est_spec_uncompress)
    est_audio = est_audio / c
    return torch.flatten(est_audio)[:length]


def main():
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(8)
    TSCNet, DilatedDenseNet, ConformerBlock, Discriminator, ref_utils = import_reference()
    sd = torch.load(os.path.join(REF, "best_ckpt", "ckpt"), map_location="cpu")
    np.savez(os.path.join(OUT, "weights_g.npz"), **{k: v.numpy() for k, v in sd.items()})
    model = TSCNet(64, 201)
    model.load_state_dict(sd, strict=True)
    model.eval()

    g = {}
    # ---- front/back end -------------------------------------------------------------------
    gen = torch.Generator().manual_seed(1234)
    wav = 0.05 * torch.randn(2, 4000, generator=gen) + 0.05 * torch.randn(2, 4000, generator=gen)
    spec = ref_stft(wav)
    comp = ref_utils.power_compress(spec)
    g["wav"] = wav.numpy()
    g["stft"] = spec.numpy()
    g["compress"] = comp.numpy()
    unc = ref_utils.power_uncompress(comp[:, 0:1], comp[:, 1:2])
    g["uncompress"] = unc.numpy()
    g["istft"] = ref_istft(unc.squeeze(1)).numpy()

    # ---- whole generator (eval) on a short clip -------------------------------------------
    with torch.no_grad():
        x = comp.permute(0, 1, 3, 2)
        taps = {}
        hooks = [model.dense_encoder.register_forward_hook(lambda m, i, o: taps.__setitem__("encoder", o))]
        for i in range(1, 5):
            hooks.append(getattr(model, f"TSCB_{i}").register_forward_hook(
                lambda m, ii, o, i=i: taps.__setitem__(f"tscb{i}", o)))
        hooks.append(model.mask_decoder.register_forward_hook(lambda m, i, o: taps.__setitem__("mask", o)))
        hooks.append(model.complex_decoder.register_forward_hook(lambda m, i, o: taps.__setitem__("complex", o)))
        fr, fi = model(x)
        for h in hooks:
            h.remove()
        g["tscnet_real"] = fr.numpy()
        g["tscnet_imag"] = fi.numpy()
        for k, v in taps.items():
            # 64-channel taps are stored with every 4th channel only (fixture size)
            v = v[:, ::4] if v.shape[1] == 64 else v
            g["tap_" + k] = v.contiguous().numpy()
        g["enhance_short"] = ref_enhance(model, wav[0:1], ref_utils).numpy()
        # chunk-to-batch folding path (cut_len smaller than the clip)
        wav2 = 0.07 * torch.randn(1, 3950, generator=gen)
        g["wav_fold"] = wav2.numpy()
        g["enhance_fold"] = ref_enhance(model, wav2, ref_utils, cut_len=1000).numpy()

    # ---- sub-modules ----------------------------------------------------------------------
    with torch.no_grad():
        xc = torch.randn(3, 37, 64, generator=gen)
        g["conf_in"] = xc.numpy()
        g["conf_time1_out"] = model.TSCB_1.time_conformer(xc).numpy()
        g["conf_freq3_out"] = model.TSCB_3.freq_conformer(xc).numpy()
        g["attn_out"] = model.TSCB_2.time_conformer.attn(xc).numpy()
        g["ff_out"] = model.TSCB_2.time_conformer.ff1(xc).numpy()
        g["convmod_out"] = model.TSCB_2.time_conformer.conv(xc).numpy()
        xd = torch.randn(2, 64, 11, 23, generator=gen)
        g["dense_in"] = xd.numpy()
        g["dense_enc_out"] = model.dense_encoder.dilated_dense(xd).numpy()
        g["subpixel_out"] = model.mask_decoder.sub_pixel(xd).numpy()
        # long sequence: relative distance clamp at +-512 (L > 513)
        xl = torch.randn(1, 600, 64, generator=gen)
        g["attn_long_in"] = xl.numpy()
        g["attn_long_out"] = model.TSCB_1.time_conformer.attn(xl).numpy()

    # ---- train-mode conv module (batch-norm batch statistics), dropout-free ----------------
    cm = model.TSCB_2.time_conformer.conv
    cm.train()
    rm0 = cm.net[5].running_mean.clone()
    rv0 = cm.net[5].running_var.clone()
    with torch.no_grad():
        g["convmod_train_out"] = cm(xc).numpy()
    g["convmod_train_rm"] = cm.net[5].running_mean.numpy().copy()
    g["convmod_train_rv"] = cm.net[5].running_var.numpy().copy()
    cm.net[5].running_mean.copy_(rm0)
    cm.net[5].running_var.copy_(rv0)
    cm.net[5].num_batches_tracked.zero_().add_(sd["TSCB_2.time_conformer.conv.net.5.num_batches_tracked"])
    cm.eval()

    # ---- discriminator (seeded init, since the reference ships no D weights) ---------------
    torch.manual_seed(7)
    D = Discriminator(ndf=16)
    dsd = {k: v.clone() for k, v in D.state_dict().items()}
    np.savez(os.path.join(OUT, "weights_d.npz"), **{k: v.numpy() for k, v in dsd.items()})
    dx = torch.rand(2, 1, 201, 41, generator=gen) * 2.0
    dy = torch.rand(2, 1, 201, 41, generator=gen) * 2.0
    g["d_x"], g["d_y"] = dx.numpy(), dy.numpy()
    D.eval()
    with torch.no_grad():
        g["d_eval_out"] = D(dx, dy).numpy()
    D.train()
    D.layers[15].p = 0.0  # dropout off so that the train-mode output is deterministic
    with torch.no_grad():
        g["d_train_out"] = D(dx, dy).numpy()
    for li in (0, 3, 6, 9, 14, 17):
        g[f"d_train_u{li}"] = D.layers[li].weight_u.numpy().copy()
        g[f"d_train_v{li}"] = D.layers[li].weight_v.numpy().copy()

    # ---- gradients: generator loss without the GAN term, eval mode (no dropout / BN batch stats)
    model.zero_grad()
    clean = 0.05 * torch.randn(2, 1600, generator=gen)
    noisy = clean + 0.05 * torch.randn(2, 1600, generator=gen)
    g["grad_clean"], g["grad_noisy"] = clean.numpy(), noisy.numpy()
    c = torch.sqrt(noisy.size(-1) / torch.sum((noisy ** 2.0), dim=-1))
    n2 = torch.transpose(torch.transpose(noisy, 0, 1) * c, 0, 1)
    c2 = torch.transpose(torch.transpose(clean, 0, 1) * c, 0, 1)
    noisy_spec = ref_utils.power_compress(ref_stft(n2)).permute(0, 1, 3, 2)
    clean_spec = ref_utils.power_compress(ref_stft(c2))
    clean_real, clean_imag = clean_spec[:, 0:1], clean_spec[:, 1:2]
    er, ei = model(noisy_spec)
    er, ei = er.permute(0, 1, 3, 2), ei.permute(0, 1, 3, 2)
    est_mag = torch.sqrt(er ** 2 + ei ** 2)
    clean_mag = torch.sqrt(clean_real ** 2 + clean_imag ** 2)
    est_audio = ref_istft(ref_utils.power_uncompress(er, ei).squeeze(1))
    import torch.nn.functional as F
    loss = 0.1 * (F.mse_loss(er, clean_real) + F.mse_loss(ei, clean_imag)) + 0.9 * F.mse_loss(est_mag, clean_mag) \
        + 0.2 * torch.mean(torch.abs(est_audio - clean))
    loss.backward()
    g["grad_loss"] = np.array(loss.item(), dtype=np.float64)
    norms = {}
    for k, p in model.named_parameters():
        norms[k] = float(p.grad.norm()) if p.grad is not None else -1.0
    g["grad_norm_keys"] = np.array(list(norms.keys()))
    g["grad_norm_vals"] = np.array(list(norms.values()), dtype=np.float64)
    for k in ["dense_encoder.conv_1.0.weight", "dense_encoder.dilated_dense.conv2.weight", "TSCB_1.time_conformer.attn.fn.to_q.weight",
              "TSCB_4.freq_conformer.conv.net.4.conv.weight", "mask_decoder.prelu_out.weight", "complex_decoder.conv.weight",
              "TSCB_2.freq_conformer.ff1.fn.fn.net.0.bias", "TSCB_3.time_conformer.post_norm.weight"]:
        g["grad::" + k] = dict(model.named_parameters())[k].grad.numpy().copy()

    np.savez_compressed(os.path.join(OUT, "golden_small.npz"), **g)

    # ---- one real utterance from AudioSamples (first 1.0 s and the full 2.09 s file) -------
    from scipy.io import wavfile
    sr, w = wavfile.read(os.path.join(REF, "..", "AudioSamples", "noisy", "p232_170.wav"))
    assert sr == 16000
    wavfile.write(os.path.join(OUT, "p232_170_noisy.wav"), sr, w)
    wf = torch.from_numpy(w.astype(np.float32) / 32768.0).unsqueeze(0)
    with torch.no_grad():
        enh = ref_enhance(model, wf, ref_utils, cut_len=16000 * 16)
    np.save(os.path.join(OUT, "p232_170_enhanced_ref.npy"), enh.numpy())
    print("golden written to", os.path.abspath(OUT))
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
