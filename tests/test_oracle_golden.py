"""The oracle (oracle/cmgan_oracle.py) against fixtures produced by the REFERENCE modules
(tools/make_golden.py).  Runs everywhere (no reference checkout needed)."""
import numpy as np
import torch

from oracle import cmgan_oracle as O


def _t(a):
    return torch.from_numpy(np.asarray(a))


def _close(a, b, atol, rtol=0.0, name=""):
    a, b = _t(a).double(), _t(b).double()
    err = (a - b).abs().max().item()
    ref = b.abs().max().item()
    assert err <= atol + rtol * ref, f"{name}: max-abs err {err:.3e} (ref max {ref:.3e})"


def test_stft_compress(golden):
    wav = _t(golden["wav"])
    spec = O.stft(wav)
    _close(spec, golden["stft"], 2e-5, name="stft")            # FFT vs direct DFT rounding, |X| up to ~3
    comp = O.power_compress(_t(golden["stft"]))
    _close(comp, golden["compress"], 1e-6, name="compress")


def test_uncompress_istft(golden):
    comp = _t(golden["compress"])
    unc = O.power_uncompress(comp[:, 0:1], comp[:, 1:2])
    _close(unc, golden["uncompress"], 2e-6, name="uncompress")
    wav = O.istft(_t(golden["uncompress"]).squeeze(1))
    _close(wav, golden["istft"], 2e-6, name="istft")
    # stft -> compress -> uncompress -> istft is the identity on the waveform
    _close(wav, golden["wav"], 5e-6, name="round trip")


def test_tscnet_eval(golden, g_weights):
    x = _t(golden["compress"]).permute(0, 1, 3, 2)
    taps = {}
    with torch.no_grad():
        fr, fi = O.tscnet_forward(x, g_weights, taps=taps)
    for k, v in taps.items():
        v = v[:, ::4] if v.shape[1] == 64 else v
        _close(v, golden["tap_" + k], 1e-4, name="tap " + k)
    _close(fr, golden["tscnet_real"], 1e-4, name="final_real")
    _close(fi, golden["tscnet_imag"], 1e-4, name="final_imag")


def test_submodules(golden, g_weights):
    xc = _t(golden["conf_in"])
    with torch.no_grad():
        _close(O.conformer_block(xc, g_weights, "TSCB_1.time_conformer"), golden["conf_time1_out"], 2e-5, name="conf t1")
        _close(O.conformer_block(xc, g_weights, "TSCB_3.freq_conformer"), golden["conf_freq3_out"], 2e-5, name="conf f3")
        _close(O.attention(xc, g_weights, "TSCB_2.time_conformer.attn"), golden["attn_out"], 1e-5, name="attn")
        _close(O.feed_forward(xc, g_weights, "TSCB_2.time_conformer.ff1"), golden["ff_out"], 1e-5, name="ff")
        _close(O.conv_module(xc, g_weights, "TSCB_2.time_conformer.conv"), golden["convmod_out"], 1e-5, name="convmod")
        xd = _t(golden["dense_in"])
        _close(O.dilated_dense(xd, g_weights, "dense_encoder.dilated_dense"), golden["dense_enc_out"], 2e-5, name="dense")
        _close(O.sp_conv_transpose(xd, g_weights, "mask_decoder.sub_pixel"), golden["subpixel_out"], 1e-5, name="subpixel")
        _close(O.attention(_t(golden["attn_long_in"]), g_weights, "TSCB_1.time_conformer.attn"), golden["attn_long_out"], 1e-5,
               name="attn L=600 (clamp)")


def test_convmod_train_batchnorm(golden, g_weights):
    xc = _t(golden["conf_in"])
    bn = {}
    p = "TSCB_2.time_conformer.conv"
    with torch.no_grad():
        out = O.conv_module(xc, g_weights, p, training=True, bn_out=bn)
    _close(out, golden["convmod_train_out"], 2e-5, name="convmod train")
    mean, var_unb = bn[p]
    rm = 0.9 * g_weights[p + ".net.5.running_mean"] + 0.1 * mean
    rv = 0.9 * g_weights[p + ".net.5.running_var"] + 0.1 * var_unb
    _close(rm, golden["convmod_train_rm"], 1e-6, name="running_mean")
    _close(rv, golden["convmod_train_rv"], 1e-6, name="running_var")


def test_enhance(golden, g_weights):
    with torch.no_grad():
        e = O.enhance(_t(golden["wav"])[0:1], g_weights)
        _close(e, golden["enhance_short"], 2e-6, name="enhance short")
        e = O.enhance(_t(golden["wav_fold"]), g_weights, cut_len=1000)
        _close(e, golden["enhance_fold"], 2e-6, name="enhance fold")


def test_discriminator(golden, d_weights):
    x, y = _t(golden["d_x"]), _t(golden["d_y"])
    with torch.no_grad():
        _close(O.discriminator_forward(x, y, d_weights, training=False), golden["d_eval_out"], 1e-6, name="D eval")
        uv = {}
        _close(O.discriminator_forward(x, y, d_weights, training=True, uv_out=uv), golden["d_train_out"], 1e-6, name="D train")
        for li, (u, v) in uv.items():
            _close(u, golden[f"d_train_u{li}"], 1e-6, name=f"u{li}")
            _close(v, golden[f"d_train_v{li}"], 1e-6, name=f"v{li}")


def test_generator_grads(golden, g_weights):
    """Autograd through the oracle reproduces the reference's parameter gradients."""
    # fp64 oracle: the reference's own fp32 backward carries ~1e-3 relative rounding noise in the
    # deepest (encoder) gradients [measured: reference-fp32 vs oracle-fp64 2.8e-3 of max on conv_1],
    # so the comparison is made against the noise-free side with that tolerance.
    sd = {k: (v.double().requires_grad_(True) if v.is_floating_point() else v) for k, v in g_weights.items()}
    clean, noisy = _t(golden["grad_clean"]).double(), _t(golden["grad_noisy"]).double()
    go = O.forward_generator_step(clean, noisy, sd)
    import torch.nn.functional as F
    loss = 0.1 * (F.mse_loss(go["est_real"], go["clean_real"]) + F.mse_loss(go["est_imag"], go["clean_imag"])) \
        + 0.9 * F.mse_loss(go["est_mag"], go["clean_mag"]) + 0.2 * torch.mean(torch.abs(go["est_audio"] - clean))
    loss.backward()
    assert abs(loss.item() - float(golden["grad_loss"])) < 1e-6
    keys = [str(k) for k in golden["grad_norm_keys"]]
    vals = golden["grad_norm_vals"]
    for k, v in zip(keys, vals):
        gn = sd[k].grad.norm().item()
        assert abs(gn - v) <= 1e-3 * max(v, 1e-3), f"{k}: grad norm {gn} vs ref {v}"
    for k in golden.files:
        if k.startswith("grad::"):
            _close(sd[k[6:]].grad, golden[k], 1e-6, rtol=5e-3, name=k)


def test_real_utterance(g_weights):
    import os
    from scipy.io import wavfile
    from conftest import GOLDEN
    sr, w = wavfile.read(os.path.join(GOLDEN, "p232_170_noisy.wav"))
    wf = torch.from_numpy(w[:16000].astype(np.float32) / 32768.0).unsqueeze(0)
    ref_full = np.load(os.path.join(GOLDEN, "p232_170_enhanced_ref.npy"))
    # the fixture is the full 2.09 s file; run the oracle on the full file (about 2 s of CPU)
    wfull = torch.from_numpy(w.astype(np.float32) / 32768.0).unsqueeze(0)
    with torch.no_grad():
        e = O.enhance(wfull, g_weights, cut_len=16000 * 16)
    _close(e, ref_full, 2e-6, name="p232_170 enhanced")
    assert wf.shape[1] == 16000
