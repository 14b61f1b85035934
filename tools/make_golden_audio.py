#!/usr/bin/env python
"""Generate tests/golden/audiosamples.npz from the REFERENCE (run in the build container only).

For each of the 25 utterances shipped under $CMGAN_REFERENCE/AudioSamples (2.1 .. 9.8 s, so the time-axis sequences reach
L = 1564 > 513: the relative-position clamp is exercised inside the whole network), this stores
  * the noisy and clean waveforms (int16, as shipped),
  * the reference's enhanced waveform: the reference's own TSCNet + power_compress/uncompress modules with the shipped
    checkpoint on CPU fp32, driven by the evaluation.py:21-53 glue replayed with the torch>=2 complex API
    (tools/make_golden.py:ref_enhance),
  * SSNR / STOI of (clean, reference-enhanced) and of (clean, noisy) computed by the reference's own
    src/tools/compute_metrics.py functions ``snr`` and ``stoi`` (imported with a stub ``pesq`` module),
  * the SSNR / STOI the reference's shipped log (src/tools/Noisy_metrics_results/python_noisy_metrics.log) lists for the
    same tracks' noisy inputs -- a known-answer check for the metrics port (oracle/metrics_oracle.py).
Nothing in here is used at test time: tests read only the .npz this script wrote.
"""
import glob
import os
import re
import sys

import numpy as np
import torch
from scipy.io import wavfile

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import REF, OUT, import_reference, ref_enhance  # noqa: E402


def main():
    torch.set_num_threads(8)
    TSCNet, _, _, _, ref_utils = import_reference()
    sys.path.insert(0, os.path.join(REF, "tools"))
    import compute_metrics as cm           # the pesq stub is already in sys.modules
    sd = torch.load(os.path.join(REF, "best_ckpt", "ckpt"), map_location="cpu")
    model = TSCNet(64, 201)
    model.load_state_dict(sd, strict=True)
    model.eval()
    log = {}
    pat = re.compile(r"Track name: (\S+)\s+PESQ: (\S+)\s+CSIG: (\S+)\s+CBAK: (\S+)\s+COVL: (\S+)\s+SSNR: (\S+)\s+STOI: (\S+)")
    for line in open(os.path.join(REF, "tools", "Noisy_metrics_results", "python_noisy_metrics.log")):
        m = pat.search(line)
        if m:
            log[m.group(1)] = (float(m.group(6)), float(m.group(7)))
    names, lens, noisy_all, clean_all, enh_all = [], [], [], [], []
    met = []
    for f in sorted(glob.glob(os.path.join(REF, "..", "AudioSamples", "noisy", "*.wav"))):
        name = os.path.basename(f)[:-4]
        sr, n16 = wavfile.read(f)
        sr2, c16 = wavfile.read(f.replace("/noisy/", "/clean/"))
        assert sr == 16000 and sr2 == 16000 and len(n16) == len(c16)
        wf = torch.from_numpy(n16.astype(np.float32) / 32768.0).unsqueeze(0)
        with torch.no_grad():
            enh = ref_enhance(model, wf, ref_utils, cut_len=16000 * 16).numpy()
        clean = c16.astype(np.float64) / 32768.0
        noisy = n16.astype(np.float64) / 32768.0
        _, seg_e = cm.snr(clean, enh.astype(np.float64), 16000)
        _, seg_n = cm.snr(clean, noisy, 16000)
        row = [float(np.mean(seg_e)), float(cm.stoi(clean, enh.astype(np.float64), 16000)), float(np.mean(seg_n)), float(cm.stoi(clean, noisy, 16000)),
               log.get(name, (np.nan, np.nan))[0], log.get(name, (np.nan, np.nan))[1]]
        print(name, len(n16), ["%.4f" % v for v in row], flush=True)
        names.append(name); lens.append(len(n16)); noisy_all.append(n16); clean_all.append(c16); enh_all.append(enh.astype(np.float32))
        met.append(row)
    np.savez_compressed(os.path.join(OUT, "audiosamples.npz"), names=np.array(names), lengths=np.array(lens, dtype=np.int64),
                        noisy=np.concatenate(noisy_all), clean=np.concatenate(clean_all), enhanced_ref=np.concatenate(enh_all),
                        metrics=np.array(met, dtype=np.float64),
                        metrics_cols=np.array(["ssnr_ref_enh", "stoi_ref_enh", "ssnr_noisy", "stoi_noisy", "log_ssnr_noisy", "log_stoi_noisy"]))
    print("written", os.path.getsize(os.path.join(OUT, "audiosamples.npz")))


if __name__ == "__main__":
    main()
