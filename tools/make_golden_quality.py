#!/usr/bin/env python
"""Generate tests/golden/audiosamples_quality.npz from the REFERENCE (build container only): for the 25 AudioSamples utterances already in
tests/golden/audiosamples.npz, the log-likelihood-ratio and weighted-spectral-slope figures the reference's own
src/tools/compute_metrics.py functions ``llr`` / ``wss`` give (aggregated as compute_metrics.py:45-55 does: mean of the lowest 95 %),
for (clean, noisy) at 16-bit sample scale -- how the shipped log was produced -- and for (clean, reference-enhanced) at unit scale -- how
evaluation.py calls it -- plus per-frame values of two utterances, and the PESQ / CSIG / CBAK / COVL columns of the reference's shipped log
src/tools/Noisy_metrics_results/python_noisy_metrics.log (known answers for the composite measures).  Tests read only the .npz."""
import os
import re
import sys
import types

import numpy as np

REF = os.path.join(os.environ.get("CMGAN_REFERENCE", "CMGAN"), "src")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    sys.modules.setdefault("pesq", types.SimpleNamespace(pesq=lambda *a, **k: float("nan")))
    sys.path.insert(0, os.path.join(REF, "tools"))
    import compute_metrics as cm
    z = np.load(os.path.join(ROOT, "tests", "golden", "audiosamples.npz"))
    off = np.concatenate([[0], np.cumsum(z["lengths"])])
    names = [str(n) for n in z["names"]]
    pat = re.compile(r"Track name: (\S+)\s+PESQ: (\S+)\s+CSIG: (\S+)\s+CBAK: (\S+)\s+COVL: (\S+)\s+SSNR: (\S+)\s+STOI: (\S+)")
    log = {}
    for line in open(os.path.join(REF, "tools", "Noisy_metrics_results", "python_noisy_metrics.log")):
        m = pat.search(line)
        if m:
            log[m.group(1)] = [float(m.group(k)) for k in range(2, 8)]

    def agg(v):
        s = np.sort(v)
        return float(np.mean(s[: round(np.size(s) * 0.95)]))
    rows, frames = [], {}
    for i, nm in enumerate(names):
        c16 = z["clean"][off[i]:off[i + 1]].astype(np.float64)
        n16 = z["noisy"][off[i]:off[i + 1]].astype(np.float64)
        enh = z["enhanced_ref"][off[i]:off[i + 1]].astype(np.float64)
        cf = c16 / 32768.0
        l_n, w_n = cm.llr(c16, n16, 16000), cm.wss(c16, n16, 16000)
        l_e, w_e = cm.llr(cf, enh, 16000), cm.wss(cf, enh, 16000)
        rows.append([agg(l_n), agg(w_n), agg(l_e), agg(w_e)] + log.get(nm, [np.nan] * 6)[:4])
        if i in (0, 7):
            frames[f"llr_noisy_{i}"], frames[f"wss_noisy_{i}"] = l_n, w_n
            frames[f"llr_enh_{i}"], frames[f"wss_enh_{i}"] = l_e, w_e
        print(nm, ["%.5f" % v for v in rows[-1]], flush=True)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "audiosamples_quality.npz"), names=np.array(names),
                        quality=np.array(rows, dtype=np.float64),
                        quality_cols=np.array(["llr_noisy_int16", "wss_noisy_int16", "llr_ref_enh_unit", "wss_ref_enh_unit", "log_pesq", "log_csig",
                                               "log_cbak", "log_covl"]), **frames)


if __name__ == "__main__":
    main()
