#!/usr/bin/env python
"""Generate tests/golden/reference_pins.npz: outputs of the REFERENCE modules that tests/test_oracle_vs_reference.py pins the oracle to.

    CMGAN_REFERENCE=/path/to/CMGAN python tools/make_golden_pins.py

Runs the reference's TSCNet (shipped checkpoint = tests/golden/weights_g.npz), its power_compress / power_uncompress and its
Discriminator (train mode, weights_d.npz, dropout off) on CPU fp32 with fixed seeds and stores inputs and outputs.
Nothing in here is used at test time.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import cmgan_oracle as O  # noqa: E402


def main(src: str) -> None:
    sys.path.insert(0, src)
    stub = types.ModuleType("pesq")
    stub.pesq = lambda *a, **k: 0.0
    sys.modules["pesq"] = stub
    try:                            # discriminator.py imports joblib for its PESQ batch helper, which is not called here
        import joblib  # noqa: F401
    except ImportError:
        stub = types.ModuleType("joblib")
        stub.Parallel = stub.delayed = None
        sys.modules["joblib"] = stub
    from models.generator import TSCNet
    from models.discriminator import Discriminator
    import utils as U

    out = {}
    m = TSCNet(64, 201)
    m.load_state_dict(O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_g.npz")))
    m.eval()
    torch.manual_seed(3)
    x = torch.randn(1, 2, 23, 201) * 0.7
    with torch.no_grad():
        a = m(x)
    out.update(tscnet_x=x, tscnet_real=a[0], tscnet_imag=a[1])

    torch.manual_seed(1)
    s = torch.randn(2, 201, 9, 2)
    s[0, 0, 0] = 0.0
    c = U.power_compress(s)
    out.update(compress_x=s, compress_y=c, uncompress_y=U.power_uncompress(c[:, 0:1], c[:, 1:2]))

    D = Discriminator(ndf=16)
    D.load_state_dict(O.load_weights_npz(os.path.join(ROOT, "tests", "golden", "weights_d.npz")))
    D.train()
    D.layers[15].p = 0.0
    torch.manual_seed(11)
    dx, dy = torch.rand(3, 1, 201, 33), torch.rand(3, 1, 201, 33)
    with torch.no_grad():
        out.update(disc_x=dx, disc_y=dy, disc_out=D(dx, dy))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "reference_pins.npz"),
                        **{k: v.detach().numpy().astype(np.float32) for k, v in out.items()})


if __name__ == "__main__":
    main(os.path.join(os.environ.get("CMGAN_REFERENCE", "CMGAN"), "src"))
