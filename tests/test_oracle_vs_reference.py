"""Pin the oracle against outputs of the reference modules stored by tools/make_golden_pins.py (tests/golden/reference_pins.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import cmgan_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def pins():
    z = np.load(os.path.join(GOLDEN, "reference_pins.npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


def test_tscnet_random_input(pins, g_weights):
    with torch.no_grad():
        b = O.tscnet_forward(pins["tscnet_x"], g_weights)
    for u, v in zip((pins["tscnet_real"], pins["tscnet_imag"]), b):
        assert (u - v).abs().max().item() < 3e-5


def test_stft_matches_torch():
    torch.manual_seed(0)
    x = torch.randn(3, 1700) * 0.1
    a = torch.view_as_real(torch.stft(x, 400, 100, window=torch.hamming_window(400), onesided=True, return_complex=True))
    assert (a - O.stft(x)).abs().max().item() < 2e-5
    y = torch.istft(torch.view_as_complex(a.contiguous()), 400, 100, window=torch.hamming_window(400), onesided=True)
    assert (y - O.istft(a)).abs().max().item() < 2e-6


def test_compress_matches(pins):
    c = pins["compress_y"]
    assert (c - O.power_compress(pins["compress_x"])).abs().max().item() < 1e-6
    assert (pins["uncompress_y"] - O.power_uncompress(c[:, 0:1], c[:, 1:2])).abs().max().item() < 1e-5


def test_discriminator_train_mode(pins, d_weights):
    dsd = {k: v.clone() for k, v in d_weights.items()}
    b = O.discriminator_forward(pins["disc_x"], pins["disc_y"], dsd, training=True)
    assert (pins["disc_out"] - b).abs().max().item() < 1e-6
