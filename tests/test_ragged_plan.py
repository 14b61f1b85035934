"""Batch planning of the ragged file front end (evaluation.plan_batches) and the ragged C entry points' presence in the library; no GPU."""
import random

import pytest

from cmgan_b200 import evaluation, signal

SR = 16000


def _T(L):
    return signal.ragged_padded_length(L) // 100 + 1


def test_plan_every_file_once_sorted_and_bounded():
    rnd = random.Random(0)
    lengths = [rnd.randint(int(1.5 * SR), 15 * SR) for _ in range(824)] + [SR * 2] * 5       # includes ties
    batches, solo = evaluation.plan_batches(lengths, cut_len=SR * 16, max_batch=16)
    assert solo == []
    flat = [i for b in batches for i in b]
    assert sorted(flat) == list(range(len(lengths)))                   # every file exactly once
    assert [lengths[i] for i in flat] == sorted(lengths)               # sorted by length
    assert all(1 <= len(b) <= 16 for b in batches)
    for b, nxt in zip(batches, batches[1:]):                           # a batch closes only when full or at the 2^31-element bound
        tmax = _T(lengths[b[-1]])
        assert len(b) * tmax * 201 * 320 < 2 ** 31
        assert len(b) == 16 or (len(b) + 1) * _T(lengths[nxt[0]]) * 201 * 320 >= 2 ** 31
    waste = evaluation.padding_waste(lengths, batches)
    assert 0.0 <= waste < 0.05                                         # neighbours in length share a batch


def test_plan_element_bound():
    # 16 s clips: T = 2561 frames, 2561 * 201 * 320 = 1.65e8 elements per clip -> at most 13 clips below 2^31
    lengths = [SR * 16] * 40
    batches, _ = evaluation.plan_batches(lengths, cut_len=SR * 16, max_batch=64)
    per = max(len(b) for b in batches)
    assert per * _T(SR * 16) * 201 * 320 < 2 ** 31 <= (per + 1) * _T(SR * 16) * 201 * 320
    assert sorted(i for b in batches for i in b) == list(range(40))


def test_plan_routes_long_files_to_fold_path():
    lengths = [SR * 3, SR * 20, SR * 5, SR * 16 + 1, SR * 16]
    batches, solo = evaluation.plan_batches(lengths, cut_len=SR * 16, max_batch=4)
    assert solo == [1, 3]                                              # padded length > cut_len
    assert batches == [[0, 2, 4]]


def test_plan_max_batch_one_is_per_file():
    lengths = [300, 5000, 1234]
    batches, solo = evaluation.plan_batches(lengths, max_batch=1)
    assert batches == [[0], [2], [1]] and solo == []


@pytest.mark.parametrize("L", [1, 50, 150, 199, 200])
def test_plan_rejects_too_short(L):
    # wrap padding takes the pad from the clip's own head; the padded clip must exceed the 200-sample reflect padding
    with pytest.raises(ValueError, match="too short"):
        evaluation.plan_batches([SR, L])


def test_padded_length():
    assert signal.ragged_padded_length(250) == 300                     # 50 samples of wrap padding from a 250-sample clip
    assert signal.ragged_padded_length(4100) == 4100
    assert signal.ragged_padded_length(33483) == 33500
    with pytest.raises(ValueError):
        signal.ragged_padded_length(SR * 16 + 1, cut_len=SR * 16)


def test_ragged_entry_points_declared_and_exported():
    from cmgan_b200._lib import lib, parse_header
    names = {"cmgan_attention_fwd_ragged", "cmgan_attention_fwd_tf32_ragged", "cmgan_glu_dwconv_fwd_ragged", "cmgan_norm_stats_ragged",
             "cmgan_norm_finalize_ragged", "cmgan_rms_scale_ragged", "cmgan_pad_wrap_reflect_ragged", "cmgan_ola_ragged",
             "cmgan_tscnet_fwd_ragged"}
    protos = parse_header()
    assert names <= set(protos)
    for n in names:
        getattr(lib().cdll, n)
    assert lib().cdll.cmgan_abi_version() == 1
