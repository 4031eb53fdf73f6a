"""Data-parallel training of the spectrogram U-Net without a GPU: the sharded float64 step (tests/spectrogram_shards.py) against
the whole-batch oracle at 2 and 3 ranks, even and uneven shards; the shards' dropout masks against the whole batch's; the
exported C entry point; and Training.py's sync_batch_norm option."""
import numpy as np
import pytest

import Training
import wun
from oracle import spectrogram_oracle as S
from oracle import spectrogram_train_oracle as O
from spectrogram_shards import shard_bounds, shard_masks, sharded_step

NAMES = ["accompaniment", "vocals"]

CASES = [
    # (label, layers, filters, STFT frames, shard sizes, raw_audio_loss)
    ("l3_u7_2+2", 3, 2, 8, (2, 2), True),
    ("l3_u7a_3+1", 3, 2, 8, (3, 1), False),
    ("l2_u7_2+1+1", 2, 3, 4, (2, 1, 1), True),
    ("l4_u7a_1+2+1", 4, 2, 16, (1, 2, 1), False),
]


def problem(L, Fi, n, B, seed):
    T = 1024 + 768 * (n - 1)
    rng = np.random.default_rng(seed)
    params = S.random_params(L, Fi, seed=seed)
    mix = rng.uniform(-0.5, 0.5, (B, T, 1)).astype(np.float32)
    targets = [rng.uniform(-0.3, 0.3, (B, T, 1)).astype(np.float32) for _ in range(2)]
    return params, mix, targets


@pytest.mark.parametrize("label,L,Fi,n,sizes,raw", CASES, ids=[c[0] for c in CASES])
def test_sharded_step_is_the_whole_batch_step(label, L, Fi, n, sizes, raw):
    B, seed, step = sum(sizes), 1337, 5
    params, mix, targets = problem(L, Fi, n, B, seed=len(sizes) + L)
    want_loss, want_g, want_moving = O.forward_backward(params, mix, targets, L, NAMES, raw,
                                                        O.engine_masks(seed, step, B, n, L, Fi))
    one = sharded_step(params, mix, targets, L, NAMES, raw, seed, step, Fi, [(0, B)])
    got = sharded_step(params, mix, targets, L, NAMES, raw, seed, step, Fi, shard_bounds(sizes))
    # float64 rounding: the one-pass variance and the regrouped sums differ from the oracle's in the last bits only
    assert abs(one["loss"] - want_loss) <= 1e-12 * abs(want_loss)
    assert abs(got["loss"] - want_loss) <= 1e-12 * abs(want_loss)
    weighted = sum(l * (hi - lo) / B for l, (lo, hi) in zip(got["shard_losses"], shard_bounds(sizes)))
    assert abs(weighted - want_loss) <= 1e-12 * abs(want_loss)
    assert len(got["stats"]) == len(one["stats"]) == 2 * (2 * L - 1)
    for (m, v), (m1, v1) in zip(got["stats"], one["stats"]):
        assert np.allclose(m, m1, rtol=1e-11, atol=1e-14) and np.allclose(v, v1, rtol=1e-10, atol=1e-14)
    for name, want in want_moving.items():
        assert np.allclose(got["moving"][name], want, rtol=1e-11, atol=1e-14), name
    assert set(got["grads"]) == set(want_g)
    for name, want in want_g.items():
        err = np.abs(got["grads"][name] - want).max()
        # a conv bias that feeds batch norm has gradient 0 plus float64 noise
        assert err <= 1e-9 * np.abs(want).max() or err <= 1e-14, (label, name, err)


@pytest.mark.parametrize("sizes", [(2, 2), (3, 1), (2, 1, 1), (1, 1, 1, 1)])
def test_shard_masks_are_the_whole_batch_masks(sizes):
    L, Fi, n, seed, step = 5, 2, 32, 99, 12
    B = sum(sizes)
    whole = O.engine_masks(seed, step, B, n, L, Fi)
    parts = [shard_masks(seed, step, lo, hi, n, L, Fi) for lo, hi in shard_bounds(sizes)]
    for key, want in whole.items():
        assert np.array_equal(np.concatenate([p[key] for p in parts]), want), key


def test_the_data_parallel_entry_point_is_exported():
    assert "wun_spec_forward_backward_dp" in wun.SYMBOLS
    assert hasattr(wun.lib, "wun_spec_forward_backward_dp")
    assert [f[0] for f in wun.WunSpecShard._fields_] == ["rank", "world", "global_batch", "sample_offset", "gathered",
                                                         "gathered_bytes", "gather", "ctx"]


def test_command_line_turns_sync_batch_norm_into_the_keyword(monkeypatch):
    seen = []
    monkeypatch.setattr(Training, "run", lambda cfg, **kw: seen.append((cfg, kw)))
    Training.main(["with", "cfg.unet_spectrogram", "sync_batch_norm=1", "max_epochs=2"])
    Training.main(["with", "cfg.unet_spectrogram_l1"])
    (cfg, kw), (cfg2, kw2) = seen
    assert cfg["model_config"]["network"] == "unet_spectrogram"
    assert kw == {"max_epochs": 2, "sync_batch_norm": True}
    assert kw2 == {"max_epochs": None, "sync_batch_norm": False}
