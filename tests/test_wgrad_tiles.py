"""The tensor-core weight gradient's warpgroup-owned tiles (kernels_umma.cu wgrad_body / umma_plan_wgrad).

Host: at the benchmark's shapes (M4, batch 16) the plan audit's issued MACs - every 64-row chunk x tap x 64-channel M block x
N-tile column the kernel issues - stay well below what 128-channel M tiles issued (223.9 GMAC), and no 64-channel M block
without a real channel is issued.
GPU: one synthetic layer per new variant - warpgroups that split the taps of a tile with one real M block (odd and single tap
counts included), a 144-channel M side of 3 blocks, and split and unsplit tiles in one launch - against float64, in the
bulk-fed and the converter-fed forms (tests/test_kernels_gpu.py runs them the same way)."""
import pytest

from configurations import plan_audit
from conv_launches import p, run_wgrad_case, wgrad_layer
from launch_checks import H, gpu_lib, lib_or_skip

OLD_ISSUED_GMAC = 223.9        # 128-channel M tiles, same swap / NT rules: the same audit at the parent's tiling


def _wgrad_lines():
    return [d for d in plan_audit("baseline_stereo", 16) if d["op"] == "wgrad"]


def test_issued_macs_of_the_benchmark_step():
    wgs = _wgrad_lines()
    issued = sum(d["issued_macs"] for d in wgs)
    useful = sum(d["useful_macs"] for d in wgs)
    assert abs(useful / 1e9 - 126.0) < 0.1, useful                # the real-channel MACs do not depend on the tiling
    assert issued <= 0.81 * OLD_ISSUED_GMAC * 1e9, issued / 1e9
    layer1 = [d for d in wgs if d["layer"] == 1]
    share = sum(d["useful_macs"] for d in layer1) / sum(d["issued_macs"] for d in layer1)
    assert share >= 0.5, share


def test_no_m_block_without_a_real_channel():
    for d in _wgrad_lines():
        Cm, Cn = (d["Cg"], d["Cp"]) if d["swap"] else (d["Cp"], d["Cg"])
        blocks = (Cm + 63) // 64
        assert blocks * 64 - Cm < 64, d
        rows = d["chunks"] * 64
        assert d["issued_macs"] == rows * d["ntaps"] * 64 * blocks * d["NT"] * d["ntiles"], d
        assert d["useful_macs"] == rows * d["ntaps"] * d["Cp"] * d["Cg"], d


def tile_cases():
    return [
        # M side of 48 channels (down1's shape, 8 taps): both warpgroups on one block, 4 taps each
        wgrad_layer(name="tsplit_8taps", batch=3, cout=48, planes=[p(24, -4, 400)], classes=[(0, 390)],
                    groups=[(0, 0, [(j, j - 4) for j in range(8)])]),
        # one tap (warpgroup 1 issues nothing) and three taps (2 + 1) in one launch
        wgrad_layer(name="tsplit_1_and_3_taps", batch=2, cout=40, planes=[p(16, 0, 300), p(32, -1, 301)], classes=[(0, 290)],
                    groups=[(0, 0, [(0, 0)]), (0, 1, [(0, -1), (1, 0), (2, 1)])]),
        # 144-channel M side: tile 0 = two blocks, tile 1 = one block whose taps the warpgroups split
        wgrad_layer(name="m144_three_blocks", batch=2, cout=144, planes=[p(120, -2, 333)], classes=[(0, 320)],
                    groups=[(0, 0, [(j, j - 2) for j in range(5)])]),
        # one launch: Cp 72 on M (two blocks, 8 real channels in the second) next to Cp 48 on M (one block, taps split), NT 48
        wgrad_layer(name="m72_next_to_m48", batch=2, cout=48, planes=[p(72, -1, 260), p(48, 0, 260)], classes=[(0, 250)],
                    groups=[(0, 0, [(0, -1), (1, 0), (2, 1)]), (0, 1, [(0, 0), (1, 1)])]),
    ]


def test_tile_cases_plan_the_variants_they_are_for():
    lib_or_skip()
    plans = {W["name"]: H.plan_wgrad(H.wgrad_text(W["groups"])) for W in tile_cases()}
    for name, pw in plans.items():
        assert pw["eligible"] and pw["bulk"], name
    g = plans["tsplit_8taps"]["groups"][0]
    assert g["swap"] == 1 and g["n_mtiles"] == 1 and g["taps_per_cta"] == 8 and g["NT"] == 32, g
    g = plans["m144_three_blocks"]["groups"][0]
    assert g["swap"] == 1 and g["n_mtiles"] == 2 and g["NT"] == 128, g
    for g in plans["m72_next_to_m48"]["groups"]:
        assert g["swap"] == 0 and g["NT"] == 48 and g["n_mtiles"] == 1, g
    assert [g["taps_per_cta"] for g in plans["tsplit_1_and_3_taps"]["groups"]] == [1, 3]


@pytest.mark.gpu
@pytest.mark.parametrize("regime", ["exact", "float"])
@pytest.mark.parametrize("mode", [0, 1, 2], ids=["bulk_fused", "bulk_colsum", "converter"])
def test_tile_variants_match_float64(mode, regime):
    gpu_lib()
    for k, W in enumerate(tile_cases()):
        run_wgrad_case(W, mode, regime, 3000 + k, 0.5 if k % 2 else 2.0)
