"""Phase D of the candidates kernel at the narrow CTA shape (R = 4) with more hull candidates than the warp scratch holds.
Every pose of a rotation is a separate contour (four level images of isolated pixels), so a bin has up to 4 * 256 = 1024
candidates; the kernel keeps the candidate lists of a bin in its warp's shared-memory scratch up to LIST_CAP_WS (768)
candidates and in the global list scratch (Params::dlist) beyond.  Bins at 1024, 768 (the largest that stays in shared
memory) and 769 candidates, through irbpp_debug_hulls at three table sizes (truncation to a few rows, to the usual 500,
and no truncation), against the oracle's convex_hull_actions + select_candidates.  Run on host threads under the CUDA
emulator here and on the device with -m gpu."""
import numpy as np
import pytest

from test_kernels_emulated import EmuEnv, _P, build_emulated

R = 4
N_BINS = 4
SELS = (24, 500, 1024)


def spill_inputs():
    """posZValid / mask [N_BINS, R, 16, 16]: feasible poses on levels 1..4 by the parity of (x, y), so no two poses of one
    level image touch and every feasible pose is a one-pixel contour; heights vary inside a level (truncation ranking)."""
    rng = np.random.default_rng(11)
    xs, ys = np.meshgrid(np.arange(16), np.arange(16), indexing="ij")
    level = (xs % 2) + 2 * (ys % 2)
    pv = np.full((N_BINS, R, 16, 16), 1e3)
    mk = np.zeros((N_BINS, R, 16, 16))
    for i, nrot in enumerate((R, R, 3, 3)):           # 1024, 1024, 768, 769 candidates
        for r in range(nrot):
            mk[i, r] = 1
            pv[i, r] = 0.015 + 0.01 * level + 0.004 * np.round(rng.random((16, 16)), 2)
    mk[3, 3, 5, 9] = 1
    pv[3, 3, 5, 9] = 0.021
    return pv, mk


def check_spill(run_hulls, sel):
    """``run_hulls(posZValid, mask) -> (cand[N_BINS, sel, 5], num_hull[N_BINS])`` for a handle with selectedAction = sel."""
    from oracle.oracle_env import OracleConfig, convex_hull_actions, select_candidates
    pv, mk = spill_inputs()
    cand, nh = run_hulls(pv, mk)
    cfg = OracleConfig(ZRotNum=R, selectedAction=sel)
    for i in range(N_BINS):
        hull = convex_hull_actions(pv[i], mk[i], cfg.resolutionZ, "port")
        assert nh[i] == len(hull) == int(mk[i].sum()), i
        assert np.array_equal(cand[i], select_candidates(cfg, hull, pv[i], mk[i])), (sel, i)
    assert list(nh) == [1024, 1024, 768, 769]


def _cube_library():
    from irbpp_b200 import shapes
    return shapes.make_cube_library(seed=1, num_rotations=R, num_shapes=4)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emulated(str(tmp_path_factory.mktemp("emu_spill")))


@pytest.mark.timeout(900)
def test_emulated_narrow_shape_list_spill(emu):
    for sel in SELS:
        env = EmuEnv(emu, _cube_library(), np.zeros((N_BINS, 8), np.int32), selected_action=sel)

        def run(pv, mk):
            cand, nh = np.zeros((N_BINS, sel, 5)), np.zeros(N_BINS, np.int32)
            pv, mk = np.ascontiguousarray(pv), np.ascontiguousarray(mk)
            assert emu.emu_irbpp_debug_hulls(env.h, _P(pv), _P(mk), _P(cand), _P(nh)) == 0
            return cand, nh
        check_spill(run, sel)
        env.close()


@pytest.mark.gpu
def test_narrow_shape_list_spill_on_device():
    from irbpp_b200.vec_env import GpuVecEnv
    for sel in SELS:
        env = GpuVecEnv(_cube_library(), np.zeros((N_BINS, 8), np.int32), device="cuda:0", selected_action=sel)

        def run(pv, mk):
            out = env.debug_hulls(pv, mk)
            return out["cand"], out["num_hull"]
        check_spill(run, sel)
        env.close()
