"""``irbpp_dqn_act`` over the whole range its C ABI supports, under the host emulator, against the float64 port.

``tests/test_actor.py`` checks the kernels on the quantized fixture network (whose weights have at most 8 significant
bits, so the low half of the 3xTF32 split of most weights is zero) at 31 atoms, with column 4 of the observation as
the mask.  Here every case uses a seeded ``DQNPort`` with full float32 mantissas, in train mode, in eval mode and after
``reset_noise()``, and drives every argument of ``irbpp_dqn_act``:

* ``atoms`` in 1, 2, 8, 31, 32 with a support that is neither symmetric nor evenly spaced;
* ``selected_action`` in 1, 31, 32, 33, 64, 65, 500, 1000 and, per bin, ``n_valid`` at the edges of the 64-row tiles
  and the 32-row ballot rounds of the row list;
* exact ties (at one atom every row's expected value is exactly ``support[0]``): the first row whose mask is 1 is
  taken, the first row of all when nothing is masked;
* a mask of its own that differs from column 4 (column 4 zeroes embeddings, the mask sets ``-inf``);
* an ``obs_stride`` wider than the row, and ``sum_q_map = NULL``.

The emulator restates ``cvt.rna`` and ``mma.sync`` deterministically, so the emulated kernels are held to their own bar,
``EMU_RTOL`` on ``|q - q64| / (1 + |q64|)``, besides the accuracy contract of ``test_actor.check_contract``.  Measured
on these cases: the committed kernels reach at most 4.2e-7 (atoms 2, eval mode); builds with one product of the
3xTF32 split deleted from ``ac_layer`` reach at least 3.3e-5 (``a_lo . b_hi`` deleted) and 1.5e-5 (``a_hi . b_lo``
deleted, the weights' low half) on the mutant case, in eval mode (5.9e-5 and 4.2e-5 in train mode).
``EMU_RTOL = 3e-6`` sits 7x above the first and 5x below the smallest mutant error.
The mutant tests rebuild the emulated library with such an edit, and with the argmax's tie rule reversed, and require
the named check to fail."""
import copy
import ctypes
import os
import shutil

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.dqn_port import DQNPort
from test_actor import SEL, check_contract, decode_fixture, small_sel

pytestmark = pytest.mark.timeout(900)

EMU_RTOL = 3e-6
ATOMS = (1, 2, 8, 31, 32)
SELS = (1, 31, 32, 33, 64, 65, 500, 1000)
TILE_EDGES = (0, 1, 63, 64, 65, 128, 129)          # 64-row tiles of the rows kernel
MODES = ("train", "eval", "reset_noise")
# first valid rows of the tie cases: each of the eight warps of the final phase (warp = row % 8), and rows in later
# 64-row blocks up to 447
TIE_FIRSTS = (0, 9, 18, 27, 36, 45, 54, 63, 77, 130, 200, 447)
TIE_AFTER = (1, 3, 8, 16, 50)                        # later valid rows: same warp (+8, +16) and other warps


@pytest.fixture(scope="module")
def fx():
    return decode_fixture(load_golden("dqn_act"))


def emulated_library(tmp):
    from irbpp_b200._lib import SIGNATURES
    from test_kernels_emulated import build_emulated
    lib = build_emulated(tmp)
    for name in ("irbpp_dqn_act", "irbpp_dqn_scratch_bytes"):
        fn = getattr(lib, "emu_" + name)
        fn.restype, fn.argtypes = SIGNATURES[name]
    return lib


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return emulated_library(str(tmp_path_factory.mktemp("emu_actor_range")))


# ---- inputs ----

def support_for(atoms):
    """Increasing atom values, unevenly spaced, from -7 to 10 (one atom: 2.5)."""
    if atoms == 1:
        return np.array([2.5], np.float32)
    s = np.cumsum(np.random.default_rng(atoms).uniform(0.3, 1.0, atoms))
    return (-7.0 + 17.0 * (s - s[0]) / (s[-1] - s[0])).astype(np.float32)


def seeded_net(sel, atoms, mode, seed=5):
    """The reference's initialisation (full float32 mantissas) in train mode, eval mode, or train mode after a second
    ``reset_noise()``."""
    torch.manual_seed(seed)
    net = DQNPort(selected_action=sel, atoms=atoms)
    if mode == "reset_noise":
        net.reset_noise()
    return net.train(mode != "eval")


def make_bins(fx, sel, n_valid, seed=0):
    """One observation of ``sel`` candidate rows per entry of ``n_valid``, from the fixture's truncated irregular bins
    (all their 500 rows are real candidates; heightmap and item vector kept): their first ``sel`` rows, for
    ``sel > 500`` followed by synthetic rows ``[rot, x, y, H]`` in the observation's ranges; column 4 marks
    ``n_valid[i]`` rows chosen at random.  Returns the observations and the fixture bin of each."""
    rng = np.random.default_rng(seed)
    N = len(n_valid)
    src = np.nonzero(fx["kinds"] == 1)[0]
    src = src[np.arange(N) % len(src)]
    obs = small_sel(fx["obs"][src], min(sel, SEL))
    if sel > SEL:
        extra = np.zeros((N, sel - SEL, 5), np.float32)
        extra[:, :, 0] = rng.integers(0, 24, (N, sel - SEL))
        extra[:, :, 1:3] = rng.integers(0, 16, (N, sel - SEL, 2))
        extra[:, :, 3] = rng.uniform(0.0, 0.3, (N, sel - SEL))
        obs = np.concatenate([obs[:, :SEL * 5], extra.reshape(N, -1), obs[:, SEL * 5:]], axis=1)
    rank = rng.random((N, sel)).argsort(1).argsort(1)
    obs[:, np.arange(sel) * 5 + 4] = rank < np.asarray(n_valid)[:, None]
    return np.ascontiguousarray(obs, np.float32), src


def tie_bins(fx, sel, firsts):
    """Bins whose valid rows are ``first`` and the rows ``TIE_AFTER`` past it that fit in ``sel``."""
    obs, src = make_bins(fx, sel, [0] * len(firsts))
    for b, r in enumerate(firsts):
        for s in (0,) + TIE_AFTER:
            if r + s < sel:
                obs[b, (r + s) * 5 + 4] = 1.0
    return obs, src


def shape_features(fx, net32, src):
    """shape_feature of the fixture bins' items (model.py:330-335, the fixture's point indices), float32, on the
    network's device."""
    items, inv = np.unique(fx["obs"][src, SEL * 5].astype(np.int64), return_inverse=True)
    pts = torch.tensor(fx["shape_array"][items][:, fx["point_indices"]], device=next(net32.parameters()).device)
    with torch.no_grad():
        return net32.shape_feature(pts)[torch.from_numpy(inv.reshape(-1)).to(pts.device)]


def col4(obs, sel):
    """Column 4 of the candidate rows as a strided view (element stride 5), as get_mask_from_state returns it."""
    return obs[:, 4:sel * 5:5]


def to_np(a):
    return a.cpu().numpy() if isinstance(a, torch.Tensor) else np.array(a)


def mask_apart_from_col4(c4, seed):
    """A float32 mask that differs from column 4: half of each bin's rows with column 4 == 1 masked out, up to 10 rows
    with column 4 == 0 let through."""
    rng = np.random.default_rng(seed)
    mask = np.array(c4, np.float32)
    for b in range(mask.shape[0]):
        on, off = np.nonzero(c4[b] == 1)[0], np.nonzero(c4[b] != 1)[0]
        mask[b, rng.choice(on, len(on) // 2, replace=False)] = 0.0
        mask[b, rng.choice(off, min(10, len(off)), replace=False)] = 1.0
    return mask


# ---- the call and the reference ----

def _addr(a):
    return a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data


def _strides(a):
    return tuple(a.stride()) if isinstance(a, torch.Tensor) else tuple(s // a.itemsize for s in a.strides)


def dqn_act(lib, net32, obs, sel, sf, support, mask=None, want_q=True, prefix="emu_"):
    """``irbpp_dqn_act`` with every argument explicit.  ``obs``: [N, >= sel*5 + 9 + 1024] with element stride 1, its
    row stride passed as ``obs_stride``; ``mask``: None (no masking) or a float32 [N, sel] array whose own row and
    element strides are passed; ``want_q=False`` passes ``sum_q_map = NULL``.  NumPy arrays for the emulated library
    (host == device there), CUDA tensors for the real one (``prefix=""``).  Weights: the port's effective weights in
    its mode, float32.  Returns (actions, q or None) as NumPy arrays."""
    from irbpp_b200._lib import IrbppDqnWeights
    from irbpp_b200.actor import _FIELDS, NOISY
    dev = obs.device if isinstance(obs, torch.Tensor) else None
    sd = net32.state_dict()
    eff = {k: sd[k] for _, k in _FIELDS if k in sd}
    with torch.no_grad():
        for m in NOISY:
            eff[m + ".weight"], eff[m + ".bias"] = getattr(net32, m).effective()
    if dev is None:
        keep = {f: np.ascontiguousarray(eff[k].detach().cpu().numpy(), np.float32) for f, k in _FIELDS}
        sf, support = np.ascontiguousarray(sf, np.float32), np.ascontiguousarray(support, np.float32)
    else:
        keep = {f: eff[k].detach().to(dev, torch.float32).contiguous() for f, k in _FIELDS}
        sf, support = sf.to(dev, torch.float32).contiguous(), support.to(dev, torch.float32).contiguous()
    w = IrbppDqnWeights(*([_addr(keep[f]) for f, _ in _FIELDS] + [ctypes.c_float(0.01)]))
    assert _strides(obs)[1] == 1
    N = obs.shape[0]
    nbytes = getattr(lib, prefix + "irbpp_dqn_scratch_bytes")(N, sel)
    if dev is None:
        raw = np.zeros(nbytes + 256, np.uint8)
        scratch = raw.ctypes.data + (-raw.ctypes.data) % 256
        actions = np.full(N, -1, np.int64)
        q = np.full((N, sel), np.nan, np.float32) if want_q else None
        stream = None
    else:
        raw = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        scratch = raw.data_ptr() + (-raw.data_ptr()) % 256
        actions = torch.full((N,), -1, dtype=torch.int64, device=dev)
        q = torch.full((N, sel), float("nan"), device=dev) if want_q else None
        stream = torch.cuda.current_stream(dev).cuda_stream
    m_row, m_elem = _strides(mask) if mask is not None else (0, 0)
    rc = getattr(lib, prefix + "irbpp_dqn_act")(
        ctypes.byref(w), _addr(obs), _strides(obs)[0], N, sel, _addr(sf), _addr(support), len(support),
        _addr(mask) if mask is not None else None, m_row, m_elem, _addr(actions), _addr(q) if want_q else None,
        scratch, nbytes, stream)
    assert rc == 0, rc
    if dev is not None:
        torch.cuda.synchronize(dev)
        actions, q = actions.cpu(), q.cpu() if want_q else None
    return np.asarray(actions), (np.asarray(q) if want_q else None)


def port_q(net32, obs, sf, support, mask=None, chunk=128):
    """The float64 port's expected values (``-inf`` where ``mask != 1``) from the same parameters, in chunks of bins,
    on the device the inputs live on."""
    t = lambda a: (a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(a))).double()
    obs, sf, support = t(obs), t(sf), t(support)
    net64 = copy.deepcopy(net32).to(obs.device, torch.float64)
    mask = None if mask is None else t(mask)
    out = []
    with torch.no_grad():
        for i in range(0, obs.shape[0], chunk):
            out.append(net64.sum_q(obs[i:i + chunk], sf[i:i + chunk], support,
                                   None if mask is None else mask[i:i + chunk]).cpu())
    return torch.cat(out).numpy()


def scaled_error(q, q64):
    fin = np.isfinite(q64)
    return float((np.abs(q[fin] - q64[fin]) / (1 + np.abs(q64[fin]))).max()) if fin.any() else 0.0


def emu_contract(q, q64, act, mask):
    """The accuracy contract, then EMU_RTOL; returns the largest scaled error."""
    worst = check_contract(q, q64, act, mask)
    assert worst <= EMU_RTOL, "largest |q - q64| / (1 + |q64|) = %.3g > EMU_RTOL" % worst
    return worst


def masked(q64, mask):
    return np.where(np.asarray(mask) == 1, q64, -np.inf)


# ---- the cases, shared with the mutant builds ----

def run_range_case(lib, fx, sel, atoms, mode, n_valid, use_mask):
    """Bins with the given n_valid through the kernels; mask: column 4 as a strided view, or none.  Returns
    (q, q64, actions, mask)."""
    net = seeded_net(sel, atoms, mode)
    obs, src = make_bins(fx, sel, n_valid, seed=sel * 37 + atoms)
    sf = shape_features(fx, net, src)
    support = support_for(atoms)
    mask = col4(obs, sel) if use_mask else None
    act, q = dqn_act(lib, net, obs, sel, sf, support, mask)
    q64 = port_q(net, obs, sf, support)
    if use_mask:
        q64 = masked(q64, mask)
    return q, q64, act, None if mask is None else np.array(mask)


def check_ties(lib, fx, sel, firsts, use_mask, device=None, prefix="emu_"):
    """One atom: every row's expected value is exactly support[0] (softmax of one logit is 1), so every valid row
    ties.  The action is the first row whose mask is 1 (masked), or row 0 (unmasked)."""
    net = seeded_net(sel, 1, "train")
    obs, src = tie_bins(fx, sel, firsts)
    sf = shape_features(fx, net, src)
    support = support_for(1)
    want = np.where(col4(obs, sel) == 1, support[0], -np.inf) if use_mask else np.full((len(firsts), sel), support[0])
    if device is not None:
        obs, support, sf = torch.tensor(obs, device=device), torch.tensor(support, device=device), sf.to(device)
    mask = col4(obs, sel) if use_mask else None
    act, q = dqn_act(lib, net, obs, sel, sf, support, mask, prefix=prefix)
    q64 = port_q(net, obs, sf, support, mask)
    assert np.array_equal(q64, want) and np.array_equal(q, want)
    assert act.tolist() == (list(firsts) if use_mask else [0] * len(firsts)), act


# ---- the supported range ----

@pytest.mark.parametrize("atoms", ATOMS)
def test_every_atom_count(fx, emu, atoms):
    """Every atom count at sel 65 over the tile edges that fit (0, 1, 63, 64, 65), unmasked: every row's q, the a0
    rows included, against the port."""
    i = ATOMS.index(atoms)
    edges = [n for n in TILE_EDGES if n <= 65]
    n_valid = [edges[i % len(edges)], edges[(i + 2) % len(edges)]]
    q, q64, act, _ = run_range_case(emu, fx, 65, atoms, MODES[i % 3], n_valid, use_mask=False)
    worst = emu_contract(q, q64, act, None)
    print("atoms %d, n_valid %s, %s: largest scaled error %.3g" % (atoms, n_valid, MODES[i % 3], worst))


SEL_CASES = {1: (1, 0), 31: (1, 31), 32: (32, 1), 33: (33, 32), 64: (63, 64), 65: (64, 65), 500: (128, 129),
             1000: (129, 1)}


@pytest.mark.parametrize("sel", SELS)
def test_every_selected_action(fx, emu, sel):
    """Every selected_action at 31 atoms with the mask as column 4's strided view; n_valid at the row-list edges
    (32-row ballot rounds, 64-row tiles, all rows)."""
    i = SELS.index(sel)
    n_valid = list(SEL_CASES[sel])
    use_mask = sel != 1                      # sel 1, n_valid 0 unmasked: a bin of one a0 row
    q, q64, act, mask = run_range_case(emu, fx, sel, 31, MODES[i % 3], n_valid, use_mask)
    worst = emu_contract(q, q64, act, mask)
    print("sel %d, n_valid %s, %s: largest scaled error %.3g" % (sel, n_valid, MODES[i % 3], worst))


# ---- exact ties ----

def test_ties_take_the_first_row(fx, emu):
    check_ties(emu, fx, SEL, TIE_FIRSTS, use_mask=True)
    check_ties(emu, fx, SEL, TIE_FIRSTS[:3], use_mask=False)


# ---- the mask's own role and strides ----

def test_mask_apart_from_column_4(fx, emu):
    """mask (contiguous float32, element stride 1) differs from column 4: rows with column 4 == 1 masked out, rows with
    column 4 == 0 let through with the advantage of a zeroed embedding (a0).  The port applies the two as the
    reference does: column 4 in the embedding, the mask in agent.py:56-57."""
    sel = 65
    net = seeded_net(sel, 31, "train")
    obs, src = make_bins(fx, sel, [40, 20, 0], seed=3)
    sf = shape_features(fx, net, src)
    support = support_for(31)
    c4 = np.array(col4(obs, sel))
    mask = mask_apart_from_col4(c4, seed=4)
    let_through = (mask == 1) & (c4 == 0)
    assert let_through.any() and ((mask == 0) & (c4 == 1)).any()
    act, q = dqn_act(emu, net, obs, sel, sf, support, mask)
    q64 = port_q(net, obs, sf, support, mask)
    assert np.isfinite(q[let_through]).all()
    worst = emu_contract(q, q64, act, mask)
    print("separate mask: largest scaled error %.3g" % worst)


def test_wide_obs_stride_and_no_sum_q(fx, emu):
    """Rows taken as a column slice of a wider buffer (NaN around them), so obs_stride > sel*5 + 9 + 1024; the mask as
    column 4 of that slice.  The action without sum_q_map equals the action with it, masked and unmasked."""
    sel = 33
    net = seeded_net(sel, 31, "eval")
    obs, src = make_bins(fx, sel, [33, 20], seed=5)
    wide = np.full((obs.shape[0], obs.shape[1] + 44), np.nan, np.float32)
    wide[:, 3:3 + obs.shape[1]] = obs
    view = wide[:, 3:3 + obs.shape[1]]
    sf = shape_features(fx, net, src)
    support = support_for(31)
    q64 = port_q(net, obs, sf, support)
    for mask in (col4(view, sel), None):
        act, q = dqn_act(emu, net, view, sel, sf, support, mask)
        want = q64 if mask is None else masked(q64, mask)
        worst = emu_contract(q, want, act, None if mask is None else np.array(mask))
        act_only, none = dqn_act(emu, net, view, sel, sf, support, mask, want_q=False)
        assert none is None and np.array_equal(act_only, act), (act_only, act)
        print("obs_stride %d, masked %s: largest scaled error %.3g" % (wide.shape[1], mask is not None, worst))


# ---- mutant builds: the checks above have teeth ----

MUTANT_CASE = dict(sel=64, atoms=31, n_valid=(64, 63))
MUTANTS = {
    "no_a_lo_b_hi": ("ac_mma(acc[i][j], al[i], bh);", ""),
    "no_a_hi_b_lo": ("ac_mma(acc[i][j], ah[i], bl);", ""),
    "ties_take_the_last_row": ("r < bidx", "r > bidx"),
}


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_mutant_fails(fx, tmp_path, monkeypatch, name):
    """ac_layer without one product of the 3xTF32 split exceeds EMU_RTOL; the in-warp argmax with the tie rule
    reversed fails the tie assertions."""
    import test_kernels_emulated
    old, new = MUTANTS[name]
    csrc = str(tmp_path / "csrc")
    shutil.copytree(test_kernels_emulated.CSRC, csrc, ignore=shutil.ignore_patterns("__pycache__"))
    path = os.path.join(csrc, "irbpp_actor.cuh")
    text = open(path).read()
    assert text.count(old) == 1, "the text %r to mutate is not in irbpp_actor.cuh once" % old
    open(path, "w").write(text.replace(old, new))
    monkeypatch.setattr(test_kernels_emulated, "CSRC", csrc)
    lib = emulated_library(str(tmp_path / "build"))
    if name.startswith("ties"):
        with pytest.raises(AssertionError):
            check_ties(lib, fx, MUTANT_CASE["sel"], (0, 13, 27, 46), use_mask=True)
        with pytest.raises(AssertionError):
            check_ties(lib, fx, MUTANT_CASE["sel"], (0, 13), use_mask=False)
        return
    for mode in ("train", "eval"):
        q, q64, act, _ = run_range_case(lib, fx, MUTANT_CASE["sel"], MUTANT_CASE["atoms"], mode,
                                        MUTANT_CASE["n_valid"], use_mask=False)
        print("mutant %s, %s: largest scaled error %.3g" % (name, mode, scaled_error(q, q64)))
        with pytest.raises(AssertionError):
            emu_contract(q, q64, act, None)
