"""The per-entry bound of the point-MLP layer checks (tc_mlp_emul.py) has teeth: on a synthetic two-tile batch (101
points of the adversarial KITTI case, the second tile ragged) emulated in float32, the bound accepts the fault-free
accumulators and rejects each injected fault by at least a factor of 10.  No GPU needed."""
import numpy as np
import pytest
import torch

import tc_mlp_emul as E
from cases import PREDICT_CASES, load_golden, params_for, pyramid_for
from oracle import scenerf_oracle as orc

N_PTS, N_ROWS = 101, 128
MIN_FACTOR = 10.0


def _setup(split, h16):
    cfg, seed = PREDICT_CASES["predict_adversarial_kitti"]
    g = load_golden("predict_adversarial_kitti")
    params = params_for(cfg)[0]
    pts = g["cam_pts"].reshape(-1, 3)[:N_PTS].astype(np.float32)
    vd = np.repeat(g["viewdir"], 8, axis=0)[:N_PTS].astype(np.float32)
    coords = g["sphere"][:N_PTS].astype(np.int64)
    pyr = pyramid_for(cfg, seed)
    z = np.zeros((N_ROWS, 2480), dtype=np.float32)
    z[:N_PTS] = orc.gather_latent(pyr, coords, cfg.sphere_W, cfg.sphere_H)
    x32 = torch.from_numpy(E.x_values(pts, vd, N_ROWS))
    z32 = torch.from_numpy(z)
    scale = E.split_scale(params) if split else 1.0
    hdr = E.expected_header(params, 4, scale, "cpu")
    W = E.weight_operands(params, split, scale, "cpu")
    W32 = {}
    for k, v in params.items():
        if k.endswith("weight"):
            w = torch.from_numpy(np.asarray(v, dtype=np.float32)) * scale
            hi = E.rn16(w)
            W32[k] = (hi, E.rn16(w - hi) if split else torch.zeros_like(hi))
    # a wrong granule: channels 80..87 (scale 1/2, inside lin_z chunk 1) sampled with the geometry of scale 1/1
    z_bad = z.copy()
    z_bad[:N_PTS, 80:88] = orc.sample_feats_2d(pyr["1_2"][:8], coords, (cfg.sphere_W, cfg.sphere_H))
    # latent-table rows for the table variant: lin_z[b](z) + c_b in float32
    z64 = torch.from_numpy(z).double()
    tab = torch.stack([(z64 @ torch.from_numpy(params["lin_z.%d.weight" % b]).double().T).float() + hdr[b] for b in range(3)], 1)
    return dict(x32=x32, z32=z32, z_bad=torch.from_numpy(z_bad), hdr=hdr, W=W, W32=W32, split=split, h16=h16, tab=tab)


_CACHE = {}


def _case(split, h16):
    if (split, h16) not in _CACHE:
        _CACHE[(split, h16)] = _setup(split, h16)
    return _CACHE[(split, h16)]


def _worst(c, dumps, tab=None):
    res = E.check_layers(dumps, c["hdr"], c["x32"], c["z32"], c["W"], c["split"], c["h16"], kz=39, tab=tab)
    return {L: w for L, (w, _) in res.items()}


@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("split,h16", [(False, True), (False, False), (True, False)])
def test_bound_accepts_the_fault_free_tile(split, h16, table):
    c = _case(split, h16)
    tab = c["tab"] if table else None
    worst = _worst(c, E.emulate_tile(c["x32"], c["z32"], c["W32"], c["hdr"], split, h16, tab=tab), tab)
    print("fault-free split=%s h16=%s table=%s: worst err/bound per layer %s"
          % (split, h16, table, {L: "%.3g" % v for L, v in worst.items()}))
    assert max(worst.values()) <= 1.0


# (fault, precision mode, fp16 hidden state, layer whose check must reject it)
FAULTS = [
    ("dropped_kstep", False, True, 1),        # one 16-wide k-step of lin_z chunk 5 missing
    ("no_lo_weights", True, False, 1),        # split mode without its lo weight images (table variant: layer 1 is
                                              # lin_in alone, K = 64, where the bound is tight enough to see it)
    ("pbuf_lost", True, False, 5),            # first K half of an fc layer lost
    ("pbuf_twice", True, False, 5),           # ... or added twice
    ("ragged_shift", False, True, 1),         # rows of the ragged tile shifted by one
    ("ragged_shift", True, False, 1),
    ("wrong_granule", False, True, 1),        # granule 80..87 read with another scale's geometry
    ("wrong_granule", True, False, 1),
    ("h_fp16", False, False, 5),              # h rounded to fp16 in the fp32-hidden variant
    ("wrong_bias", False, True, 7),           # E2 of block 1 reads the bias row of the next block
    ("wrong_bias", True, False, 7),
]


@pytest.mark.parametrize("fault,split,h16,layer", FAULTS)
def test_bound_rejects_fault(fault, split, h16, layer):
    c = _case(split, h16)
    z_in = c["z_bad"] if fault == "wrong_granule" else c["z32"]
    defect = None if fault in ("ragged_shift", "wrong_granule") else fault
    tab = c["tab"] if fault == "no_lo_weights" else None
    dumps = E.emulate_tile(c["x32"], z_in, c["W32"], c["hdr"], split, h16, defect=defect, tab=tab)
    if fault == "ragged_shift":
        dumps[1] = dumps[1].clone()
        dumps[1][64:N_PTS - 1] = dumps[1][65:N_PTS].clone()
    worst = _worst(c, dumps, tab)
    print("%s split=%s h16=%s: rejected by a factor of %.3g at layer %d (worst err/bound per layer %s)"
          % (fault, split, h16, worst[layer], layer, {L: "%.3g" % v for L, v in worst.items()}))
    assert worst[layer] >= MIN_FACTOR
