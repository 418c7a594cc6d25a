"""Chain-cut emulation of the tensor-core point-MLP tile program (csrc/mlp_tc.cu) and its per-entry error bound.

Each layer L is checked on the operands the kernel really used.  Its A operand is rebuilt in float32 from the dumped
accumulators of the layers before it (srf_debug_tc_layer; the kernel is deterministic, so dumps from separate
launches are consistent) by replaying the epilogue in the kernel's order (`finish`):
    r = acc (split: the dump already holds both K halves) ; r *= inv_scale (split) ; r += bias (unless a latent-table
    row is added) ; r += h (fp16-rounded in the fp16-hidden variant) ; r += table row ; store h ;
    A = rn16(relu r), split: hi = rn16(relu r), lo = rn16(relu r - hi)
so the reference of layer L carries no drift from the layers before it.  For entry (i, j) of layer L:

    |got - ref| <= ACC_C m_L 2^-24 S   (+ 2^-24 |ref|: split fc layers, the add of their two K halves)
                                       (+ x allowance: layer 1)

ref = sum_k a_k w_k and S = sum_k |a_k| |w_k|, both float64 over the fp16 operands (split mode: over all four hi/lo
products; every product of fp16 values is exact in float64), m_L = number of 8-wide k-groups that land in the
accumulator: K_pad / 8, times 4 in split mode (four MMAs per k-step).  ACC_C is the wgmma accumulation constant of
helpers.TF32_ACC_C: one truncating float32 rounding per 8 products, the conservative reading for the fp16 k16 MMA.
Measured by test_gpu_tc_layers.py / test_gpu_fp32tc.py on an H100 80GB HBM3 (700 W power limit), worst err/bound
over all shapes and both networks, layers 1 2 4 5 7 8 9 10:
    fp16, fp16 hidden state    0.104 0.056 0.064 0.062 0.063 0.058 0.058 0.035   (+ table: 0.076 ... <= 0.060)
    fp16, fp32 hidden state    0.104 0.056 0.064 0.054 0.063 0.065 0.058 0.036   (+ table: 0.076 ... <= 0.067)
    split                      0.128 0.021 0.028 0.021 0.028 0.020 0.018 0.024   (+ table: 0.337 ... <= 0.024)
Layer 1 of the table variants is lin_in alone (K = 64, the smallest accumulation term of any layer).
The latent table (test_gpu_preproj.py) measured at most 0.044 of its bound.

The functions take torch tensors on any device (float64 matmuls on the GPU keep the large cases fast)."""
import math

import numpy as np
import torch

from helpers import TF32_ACC_C

U = 2.0 ** -24
ACC_C = TF32_ACC_C
HIDDEN = 512
LAYERS = (1, 2, 4, 5, 7, 8, 9, 10)
FC_LAYERS = (2, 4, 5, 7, 8, 9)                  # split mode sums their K in two halves (mlp_tc.cu flush)
SCALE_SLOT, INV_SLOT = 7 * HIDDEN + 256, 7 * HIDDEN + 257
_FC = {2: "blocks.0.fc_0", 4: "blocks.0.fc_1", 5: "blocks.1.fc_0", 7: "blocks.1.fc_1", 8: "blocks.2.fc_0",
       9: "blocks.2.fc_1", 10: "lin_out"}
SIN_COLS = slice(3, 39)                          # the 36 sin columns of x (pe.py order: x, y, z, then sin terms)
# x allowance per sin column (device sinf vs float64 sin):
#   fp16 mode: rn16 of the two can differ by one fp16 ulp, <= 2^-10 |x| (normal) or 2^-24 (subnormal);
#   split mode: sinf is within 2 float32 ulp (<= 2^-22 |x|) and each side's hi + lo misses its float32 value by
#   <= 2^-23 |x| (lo's half ulp) or 2^-25 (subnormal lo): 2^-21 |x| + 2^-24 in all.
X_ALLOW = {False: (2.0 ** -10, 2.0 ** -24), True: (2.0 ** -21, 2.0 ** -24)}


def rn16(t):
    return t.to(torch.float16).to(torch.float32)


def operand(v32, split):
    """float32 values -> (A, |A|) in float64: rn16(v), or in split mode hi + lo with hi = rn16(v), lo = rn16(v - hi)
    (and |hi| + |lo|)."""
    hi = rn16(v32)
    if not split:
        a = hi.double()
        return a, a.abs()
    lo = rn16(v32 - hi)
    return hi.double() + lo.double(), hi.double().abs() + lo.double().abs()


def weight_operands(params, split, scale, device):
    """state-dict weights -> name -> (W, |W|) float64 as packed: rn16(W), split mode hi/lo of W 2^s (exact scaling)."""
    out = {}
    for k, v in params.items():
        if k.endswith("weight"):
            w = torch.as_tensor(np.asarray(v, dtype=np.float32), device=device)
            out[k] = operand(w * scale if split else w, split)
    return out


def split_scale(params):
    """2^s with max|W| 2^s in [2^13, 2^14) (mlp_tc.cu weight_scale_kernel)."""
    m = max(float(np.abs(v).max()) for k, v in params.items() if k.endswith("weight"))
    return 2.0 ** (14 - math.frexp(m)[1])


def expected_header(params, d_out, scale, device):
    """The 8 x 512 float32 bias header of a packed blob (mlp_tc.cu pack_header_kernel + the scale slots)."""
    f = lambda k: torch.as_tensor(np.asarray(params[k], dtype=np.float32), device=device)
    h = torch.zeros(8, HIDDEN, dtype=torch.float32, device=device)
    h[0] = f("lin_in.bias") + f("lin_z.0.bias")
    h[1] = f("blocks.0.fc_1.bias") + f("lin_z.1.bias")
    h[2] = f("blocks.1.fc_1.bias") + f("lin_z.2.bias")
    for b in range(3):
        h[3 + b] = f("blocks.%d.fc_0.bias" % b)
    h[6] = f("blocks.2.fc_1.bias")
    h[7, :d_out] = f("lin_out.bias")
    h.view(-1)[SCALE_SLOT] = scale
    h.view(-1)[INV_SLOT] = 1.0 / scale
    return h


def blob_header(blob):
    return blob[:8 * HIDDEN * 4].view(torch.float32).reshape(8, HIDDEN).clone()


def x_values(pts, vd_rows, n_rows):
    """(n_rows, 42) float32 x operand: the point, its 36 sin terms and the view direction; rows >= len(pts) are 0.
    The sin argument is the kernel's float32 fmul(x, pi 2^k) (+ pi/2), the sine is float64."""
    f32 = np.float32
    n = pts.shape[0]
    x = np.zeros((n_rows, 42), dtype=f32)
    x[:n, :3] = pts
    k_pi, k_half_pi = f32(3.14159274101257324), f32(1.57079637050628662)
    for fp in range(12):
        for cc in range(3):
            arg = (pts[:, cc].astype(f32) * f32(k_pi * f32(1 << (fp >> 1)))).astype(f32)
            if fp & 1:
                arg = (k_half_pi + arg).astype(f32)
            x[:n, 3 + 3 * fp + cc] = np.sin(arg.astype(np.float64)).astype(f32)
    x[:n, 39:42] = vd_rows
    return x


def layer_terms(L, pre):
    """(A operand, weight) pairs accumulated into layer L's accumulator: lin_z passes are absent in table variants."""
    t = [("x", "lin_in")] if L == 1 else [("act", _FC[L])]
    if not pre and L in (1, 4, 7):
        t.append(("z", "lin_z.%d" % ((L - 1) // 3)))
    return t


def finish(acc, hdr, idx, split, h=None, tab=None):
    """The epilogue's float32 sum r for bias row idx (mlp_tc.cu finish): tab is the (rows, 3, 512) table-row block."""
    r = acc.clone()
    if split:
        r = r * hdr.view(-1)[INV_SLOT]
    if tab is None:
        r = r + hdr[idx]
    if h is not None:
        r = r + h
    if tab is not None:
        r = r + tab[:, idx]
    return r


def replay(dumps, hdr, split, h16, tab=None):
    """float32 replay of E1/E2/E3 on the dumped accumulators: L -> the pre-ReLU r whose relu is layer L's A operand."""
    store = rn16 if h16 else (lambda v: v)
    A = {}
    r = finish(dumps[1], hdr, 0, split, tab=tab)
    h = store(r)
    A[2] = r
    for b in range(3):
        A[4 + 3 * b if b < 2 else 9] = finish(dumps[2 + 3 * b], hdr, 3 + b, split)
        if b < 2:
            r = finish(dumps[4 + 3 * b], hdr, b + 1, split, h=h, tab=tab)
            h = store(r)
            A[5 + 3 * b] = r
        else:
            A[10] = finish(dumps[9], hdr, 6, split, h=h)
    return A


def layer_bound(L, ops, W, split, kz, pre):
    """(ref, bound) float64 of layer L: ops maps 'x' / 'z' / 'act' to (A, |A|), W the weight operands."""
    ref = S = 0.0
    kpad = 0
    for name, wname in layer_terms(L, pre):
        a, aa = ops[name]
        w, wa = W[wname + ".weight"]
        ref = ref + a @ w.T
        S = S + aa @ wa.T
        kpad += {"x": 64, "act": HIDDEN, "z": 64 * kz}[name]
    m = kpad // 8 * (4 if split else 1)
    bound = ACC_C * m * U * S
    if split and L in FC_LAYERS:
        bound = bound + U * ref.abs()
    if L == 1:
        u_x, a_x = X_ALLOW[split]
        xs = ops["x_f32"][:, SIN_COLS].double().abs()
        bound = bound + (u_x * xs + a_x) @ W["lin_in.weight"][1][:, SIN_COLS].T
    return ref, bound


def ratio(got, ref, bound):
    """err / bound per entry (an entry with a zero bound must be exact)."""
    err = (got.double() - ref).abs()
    return torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))


def check_layers(dumps, hdr, x32, z32, W, split, h16, kz, tab=None):
    """Worst err/bound per layer of the dumps (rows = points, float32, only the d_out columns for layer 10).
    x32 / z32: float32 operand values before rounding.  Returns {L: (worst ratio, ratio tensor)}."""
    pre = tab is not None
    ops = {"x": operand(x32, split), "x_f32": x32}
    if not pre:
        ops["z"] = operand(z32, split)
    A = replay(dumps, hdr, split, h16, tab)
    out = {}
    for L in LAYERS:
        if L != 1:
            ops["act"] = operand(torch.relu(A[L]), split)
        ref, bound = layer_bound(L, ops, W, split, kz, pre)
        rt = ratio(dumps[L][:, :ref.shape[1]], ref, bound)
        out[L] = (float(rt.max()), rt)
    return out


def emulate_tile(x32, z32, W32, hdr, split, h16, defect=None, tab=None):
    """A float32 stand-in for the kernel (tests of the bound): every layer's accumulator is a float32 matmul of the
    exact operand values, with the epilogues of `finish`.  W32: name -> (hi, lo) float32 weight images (lo zero in
    fp16 mode); tab: table rows (the table variant: no lin_z passes).  `defect` injects one of the faults the
    per-entry bound must reject."""
    def A_of(v):
        hi = rn16(v)
        return (hi, rn16(v - hi)) if split else (hi, torch.zeros_like(hi))

    def mm(a, wname, L):
        ahi, alo = a
        whi, wlo = W32[wname + ".weight"]
        if defect == "no_lo_weights":
            wlo = torch.zeros_like(wlo)
        aa, ww = ahi + alo, whi + wlo                        # exact in float32 (22 significant bits)
        if L in FC_LAYERS and split:
            h1 = aa[:, :256] @ ww[:, :256].T
            h2 = aa[:, 256:] @ ww[:, 256:].T
            if defect == "pbuf_lost" and L == 5:
                return h2
            if defect == "pbuf_twice" and L == 5:
                return h2 + h1 + h1
            return h2 + h1
        if defect == "dropped_kstep" and wname == "lin_z.0":
            keep = torch.ones(aa.shape[1], dtype=aa.dtype, device=aa.device)
            keep[5 * 64 + 16:5 * 64 + 32] = 0                # the second k16 step of chunk 5
            return (aa * keep) @ ww.T
        return aa @ ww.T

    store = rn16 if h16 else (lambda v: v)
    if defect == "h_fp16":
        store = rn16
    bias_ix = lambda i: (i + 1) % 8 if defect == "wrong_bias" and i == 4 else i
    d = {}
    xa, za = A_of(x32), A_of(z32)
    lin_z = (lambda b, L: 0.0) if tab is not None else (lambda b, L: mm(za, "lin_z.%d" % b, L))
    d[1] = mm(xa, "lin_in", 1) + lin_z(0, 1)
    r = finish(d[1], hdr, 0, split, tab=tab)
    h = store(r)
    for b in range(3):
        d[2 + 3 * b] = mm(A_of(torch.relu(r)), _FC[2 + 3 * b], 2 + 3 * b)
        net = finish(d[2 + 3 * b], hdr, bias_ix(3 + b), split)
        Lf = 4 + 3 * b if b < 2 else 9
        acc = mm(A_of(torch.relu(net)), _FC[Lf], Lf)
        if b < 2:
            d[Lf] = acc + lin_z(b + 1, Lf)
            r = finish(d[Lf], hdr, b + 1, split, h=h, tab=tab)
            h = store(r)
        else:
            d[9] = acc
            r = finish(d[9], hdr, 6, split, h=h)
    d[10] = mm(A_of(torch.relu(r)), "lin_out", 10)
    return d


# ---------------------------------------------------------------------------------------------------------------
# Device side: dumps of the kernel, their contract, and the per-entry check of one variant
# ---------------------------------------------------------------------------------------------------------------
SPHERE_INVALID = -(1 << 28)          # common.cuh kSphereInvalid: the sphere coordinate of a padded row
NAN_BITS = 0x7FC00000                # torch.full(nan)


def dump_rows(n, split):
    """Rows of the debug buffer and the rows the kernel writes for points (fp16: every row of every tile)."""
    if split:
        i = torch.arange(n)
        return (n + 31) // 32 * 64, 64 * (i // 32) + i % 32
    rows = (n + 63) // 64 * 64
    return rows, torch.arange(rows)


def dump_layers(r, which, pts_t, x_rgb, K, vd_t, n):
    rows, _ = dump_rows(n, r.precision == "fp32tc")
    out = {}
    for L in LAYERS:
        buf = torch.full((rows, HIDDEN), float("nan"), dtype=torch.float32, device=r.device)
        r.debug_tc_layer(which, pts_t, x_rgb, K, vd_t, L, out=buf)
        out[L] = buf
    torch.cuda.synchronize()
    return out


def check_dump_contract(dumps, n, split, d_out):
    """Written rows are finite, every other entry keeps the NaN it was filled with; layer 10 writes columns 0..15 only,
    and columns d_out..15 (zero weight rows) are exactly 0."""
    rows, idx = dump_rows(n, split)
    written = torch.zeros(rows, dtype=torch.bool)
    written[idx] = True
    written = written.to(dumps[1].device)
    for L, d in dumps.items():
        cols = 16 if L == 10 else HIDDEN
        assert torch.isfinite(d[written, :cols]).all(), "layer %d: a written entry is not finite" % L
        assert (d[~written].view(torch.int32) == NAN_BITS).all(), "layer %d wrote a row it does not own" % L
        if L == 10:
            assert (d[:, 16:].view(torch.int32) == NAN_BITS).all(), "layer 10 wrote beyond column 15"
            assert (d[written, d_out:16] == 0).all(), "layer 10: padded columns d_out..15 are not 0"


def table_of(r, which):
    """(rows, 3, 512) float32 view of a network's latent table in r._tab_buf (main network, then mlp_gaussian)."""
    nbytes = r._tab_buf.numel() // 2
    W1, H1 = r.hp["out_img_W"] + 1, r.hp["out_img_H"] + 1
    n_rows = W1 * H1 + 1
    esize = 2 if r.precision == "fp16" else 4
    base = (0 if which == "mlp" else 1) * nbytes
    raw = r._tab_buf[base:base + n_rows * 3 * HIDDEN * esize]
    return raw.view(torch.float16 if esize == 2 else torch.float32).reshape(n_rows, 3, HIDDEN).float()


def table_index(coords, W1, H1):
    sx, sy = coords[:, 0], coords[:, 1]
    inside = (sx >= 0) & (sx < W1) & (sy >= 0) & (sy < H1)
    return np.where(inside, sy * W1 + sx, W1 * H1)


def check_variant(cfg, seed, prec, which, pts, vd, h16=True, pre=False, skip=False, label=""):
    """Run one tensor-core variant on the points (n_cols, n_per, 3) and check it: the blob header, the dump contract,
    predict's raw output against the lin_out dump (E4, bit for bit) and every dumped layer entry by entry.
    Returns (worst err/bound per layer, dumps, raw output)."""
    from cases import params_for, pyramid_for
    from helpers import make_renderer, torch_pyramid
    from oracle import scenerf_oracle as orc
    split = prec == "fp32tc"
    r = make_renderer(cfg, prec, hidden_fp16=h16, preproject=pre, skip_zero_chunks=skip)
    dev = r.device
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    pts_t, vd_t = torch.from_numpy(pts), torch.from_numpy(vd)
    n_cols, n_per = pts.shape[:2]
    n = n_cols * n_per
    raw, dbg = r.predict(which, pts_t, x_rgb, K, None, vd_t, output_type="offset", debug=True)
    net = r.mlp if which == "mlp" else r.mlp_gaussian
    d_out = net.struct.d_out
    params = params_for(cfg)[0 if which == "mlp" else 1]
    scale = split_scale(params) if split else 1.0
    hdr = blob_header(net.packed_split if split else net.packed)
    assert torch.equal(hdr.view(torch.int32), expected_header(params, d_out, scale, dev).view(torch.int32))
    dumps = dump_layers(r, which, pts_t, x_rgb, K, vd_t, n)
    check_dump_contract(dumps, n, split, d_out)
    _, idx = dump_rows(n, split)
    pr = {L: d[idx.to(dev)] for L, d in dumps.items()}
    # E4: out = float32(acc10 * inv) + b_out (fp16 mode: acc10 + b_out), bit for bit
    d10 = pr[10][:n, :d_out]
    want = (d10 * hdr.view(-1)[INV_SLOT] if split else d10) + hdr[7, :d_out]
    assert torch.equal(raw.reshape(n, d_out), want), "predict's raw output is not E4 of the lin_out accumulator"
    n_rows = idx.numel()
    coords = np.full((n_rows, 2), SPHERE_INVALID, dtype=np.int64)
    coords[:n] = dbg.cpu().numpy()
    x32 = torch.from_numpy(x_values(pts.reshape(-1, 3), np.repeat(vd, n_per, axis=0), n_rows)).to(dev)
    z32 = tab = None
    if pre:
        tab = table_of(r, which)[torch.from_numpy(table_index(coords, cfg.sphere_W + 1, cfg.sphere_H + 1)).to(dev)]
    else:
        pyr = pyramid_for(cfg, seed)
        if not split:                  # the fp16 mode gathers from the fp16 pack of the pyramid
            pyr = {k: v.astype(np.float16).astype(np.float32) for k, v in pyr.items()}
        z32 = torch.from_numpy(orc.gather_latent(pyr, coords, cfg.sphere_W, cfg.sphere_H)).to(dev)
    W = weight_operands(params, split, scale, dev)
    kz = (int(params["lin_z.0.weight"].shape[1]) + 63) // 64
    res = check_layers(pr, hdr, x32, z32, W, split, h16 and not split, kz, tab)
    worst = {L: w for L, (w, _) in res.items()}
    print("%s %s %s h16=%s table=%s skip=%s n=%d n_per=%d: worst err/bound %s" % (
        label, prec, which, h16 and not split, pre, skip, n, n_per, " ".join("L%d %.3g" % kv for kv in worst.items())))
    for L, (w, rt) in res.items():
        if w > 1.0:
            i, j = divmod(int(torch.argmax(torch.nan_to_num(rt, posinf=1e300))), rt.shape[1])
            raise AssertionError("%s layer %d: err/bound %.3g at point row %d column %d" % (label, L, w, i, j))
    return worst, dumps, raw


def tap_scales(cfg, pyr, coords):
    """(n, 5) bool: scale s has at least one in-range bilinear tap at the integer sphere coords (float32 tap
    arithmetic of oracle.sample_feats_2d / common.cuh scale_taps)."""
    f32 = np.float32
    out = []
    for s, key in enumerate(("1_1", "1_2", "1_4", "1_8", "1_16")):
        _, H, W = pyr[key].shape
        norm = (cfg.sphere_W // (1 << s), cfg.sphere_H // (1 << s))
        anyv = np.zeros(coords.shape[0], dtype=bool)
        for c, size, nrm in ((0, W, norm[0]), (1, H, norm[1])):
            g = ((coords[:, c].astype(f32) / f32(nrm)).astype(f32) * f32(2) - f32(1)).astype(f32)
            i = ((g + f32(1)) * f32(size / 2.0) - f32(0.5)).astype(f32)
            i0 = np.floor(i).astype(np.int64)
            ok = ((i0 >= 0) & (i0 < size)) | ((i0 + 1 >= 0) & (i0 + 1 < size))
            anyv = ok if c == 0 else (anyv & ok)
        out.append(anyv)
    return np.stack(out, 1)


def shape_case(name, n_sms=None):
    """(cfg, seed, pts (n_cols, n_per, 3), viewdir (n_cols, 3)) of a named shape of the layer checks."""
    from cases import PREDICT_CASES, load_golden, pyramid_for
    from oracle import scenerf_oracle as orc
    from scenerf_b200 import synth
    key = "predict_adversarial_bf" if name == "adv_bf" else "predict_adversarial_kitti"
    cfg, seed = PREDICT_CASES[key]
    g = load_golden(key)
    pts, vd = g["cam_pts"].astype(np.float32), g["viewdir"].astype(np.float32)
    flat, vflat = pts.reshape(-1, 3), np.repeat(vd, pts.shape[1], axis=0)
    if name in ("adv_kitti", "adv_bf"):
        return cfg, seed, pts, vd
    if name == "n1":
        return cfg, seed, pts[:1, :1].copy(), vd[:1].copy()
    if name == "n65_per13":            # n % 64 == 1; 13 points per column: columns straddle the tile boundary
        return cfg, seed, flat[:65].reshape(5, 13, 3).copy(), vd[:5].copy()
    if name == "n127_per1":            # n % 64 == 63; one point per column
        return cfg, seed, flat[:127].reshape(127, 1, 3).copy(), vflat[:127].copy()
    assert name == "multitile"
    # 2 SMs + 1 tiles (every CTA runs two or three tiles), the last one ragged.  Tiles of three kinds: every point
    # outside every map (the tile's lin_z passes are all skipped), points that reach only some of the scales (the maps
    # are sampled at full-resolution coordinates, scenerf.py:522-527: the coarse maps cover only the top-left of the
    # sphere grid, so such points skip the coarse scales' chunks), points that reach all five; a CTA's consecutive
    # tiles are always of different kinds
    n_tiles = 2 * n_sms + 1
    u = synth.hash_uniform(71, 3 * 400000).reshape(-1, 3)
    cand = ((u - 0.5) * np.array([90.0, 40.0, 90.0]) + np.array([0.0, 0.0, 25.0])).astype(np.float32)
    inv_K = np.linalg.inv(cfg.K).astype(np.float32)
    coords, _ = orc.sphere_coords_from_pixels(orc.cam_pts_2_pix(cand, cfg.K), inv_K, cfg.angles(), cfg.sphere_W, cfg.sphere_H)
    hit = tap_scales(cfg, pyramid_for(cfg, seed), coords)
    kinds = [np.flatnonzero(~hit.any(1)), np.flatnonzero(hit.any(1) & ~hit.all(1)), np.flatnonzero(hit.all(1))]
    assert all(k.size >= 64 for k in kinds), [k.size for k in kinds]
    pick = []
    for t in range(n_tiles):
        pool = kinds[(t + t // n_sms) % 3]
        pick.append(pool[(np.arange(64) * 7919 + 131 * t) % pool.size])
    sel = np.concatenate(pick)[:n_tiles * 64 - 27]
    v = synth.hash_uniform(72, sel.size * 3).reshape(-1, 3).astype(np.float32) - np.float32(0.5)
    return cfg, seed, cand[sel].reshape(-1, 1, 3).copy(), v
