"""Training with matmul="fp32tc": the NT products of the training forward and backward on the split 3xTF32 wgmma kernel
(float32-grade products, csrc/tma.cuh), held to the STRICT float32 mode's bounds of test_backward.py -- not the tf32
mode's: the loss within 2e-4 of the reference's, parameter and feature-map gradients against the reference's autograd
digests and entry by entry against the float64 oracle at MAX_REL / L2_REL, bit-reproducible parameter gradients, the
edge sizes and a pass over several chunks."""
import os
import subprocess
import sys

import numpy as np
import pytest

from cases import load_golden
from scenerf_b200 import synth
from test_backward import (CASES, L2_REL, MAX_REL, _rel, _run_cuda, check_edge_case, check_param_grads, check_pyramid_grads,
                           cotangents, edge_case_grads)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_fp32tc_matches_reference_autograd(name):
    g, cfg, seed, out, L, tm, tg, x_rgb, t = _run_cuda(name, matmul="fp32tc")
    assert abs(float(L) - float(g["loss"])) <= 2e-4 * abs(float(g["loss"]))
    np_ = lambda d: {k: v.grad.detach().cpu().numpy() for k, v in d.items()}
    w1 = check_param_grads(np_(tm), g, "main", "cuda-fp32tc")
    w2 = check_param_grads(np_(tg), g, "gauss", "cuda-fp32tc")
    check_pyramid_grads(np_(x_rgb), g, "cuda-fp32tc")
    print("%s fp32tc: worst parameter-gradient error vs reference autograd: max-rel %.2e, L2-rel %.2e" % (
        name, max(w1[0], w2[0]), max(w1[1], w2[1])))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_fp32tc_matches_float64_oracle_and_is_reproducible(name):
    """Entry by entry against the float64 restatement (the scale-4/8/16 map gradients, all zero there, exactly zero), and
    the parameter gradients of a second run bit-identical."""
    from oracle import scenerf_oracle as so, backward_oracle as bo
    g, cfg, seed, out, L, tm, tg, x_rgb, t = _run_cuda(name, matmul="fp32tc")
    orc = so.OracleRenderer(cfg, *synth.make_model_params(cfg))
    r = bo.render_backward(orc, cfg.K, cfg.T, synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H), g["pixels"], g["noise_u"],
                           g["noise_n"], cotangents(g))
    worst = (0.0, 0.0)
    for tag, tens, ref in (("main", tm, r["g_main"]), ("gauss", tg, r["g_gauss"])):
        for k, v in tens.items():
            mx, l2 = _rel(v.grad.cpu().numpy(), ref[k])
            assert mx <= MAX_REL and l2 <= L2_REL, (tag, k, mx, l2)
            worst = (max(worst[0], mx), max(worst[1], l2))
    zero = 0
    for k, v in x_rgb.items():
        if np.abs(r["g_pyr"][k]).max() == 0:
            assert float(v.grad.abs().max()) == 0.0, k
            zero += 1
            continue
        mx, l2 = _rel(v.grad.cpu().numpy(), r["g_pyr"][k])
        assert mx <= MAX_REL and l2 <= L2_REL, (k, mx, l2)
    assert zero >= 1                                    # the coarse scales no point reaches
    _, _, _, _, _, tm2, tg2, _, _ = _run_cuda(name, matmul="fp32tc")
    for k in tm:
        assert (tm[k].grad == tm2[k].grad).all() and (tg[k].grad == tg2[k].grad).all(), k
    print("%s fp32tc vs float64 oracle: max-rel %.2e, L2-rel %.2e; %d all-zero maps exactly zero" % (name, worst[0], worst[1], zero))


@pytest.mark.gpu
@pytest.mark.parametrize("R", [1, 150])
def test_fp32tc_edge_sizes(R):
    """One ray (a single partial tile everywhere) and 150 rays in one chunk (split-K remainders, ragged TMA boxes), at the
    strict mode's bounds (check_edge_case applies the tf32 bounds to matmul="tf32" only)."""
    tm, tg, x_rgb, _ = edge_case_grads(R, "fp32tc")
    check_edge_case(R, "fp32tc", tm, tg, x_rgb)


@pytest.mark.gpu
def test_fp32tc_multi_chunk():
    """The 150-ray case with SRF_TRAIN_CHUNK=1024 (9 full chunks and a tail), in a process of its own like
    test_backward_chunks.py."""
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_train_chunk_worker.py")
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), worker, "fp32tc"]
    p = subprocess.run(cmd, env=dict(os.environ, SRF_TRAIN_CHUNK="1024"), capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "TRAIN_CHUNK_OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
    print(p.stdout.strip())
