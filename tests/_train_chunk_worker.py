"""Subprocess of tests/test_backward_chunks.py (argv[1]: "fp32" or "tf32").  The library reads SRF_TRAIN_CHUNK once per
process, so a training pass split into several chunks needs a process of its own."""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from test_backward import edge_case_grads, check_edge_case      # noqa: E402

R = 150          # x 64 samples = 9600 points of the main pass


def main():
    matmul = sys.argv[1]
    chunk = int(os.environ["SRF_TRAIN_CHUNK"])
    assert R * 64 > chunk and (R * 64) % chunk != 0, "the main pass must span several chunks and end in a tail"
    tm, tg, x_rgb, t = edge_case_grads(R, matmul)
    # every chunk issues at least build_xin, lin_in, 3 x (lin_z, fc_0, fc_1) and lin_out
    assert t.renderer.last_launches >= 12 * (R * 64 // chunk), t.renderer.last_launches
    check_edge_case(R, matmul, tm, tg, x_rgb)
    if matmul == "fp32":
        # the backward's recompute is the same arithmetic as the saved forward, chunk by chunk: identical gradients
        tm2, tg2, _, _ = edge_case_grads(R, matmul, save_activations=False)
        for k in tm:
            assert (tm[k].grad == tm2[k].grad).all() and (tg[k].grad == tg2[k].grad).all(), k
    print("TRAIN_CHUNK_OK", matmul, "launches", t.renderer.last_launches, t.renderer.last_backward_launches)


if __name__ == "__main__":
    main()
