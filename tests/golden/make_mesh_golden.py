"""Golden vectors of the TSDF mesh extraction (tests/golden/tsdf_mesh.npz), made by running the reference's own
TSDFVolume.get_point_cloud / get_mesh / get_mesh(mask) (scenerf/data/utils/fusion.py:333-379).

Runs only where the reference tree exists (like make_goldens.py, whose inputs and import shims it reuses):
    python tests/golden/make_mesh_golden.py

scikit-image is not installed, so its marching_cubes_lewiner is stubbed with the index-space core of
oracle/mesh_oracle.py.  What the golden pins is the reference's post-processing around that call: world coordinates,
colour lookup at the rounded index and unfolding, the raw (255 kept) volume, the mask written as 1s, the call order.
The volume is a 16x16x12 crop of the tsdf_fusion case, fused from the same three frames (stored in tsdf_fusion.npz)."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_goldens  # noqa: E402  (puts the repository and the reference tree on sys.path)
from oracle import mesh_oracle  # noqa: E402
from scenerf_b200 import synth  # noqa: E402

VOL_BNDS = np.array([[6.0, 9.2], [-1.6, 1.6], [-2.0, 0.4]])          # 16 x 16 x 12 voxels of 0.2 m


def mesh_mask(shape):
    """False (read as 1.0 by get_mesh) on a z slab and on a 5 % scatter of voxels."""
    m = synth.hash_unit(71, int(np.prod(shape))).reshape(shape) >= 0.05
    m[:, :, shape[2] // 2:shape[2] // 2 + 2] = False
    return m


def tsdf_mesh():
    sk = types.ModuleType("skimage")
    sk.measure = types.ModuleType("skimage.measure")
    sys.modules.setdefault("skimage", sk)
    sys.modules.setdefault("skimage.measure", sk.measure)
    sys.modules["skimage.measure"].marching_cubes_lewiner = lambda vol, level=0: mesh_oracle.marching_cubes(vol)
    import scenerf.data.utils.fusion as fusion
    fusion.measure = sys.modules["skimage.measure"]
    K, frames, _ = make_goldens.tsdf_inputs()
    vol = fusion.TSDFVolume(VOL_BNDS.copy(), voxel_size=0.2, trunc_margin=10, use_gpu=False)
    for rgb, depth, pose in frames:
        vol.integrate(rgb, depth, K, pose, obs_weight=1.)
    tsdf, color = vol.get_volume()
    out = dict(vol_bnds=VOL_BNDS, tsdf=tsdf.copy(), color=color.copy())
    out["mask"] = mask = mesh_mask(tsdf.shape)
    pc_verts, pc_colors = vol.get_point_cloud()
    out["verts"], out["faces"], out["norms"], out["colors"] = vol.get_mesh()
    # get_point_cloud returns the vertices and colours of get_mesh(): stored once
    assert np.array_equal(pc_verts, out["verts"]) and np.array_equal(pc_colors, out["colors"])
    # last: the reference's CPU path writes the masked-out 1s into its own volume
    out["mverts"], out["mfaces"], out["mnorms"], out["mcolors"] = vol.get_mesh(mask)
    return out


if __name__ == "__main__":
    g = tsdf_mesh()
    path = os.path.join(HERE, "tsdf_mesh.npz")
    np.savez_compressed(path, **g)
    print("%-32s %8.1f KB  keys=%d  verts=%d faces=%d masked faces=%d" % (
        "tsdf_mesh", os.path.getsize(path) / 1024.0, len(g), len(g["verts"]), len(g["faces"]), len(g["mfaces"])))
