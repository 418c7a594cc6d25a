"""Novel-view sweep driver: the callers' glue around `render_rays_batch` in the reference's scene-reconstruction
pipeline, kept on the device end to end ("next" row 8f-4 of the hot-path contract).

Reference (file:line):
  scenerf/models/utils.py:6-49                                      sample_rel_poses_bf / sample_rel_poses
  scenerf/scripts/reconstruction/generate_novel_depths.py:52,103-152   pixel grid -> render -> transpose + bilinear upsample
  scenerf/scripts/reconstruction/depth2tsdf.py:87-103                  TSDF integration of the saved sweep
The reference serialises one render call per pose and round-trips depth (.npy) and colour (.png) through disk; here a
sweep is pose loop -> render (depth+colour only) -> `srf_upsample_render` -> `srf_tsdf_integrate`, all on one stream,
and across GPUs the poses are sharded with one volume merge at the end (`srf_tsdf_merge`)."""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Iterable, Optional, Tuple

import numpy as np
import torch

from . import _lib
from .tsdf import TSDFVolume


def _rot_y_pose(step: float, angle: float) -> torch.Tensor:
    rad = angle / 180 * math.pi
    rel = torch.eye(4)
    rel[2, 3] += step
    rot = torch.eye(4)
    rot[:3, :3] = torch.tensor([[math.cos(rad), 0, math.sin(rad)], [0, 1, 0], [-math.sin(rad), 0, math.cos(rad)]])
    return rot @ rel


def sample_rel_poses(step=0.5, angle=0, max_distance=10.1) -> Dict[Tuple[float, float], torch.Tensor]:
    """utils.py:29-49.  Keys are (step, angle) python numbers (the reference's keys are 0-d tensors that only end up in
    file names); values (4,4) float32 CPU tensors; insertion order = the reference's (angles [0, +a, -a] per step)."""
    angles = [0] + ([angle, -angle] if angle != 0 else [])
    steps = torch.arange(start=0, end=max_distance, step=step)
    return {(float(s), a): _rot_y_pose(s, a) for s in steps for a in angles}


def sample_rel_poses_bf(angle=0, max_distance=2.1, step=0.2) -> Dict[Tuple[float, float], torch.Tensor]:
    """utils.py:6-26 (angles [0, -a, +a] per step)."""
    angles = [0] + ([-angle, angle] if angle != 0 else [])
    steps = torch.arange(start=0, end=max_distance, step=step)
    return {(float(s), a): _rot_y_pose(s, a) for s in steps for a in angles}


def pixel_grid(img_size: Tuple[int, int], scale: int, device) -> Tuple[torch.Tensor, Tuple[int, int]]:
    """generate_novel_depths.py:103-112: x-major (x, y) float pixel grid of stride `scale`; returns (pixels, (gw, gh))."""
    xs = torch.arange(start=0, end=img_size[0], step=scale, dtype=torch.float32, device=device)
    ys = torch.arange(start=0, end=img_size[1], step=scale, dtype=torch.float32, device=device)
    gx, gy = torch.meshgrid(xs, ys, indexing="ij")
    return torch.stack([gx, gy], dim=2).reshape(-1, 2).contiguous(), (int(xs.numel()), int(ys.numel()))


# colour of rays_to_images: raw, clamped to [0,1], the PNG round trip of the TSDF stage (x255), the PNG round trip the
# colour evaluation reads back (float32(uint8(c*255))/255, eval_color.py)
COLOR_RAW, COLOR_CLAMP, COLOR_PNG, COLOR_EVAL = 0, 1, 2, 3


def rays_to_images(depth_rays: Optional[torch.Tensor], color_rays: Optional[torch.Tensor], grid: Tuple[int, int],
                   img_size: Tuple[int, int], color_mode: int = COLOR_CLAMP):
    """generate_novel_depths.py:125-147 in one kernel: x-major ray buffers -> depth (H,W), colour (H,W,3)."""
    lib = _lib.load()
    ref = depth_rays if depth_rays is not None else color_rays
    gw, gh = grid
    W, H = img_size
    d_out = c_out = None
    if depth_rays is not None:
        depth_rays = depth_rays.contiguous()
        assert depth_rays.numel() == gw * gh and depth_rays.dtype == torch.float32
        d_out = torch.empty((H, W), dtype=torch.float32, device=ref.device)
    if color_rays is not None:
        color_rays = color_rays.contiguous()
        assert color_rays.numel() == gw * gh * 3 and color_rays.dtype == torch.float32
        c_out = torch.empty((H, W, 3), dtype=torch.float32, device=ref.device)
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(lib.srf_upsample_render(p(depth_rays), p(color_rays), gw, gh, H, W, p(d_out), p(c_out), int(color_mode),
                                       C.c_void_p(torch.cuda.current_stream(ref.device).cuda_stream)))
    return d_out, c_out


# Frames of the colour-render scripts, as NovelDepthSweep arguments: render(T, COLOR_EVAL) gives the image eval_color.py
# reads back from the saved PNG.
#   KITTI (render_colors.py:102-127): stride 3 over 1220x370 -> 407x124 rays, transposed, no upsampling.
#   BundleFusion (render_colors_bf.py:124-163): stride 2 over 640x480, bilinear x2 back to 640x480.
RENDER_COLORS_KITTI = dict(img_size=(1220, 370), scale=3, ray_batch_size=4000, out_size=(407, 124))
RENDER_COLORS_BF = dict(img_size=(640, 480), scale=2, ray_batch_size=8000)


class NovelDepthSweep:
    """One source frame's sweep: `render(T)` = generate_novel_depths.py:103-152 for one pose (returns device images),
    `reconstruct(...)` = that loop over `rel_poses` feeding depth2tsdf.py:87-103's TSDF volume directly."""

    def __init__(self, renderer, cam_K: torch.Tensor, x_rgb: Dict[str, torch.Tensor], img_size=(1220, 370), scale: int = 2,
                 ray_batch_size: int = 5000, out_size: Optional[Tuple[int, int]] = None):
        """out_size (W, H) of the images render() returns: img_size (upsampled from the grid) by default; the grid's own
        size renders without upsampling (render_colors.py)."""
        self.r, self.cam_K, self.x_rgb = renderer, cam_K, x_rgb
        self.img_size, self.scale, self.ray_batch_size = (int(img_size[0]), int(img_size[1])), int(scale), int(ray_batch_size)
        self.pixels, self.grid = pixel_grid(self.img_size, self.scale, renderer.device)
        self.out_size = self.img_size if out_size is None else (int(out_size[0]), int(out_size[1]))
        self.launches = 0

    def render(self, T_source2infer, color_mode: int = COLOR_CLAMP, noise=None):
        out = self.r.render_rays_batch(self.cam_K, T_source2infer, self.x_rgb, ray_batch_size=self.ray_batch_size,
                                       sampled_pixels=self.pixels, noise=noise, outputs="minimal")
        self.launches += self.r.last_launches + 1
        return rays_to_images(out["depth"], out["color"], self.grid, self.out_size, color_mode)

    def reconstruct(self, rel_poses: Dict, T_velo2cam, vol_bnds, voxel_size=0.2, trunc_margin=10, noises=None,
                    rank: int = 0, world: int = 1, group=None) -> TSDFVolume:
        """Integrate the sweep into a TSDF volume.  With world > 1 every rank renders a contiguous range of the poses
        into its own volume and the volumes are merged in rank order (== pose order), which reproduces the sequential
        integration (distances and weights bit for bit; colours up to float32-exact distance ties, see
        csrc/image_ops.cu); every rank returns the merged volume."""
        from .dist import shard_range
        items = list(rel_poses.items())
        lo, hi, _ = shard_range(len(items), rank, world)
        vol = TSDFVolume(vol_bnds, voxel_size=voxel_size, trunc_margin=trunc_margin, device=self.r.device)
        inv_v2c = np.linalg.inv(np.asarray(T_velo2cam, dtype=np.float64))
        cam_K_host = self.cam_K.detach().cpu().numpy()
        for i in range(lo, hi):
            rel = items[i][1]
            depth, rgb = self.render(rel.to(self.cam_K), COLOR_PNG, None if noises is None else noises[i])
            vol.integrate(rgb, depth, cam_K_host, inv_v2c @ rel.detach().cpu().numpy().astype(np.float64), obs_weight=1.)
            self.launches += 1
        if world > 1:
            import torch.distributed as dist
            packed = torch.stack([vol._tsdf, vol._weight, vol._color])
            gathered = [torch.empty_like(packed) for _ in range(world)]
            dist.all_gather(gathered, packed, group=group)
            merged = TSDFVolume(vol_bnds, voxel_size=voxel_size, trunc_margin=trunc_margin, device=self.r.device)
            for g in gathered:                       # rank order == pose order
                merged.merge_(g[0], g[1], g[2])
            vol = merged
        return vol
