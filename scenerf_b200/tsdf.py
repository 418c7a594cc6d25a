"""Device-side TSDF fusion with the interface of the reference's `TSDFVolume`
(/root/reference/scenerf/data/utils/fusion.py:20-58 constructor, :219-324 integrate, :326-330 get_volume), so that the
scene-reconstruction script (scripts/reconstruction/depth2tsdf.py:87-103) can consume rendered depth / colour tensors
straight from device memory instead of the .npy / .png round trip.  Semantics: the reference's CPU (numba) path.
`get_mesh` / `get_point_cloud` (fusion.py:333-379, skimage's marching_cubes_lewiner there) run marching cubes on the
device (csrc/mesh.cu, DESIGN.md 6.6) and return numpy arrays in the reference's order; `get_mesh(mask)` does not
write into the volume (the reference's CPU path does)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib


class TSDFVolume:
    def __init__(self, vol_bnds, voxel_size, trunc_margin=10, use_gpu=True, device="cuda:0"):
        vol_bnds = np.asarray(vol_bnds, dtype=np.float64).copy()
        assert vol_bnds.shape == (3, 2), "[!] `vol_bnds` should be of shape (3, 2)."
        if not use_gpu or not torch.cuda.is_available():
            raise RuntimeError("scenerf_b200.tsdf.TSDFVolume is the device path (no CPU fallback)")
        self.lib = _lib.load()
        self.device = torch.device(device)
        self._voxel_size = float(voxel_size)
        self._trunc_margin = trunc_margin
        self._vol_dim = np.ceil((vol_bnds[:, 1] - vol_bnds[:, 0]) / self._voxel_size).copy(order="C").astype(int)
        vol_bnds[:, 1] = vol_bnds[:, 0] + self._vol_dim * self._voxel_size
        self._vol_bnds = vol_bnds
        self._vol_origin = vol_bnds[:, 0].copy(order="C").astype(np.float32)
        shape = tuple(int(d) for d in self._vol_dim)
        self._tsdf = torch.empty(shape, dtype=torch.float32, device=self.device)
        self._weight = torch.empty(shape, dtype=torch.float32, device=self.device)
        self._color = torch.empty(shape, dtype=torch.float32, device=self.device)
        self._dims = (C.c_int * 3)(*shape)
        _lib.check(self.lib.srf_tsdf_reset(self._tsdf.data_ptr(), self._weight.data_ptr(), self._color.data_ptr(), self._dims,
                                           C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))

    def integrate(self, color_im, depth_im, cam_intr, cam_pose, obs_weight=1.):
        """color_im (H,W,3), depth_im (H,W): numpy arrays or torch tensors (device tensors are used in place);
        cam_intr (3,3), cam_pose (4,4): numpy / tensors (tiny, read on the host like the reference does)."""
        depth = torch.as_tensor(depth_im).to(device=self.device, dtype=torch.float32).contiguous()
        col = torch.as_tensor(color_im)
        is_u8 = col.dtype == torch.uint8
        col = col.to(device=self.device, dtype=torch.uint8 if is_u8 else torch.float32).contiguous()
        im_h, im_w = depth.shape
        if tuple(col.shape) != (im_h, im_w, 3):
            raise ValueError("color_im must be (H,W,3) matching depth_im, got %s" % (tuple(col.shape),))
        pose = np.asarray(torch.as_tensor(cam_pose).detach().cpu().numpy(), dtype=np.float64)
        inv_pose = np.ascontiguousarray(np.linalg.inv(pose))           # float64, as fusion.py:265
        intr = np.ascontiguousarray(np.asarray(torch.as_tensor(cam_intr).detach().cpu().numpy()).astype(np.float32))
        origin = (C.c_float * 3)(*[float(v) for v in self._vol_origin])
        _lib.check(self.lib.srf_tsdf_integrate(
            self._tsdf.data_ptr(), self._weight.data_ptr(), self._color.data_ptr(), self._dims, origin, self._voxel_size,
            inv_pose.ctypes.data_as(C.POINTER(C.c_double)), intr.ctypes.data_as(C.POINTER(C.c_float)), depth.data_ptr(),
            col.data_ptr(), 1 if is_u8 else 0, int(im_h), int(im_w), float(self._trunc_margin), float(obs_weight),
            C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))

    def merge_(self, tsdf, weight, color):
        """Fold another volume's state (later observations) into this one: include/scenerf_b200.h srf_tsdf_merge."""
        t, w, c = (x.to(device=self.device, dtype=torch.float32).contiguous() for x in (tsdf, weight, color))
        if tuple(t.shape) != tuple(self._tsdf.shape):
            raise ValueError("volume shape mismatch %s vs %s" % (tuple(t.shape), tuple(self._tsdf.shape)))
        _lib.check(self.lib.srf_tsdf_merge(self._tsdf.data_ptr(), self._weight.data_ptr(), self._color.data_ptr(), t.data_ptr(),
                                           w.data_ptr(), c.data_ptr(), self._dims,
                                           C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)))
        return self

    def get_volume(self):
        return self._tsdf.cpu().numpy(), self._color.cpu().numpy()

    def get_weight(self):
        return self._weight.cpu().numpy()

    def _marching_cubes(self, mask, want_faces):
        """Counts, allocates and emits on the device: (verts, faces or None, normals or None, colors) tensors."""
        st = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        mask_ptr = None
        if mask is not None:
            m = torch.as_tensor(mask)
            if m.numel() != self._tsdf.numel():
                raise ValueError("mask has %d elements, the volume %d" % (m.numel(), self._tsdf.numel()))
            m = m.reshape(-1).to(device=self.device, dtype=torch.bool).to(torch.uint8).contiguous()
            mask_ptr = m.data_ptr()
        ws_bytes = self.lib.srf_tsdf_mesh_workspace_bytes(self._dims)
        ws = torch.empty(max(int(ws_bytes), 1), dtype=torch.uint8, device=self.device)
        nv, nf = C.c_longlong(0), C.c_longlong(0)
        _lib.check(self.lib.srf_tsdf_mesh_count_host(self._tsdf.data_ptr(), mask_ptr, self._dims, ws.data_ptr(), ws_bytes,
                                                     C.byref(nv), C.byref(nf), st))
        verts = torch.empty((nv.value, 3), dtype=torch.float32, device=self.device)
        norms = torch.empty((nv.value, 3), dtype=torch.float32, device=self.device) if want_faces else None
        colors = torch.empty((nv.value, 3), dtype=torch.uint8, device=self.device)
        faces = torch.empty((nf.value, 3), dtype=torch.int32, device=self.device) if want_faces else None
        if nv.value:
            origin = (C.c_float * 3)(*[float(v) for v in self._vol_origin])
            _lib.check(self.lib.srf_tsdf_mesh_emit(
                self._tsdf.data_ptr(), self._color.data_ptr(), mask_ptr, self._dims, origin, self._voxel_size, ws.data_ptr(),
                ws_bytes, verts.data_ptr(), norms.data_ptr() if want_faces else None, colors.data_ptr(),
                faces.data_ptr() if want_faces else None, st))
        return verts, faces, norms, colors

    def get_mesh(self, mask=None):
        """Marching cubes at level 0 (fusion.py:356-379): verts (V,3) float32 world coordinates, faces (F,3) int32,
        norms (V,3) float32, colors (V,3) uint8.  mask: X*Y*Z booleans (numpy or tensor); voxels where it is False
        read as 1.0 for this call only."""
        verts, faces, norms, colors = self._marching_cubes(mask, True)
        return verts.cpu().numpy(), faces.cpu().numpy(), norms.cpu().numpy(), colors.cpu().numpy()

    def get_point_cloud(self):
        """The mesh vertices and their colours (fusion.py:333-354)."""
        verts, _, _, colors = self._marching_cubes(None, False)
        return verts.cpu().numpy(), colors.cpu().numpy()
