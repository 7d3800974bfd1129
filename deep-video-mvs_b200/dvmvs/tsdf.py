"""TSDF fusion of predicted depth maps under the reference's names: `TSDFVolume` / `TSDFFusion` of
sample-data/run-tsdf-reconstruction.py (SURVEY.md section 8 row f4).  `TSDFVolume.integrate` is one launch of
dvmvs_tsdf_integrate (csrc/tsdf.cu) on volumes resident in HBM; its results are bit-identical to the reference's CPU path
(use_gpu=False -- what the reference runs wherever pycuda is missing).  There is no CPU fallback: without the CUDA library or
a GPU the constructor raises.

Same constructor / integrate / get_volume signatures and argument meaning as the reference (:34, :220, :325).  `integrate`
accepts numpy arrays (as the reference's caller passes, :500-560) or CUDA tensors (depth maps straight from the network:
no host round trip).

Mesh extraction (`get_mesh` / `get_point_cloud`, :329-358), scikit-image's marching cubes in the reference, runs on the device
too: dvmvs_mesh_count / dvmvs_mesh_extract (csrc/mesh.cu).  Sign-only face resolution makes the mesh watertight wherever it
does not reach the volume border, and its order deterministic (vertices by grid edge, faces by cube); the contract is stated in
csrc/mesh.cu and tools/gen_mc_tables.py.  `get_mesh_tensors` leaves the mesh on the device; `get_mesh` copies only the mesh
(never the volume) to the host.

Rendering (`render` / `render_tensors`), which the reference lacks: depth, normal and colour maps of the fused model at any
camera poses, ray-cast on the device by dvmvs_tsdf_raycast (csrc/raycast.cu, contract stated there), e.g. to score the fused
depth against ground truth with dvmvs.errors.compute_errors or as model-to-frame depth for tracking."""
import ctypes

import numpy as np
import torch

from . import _native as N
from ._ops import _stream


class TSDFVolume(object):
    """Volumetric TSDF fusion of RGB-D frames (run-tsdf-reconstruction.py:30-358)."""

    def __init__(self, vol_bnds, voxel_size, use_gpu=True, device=None):
        vol_bnds = np.array(vol_bnds, dtype=np.float64)
        if vol_bnds.shape != (3, 2):
            raise AssertionError("[!] `vol_bnds` should be of shape (3, 2).")          # the reference's message (:43)
        if not use_gpu:
            raise RuntimeError("TSDFVolume: this package has no CPU path (use_gpu=False is the reference's numba fallback)")
        if not N.DRYRUN and not torch.cuda.is_available():
            raise RuntimeError("TSDFVolume: needs a CUDA device (no CPU fallback)")
        self._voxel_size = float(voxel_size)
        self._trunc_margin = 5 * self._voxel_size                                     # :46
        self._color_const = 256 * 256
        self._vol_dim = np.ceil((vol_bnds[:, 1] - vol_bnds[:, 0]) / self._voxel_size).astype(int)     # :50
        vol_bnds[:, 1] = vol_bnds[:, 0] + self._vol_dim * self._voxel_size
        self._vol_bnds = vol_bnds
        self._vol_origin = vol_bnds[:, 0].astype(np.float32)                           # :52
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type == "cuda" and self.device.index is None and torch.cuda.is_available():
            self.device = torch.device("cuda", torch.cuda.current_device())
        shape = tuple(int(d) for d in self._vol_dim)
        self._tsdf_vol = torch.ones(shape, dtype=torch.float32, device=self.device)     # :57-61
        self._weight_vol = torch.zeros(shape, dtype=torch.float32, device=self.device)
        self._color_vol = torch.zeros(shape, dtype=torch.float32, device=self.device)
        self._updated = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._origin_c = (ctypes.c_float * 3)(*[float(v) for v in self._vol_origin])
        self._staging = {}
        self.gpu_mode = True

    # ---- the hot path -------------------------------------------------------------------------------------------------
    def _upload(self, a, name):
        """Host array -> device through a two-deep ring of pinned staging buffers owned by the volume (allocating pinned
        memory per frame would cost more than the kernel); a slot is reused only after its previous copy has completed."""
        key = (name, tuple(a.shape), a.dtype)
        ring = self._staging.get(key)
        if ring is None:
            ring = self._staging[key] = {"next": 0, "slots": [
                (torch.empty(a.shape, dtype=a.dtype).pin_memory(), torch.empty(a.shape, dtype=a.dtype, device=self.device), torch.cuda.Event())
                for _ in range(2)]}
        host, dev, done = ring["slots"][ring["next"]]
        ring["next"] ^= 1
        done.synchronize()
        host.copy_(a)
        dev.copy_(host, non_blocking=True)
        done.record()
        return dev

    def _to_device(self, a, allowed, name):
        if isinstance(a, np.ndarray):
            a = torch.from_numpy(np.ascontiguousarray(a))
        if not isinstance(a, torch.Tensor):
            raise TypeError("TSDFVolume.integrate: %s must be a numpy array or a tensor" % name)
        if a.dtype not in allowed:
            a = a.to(allowed[-1])
        if not a.is_cuda:
            return self._upload(a, name)
        if a.device != self.device:
            raise RuntimeError("TSDFVolume.integrate: %s lives on %s, the volume on %s" % (name, a.device, self.device))
        return a.contiguous()

    def integrate(self, color_im, depth_im, cam_intr, cam_pose, obs_weight=1.):
        """Integrate an RGB-D frame (:220-323).  color_im (H,W,3) RGB uint8 / float; depth_im (H,W) float32 / float64, 0 =
        invalid; cam_intr (3,3); cam_pose (4,4) camera-to-world; obs_weight: weight of this observation."""
        intr = np.asarray(cam_intr.cpu() if isinstance(cam_intr, torch.Tensor) else cam_intr).astype(np.float32)      # :197
        pose = np.asarray(cam_pose.cpu() if isinstance(cam_pose, torch.Tensor) else cam_pose)
        inv = np.ascontiguousarray(np.linalg.inv(pose), dtype=np.float64)              # :285, host logic as in the reference
        intr4 = (ctypes.c_float * 4)(float(intr[0, 0]), float(intr[1, 1]), float(intr[0, 2]), float(intr[1, 2]))
        inv16 = (ctypes.c_double * 16)(*[float(v) for v in inv.reshape(-1)])
        with torch.cuda.device(self.device):
            depth = self._to_device(depth_im, (torch.float64, torch.float32), "depth_im")
            color = self._to_device(color_im, (torch.uint8, torch.float32), "color_im")
            if depth.dim() != 2 or tuple(color.shape) != (depth.shape[0], depth.shape[1], 3):
                raise RuntimeError("TSDFVolume.integrate: expected depth (H,W) and colour (H,W,3), got %s and %s" % (tuple(depth.shape), tuple(color.shape)))
            N.check(N.lib().dvmvs_tsdf_integrate(
                self._tsdf_vol.data_ptr(), self._weight_vol.data_ptr(), self._color_vol.data_ptr(),
                int(self._vol_dim[0]), int(self._vol_dim[1]), int(self._vol_dim[2]), self._origin_c, self._voxel_size,
                self._trunc_margin, color.data_ptr(), 1 if color.dtype == torch.uint8 else 0, depth.data_ptr(),
                1 if depth.dtype == torch.float64 else 0, int(depth.shape[0]), int(depth.shape[1]), intr4, inv16,
                float(obs_weight), self._updated.data_ptr(), _stream()), "tsdf_integrate")

    # ---- read-back ----------------------------------------------------------------------------------------------------
    def get_volume(self):
        """(tsdf, colour) as numpy arrays, like the reference (:325-328; its GPU mode copies device -> host here too)."""
        return self._tsdf_vol.cpu().numpy(), self._color_vol.cpu().numpy()

    def get_volume_tensors(self):
        """(tsdf, weight, colour) CUDA tensors, no copy."""
        return self._tsdf_vol, self._weight_vol, self._color_vol

    def updated_voxels(self):
        """Total number of voxel updates so far (synchronises)."""
        return int(self._updated.item())

    def get_mesh_tensors(self):
        """Marching cubes at level 0 on the device (:344-358): (verts (V,3) float32 world coordinates, faces (F,3) int32,
        norms (V,3) float32, colors (V,3) uint8 RGB) as CUDA tensors, enqueued on torch's current stream.  Synchronises
        once: the host reads the vertex and face counts between the count and the extract launches to size the outputs."""
        dims = [int(d) for d in self._vol_dim]
        with torch.cuda.device(self.device):
            nbytes = ctypes.c_longlong(0)
            N.check(N.lib().dvmvs_mesh_scratch_bytes(dims[0], dims[1], dims[2], ctypes.byref(nbytes)), "mesh_scratch_bytes")
            scratch = torch.empty(max(int(nbytes.value), 8), dtype=torch.uint8, device=self.device)
            stream = _stream()
            N.check(N.lib().dvmvs_mesh_count(self._tsdf_vol.data_ptr(), dims[0], dims[1], dims[2], scratch.data_ptr(),
                                             scratch.numel(), stream), "mesh_count")
            n_verts, n_faces = (int(v) for v in scratch[:8].view(torch.int32).cpu())        # the one device -> host read
            verts = torch.empty((n_verts, 3), dtype=torch.float32, device=self.device)
            norms = torch.empty((n_verts, 3), dtype=torch.float32, device=self.device)
            colors = torch.empty((n_verts, 3), dtype=torch.uint8, device=self.device)
            faces = torch.empty((n_faces, 3), dtype=torch.int32, device=self.device)
            keys = torch.empty(max(n_verts, 1), dtype=torch.int32, device=self.device)
            N.check(N.lib().dvmvs_mesh_extract(
                self._tsdf_vol.data_ptr(), self._color_vol.data_ptr(), dims[0], dims[1], dims[2], self._origin_c,
                self._voxel_size, scratch.data_ptr(), scratch.numel(), n_verts, n_faces, keys.data_ptr(), verts.data_ptr(),
                faces.data_ptr(), norms.data_ptr(), colors.data_ptr(), stream), "mesh_extract")
        return verts, faces, norms, colors

    def get_mesh(self):
        """(verts, faces, norms, colors) as numpy arrays, like the reference's :344-358: get_mesh_tensors copied to the host."""
        return tuple(t.cpu().numpy() for t in self.get_mesh_tensors())

    def get_point_cloud(self):
        """:329-342."""
        verts, _, _, colors = self.get_mesh()
        return np.hstack([verts, colors])

    # ---- rendering (no reference counterpart) ---------------------------------------------------------------------------
    def render_tensors(self, cam_intr, cam_poses, height, width):
        """Ray-cast the fused volume at one or more camera poses (dvmvs_tsdf_raycast, csrc/raycast.cu; one launch for all
        views, enqueued on torch's current stream).  cam_intr (3,3) in pixels of the rendered (height, width) image, fx and fy
        finite and > 0; cam_poses (4,4) or (V,4,4) camera-to-world like integrate's cam_pose, a numpy array or a tensor (CUDA
        tensors on the volume's device are read there, no host round trip).  Returns CUDA tensors depth (V,H,W) float32
        camera depth of the first + -> - crossing of the tsdf (0 = no hit), normals (V,H,W,3) float32 world-frame unit normals
        toward increasing tsdf and colors (V,H,W,3) uint8 RGB (both 0 where there is no hit); a single (4,4) pose gives them
        without the V axis.  The raw tsdf is rendered: unobserved voxels are not masked (as in get_mesh)."""
        intr = np.asarray(cam_intr.detach().cpu() if isinstance(cam_intr, torch.Tensor) else cam_intr)
        if intr.shape != (3, 3):
            raise RuntimeError("TSDFVolume.render: cam_intr must be (3,3), got %s" % (intr.shape,))
        intr4 = intr.astype(np.float32)[[0, 1, 0, 1], [0, 1, 2, 2]]                  # fx fy cx cy
        if not (np.all(np.isfinite(intr4)) and intr4[0] > 0 and intr4[1] > 0):
            raise RuntimeError("TSDFVolume.render: focal lengths must be finite and > 0 and the principal point finite, got "
                               "fx %r fy %r cx %r cy %r" % tuple(float(v) for v in intr4))
        height, width = int(height), int(width)
        if height <= 0 or width <= 0:
            raise RuntimeError("TSDFVolume.render: bad image size %d x %d" % (height, width))
        poses = cam_poses
        if isinstance(poses, torch.Tensor) and poses.device.type == "cpu":
            poses = poses.detach().numpy()
        if not isinstance(poses, torch.Tensor):
            poses = np.asarray(poses)
        shape = tuple(poses.shape)
        single = shape == (4, 4)
        if not (single or (len(shape) == 3 and shape[0] > 0 and shape[1:] == (4, 4))):
            raise RuntimeError("TSDFVolume.render: cam_poses must be (4,4) or (V,4,4), got %s" % (shape,))
        n = 1 if single else shape[0]
        with torch.cuda.device(self.device):
            if isinstance(poses, torch.Tensor):
                if poses.device != self.device:
                    raise RuntimeError("TSDFVolume.render: cam_poses lives on %s, the volume on %s" % (poses.device, self.device))
                p = poses.detach().reshape(n, 4, 4)
                intr_dev = self._upload(torch.from_numpy(intr4.copy()), "intr")             # pinned: no stream synchronisation
                views = torch.cat([intr_dev.expand(n, 4), p[:, :3, :3].reshape(n, 9).to(torch.float32), p[:, :3, 3].to(torch.float32)],
                                  dim=1).contiguous()
            else:
                p = poses.reshape(n, 4, 4).astype(np.float32)
                packed = np.concatenate([np.broadcast_to(intr4, (n, 4)), p[:, :3, :3].reshape(n, 9), p[:, :3, 3]], axis=1)
                views = self._upload(torch.from_numpy(np.ascontiguousarray(packed, dtype=np.float32)), "views")
            depth = torch.empty((n, height, width), dtype=torch.float32, device=self.device)
            normals = torch.empty((n, height, width, 3), dtype=torch.float32, device=self.device)
            colors = torch.empty((n, height, width, 3), dtype=torch.uint8, device=self.device)
            N.check(N.lib().dvmvs_tsdf_raycast(
                self._tsdf_vol.data_ptr(), self._color_vol.data_ptr(), int(self._vol_dim[0]), int(self._vol_dim[1]),
                int(self._vol_dim[2]), self._origin_c, self._voxel_size, self._trunc_margin, views.data_ptr(), n, height, width,
                depth.data_ptr(), normals.data_ptr(), colors.data_ptr(), _stream()), "tsdf_raycast")
        if single:
            return depth[0], normals[0], colors[0]
        return depth, normals, colors

    def render(self, cam_intr, cam_poses, height, width):
        """render_tensors copied to the host: (depth, normals, colors) numpy arrays."""
        return tuple(t.cpu().numpy() for t in self.render_tensors(cam_intr, cam_poses, height, width))


class TSDFFusion(object):
    """Host-side helpers of the reference's driver (:360-480): frustum bounds and the per-frame loop."""

    @staticmethod
    def rigid_transform(xyz, transform):
        """(N,3) points through a 4x4 transform (:361-367)."""
        xyz = np.asarray(xyz)
        homogeneous = np.concatenate([xyz, np.ones((len(xyz), 1), dtype=np.float32)], axis=1)
        return np.dot(transform, homogeneous.T).T[:, :3]

    @staticmethod
    def get_view_frustum(depth_im, cam_intr, cam_pose):
        """The 5 corners (apex + far plane) of the camera frustum in world coordinates, (3,5) (:369-382)."""
        im_h, im_w = depth_im.shape[0], depth_im.shape[1]
        max_depth = float(np.max(depth_im))
        us = np.array([0, 0, 0, im_w, im_w], dtype=np.float64)
        vs = np.array([0, 0, im_h, 0, im_h], dtype=np.float64)
        zs = np.array([0, max_depth, max_depth, max_depth, max_depth])
        pts = np.stack([(us - cam_intr[0, 2]) * zs / cam_intr[0, 0], (vs - cam_intr[1, 2]) * zs / cam_intr[1, 1], zs], axis=1)
        return TSDFFusion.rigid_transform(pts, cam_pose).T

    @staticmethod
    def calculate_volume_bounds(depth_maps, poses, K):
        """:465-475 (bounds start at the origin, as in the reference)."""
        assert len(depth_maps) == len(poses)
        bounds = np.zeros((3, 2))
        for depth_map, pose in zip(depth_maps, poses):
            pts = TSDFFusion.get_view_frustum(depth_map, K, pose)
            bounds[:, 0] = np.minimum(bounds[:, 0], pts.min(axis=1))
            bounds[:, 1] = np.maximum(bounds[:, 1], pts.max(axis=1))
        return bounds

    @staticmethod
    def integrate(tsdf_volume, images, depths, poses, K, obs_weight=1.):
        """The fusion loop of :442-463 without the mesh files: every frame into the volume; returns frames per second
        (device-timed when on a GPU)."""
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for image, depth, pose in zip(images, depths, poses):
            tsdf_volume.integrate(image, depth, K, pose, obs_weight=obs_weight)
        stop.record()
        stop.synchronize()
        return len(images) / max(start.elapsed_time(stop) * 1e-3, 1e-9)
