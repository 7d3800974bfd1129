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
depth against ground truth with dvmvs.errors.compute_errors or as model-to-frame depth for tracking.

`SparseTSDFVolume`, which the reference lacks, fuses frames without bounds known up front (an online camera): voxel blocks are
allocated on the device as frames see them (csrc/tsdf_sparse.cu) and hold what a TSDFVolume with the same origin holds after
the same frames; `to_dense` exports any lattice-aligned box of it as a TSDFVolume, and its mesh and render methods return
exactly what the export's would, computed on the blocks without the dense box (csrc/tsdf_sparse_view.cu)."""
import collections
import contextlib
import ctypes

import numpy as np
import torch

from . import _native as N
from ._ops import _stream


class _FrameInputs(object):
    """Frame inputs of integrate on the volume's device: numpy arrays through pinned staging, CUDA tensors in place."""

    def _upload(self, a, name, dst=None):
        """Host array -> device through a two-deep ring of pinned staging buffers owned by the volume (allocating pinned
        memory per frame would cost more than the kernel); a slot is reused only after its previous copy has completed.
        The copy lands in dst when given (a device tensor of a's shape and dtype), else in a device buffer of the slot."""
        key = (name, tuple(a.shape), a.dtype)
        ring = self._staging.get(key)
        if ring is None:
            ring = self._staging[key] = {"next": 0, "slots": [[torch.empty(a.shape, dtype=a.dtype).pin_memory(), None, torch.cuda.Event()]
                                                              for _ in range(2)]}
        slot = ring["slots"][ring["next"]]
        ring["next"] ^= 1
        host, done = slot[0], slot[2]
        done.synchronize()
        host.copy_(a)
        if dst is None:
            if slot[1] is None:
                slot[1] = torch.empty(a.shape, dtype=a.dtype, device=self.device)
            dst = slot[1]
        dst.copy_(host, non_blocking=True)
        done.record()
        return dst

    def _to_device(self, a, allowed, name, keep=None):
        """a on the volume's device in an allowed dtype; keep(name, a) -> a device tensor of a's shape and dtype that the
        result is copied into (a numpy array is uploaded straight into it), else a CUDA tensor is used in place"""
        if isinstance(a, np.ndarray):
            a = torch.from_numpy(np.ascontiguousarray(a))
        if not isinstance(a, torch.Tensor):
            raise TypeError("%s.integrate: %s must be a numpy array or a tensor" % (type(self).__name__, name))
        if a.dtype not in allowed:
            a = a.to(allowed[-1])
        if not a.is_cuda:
            return self._upload(a, name, None if keep is None else keep(name, a))
        if a.device != self.device:
            raise RuntimeError("%s.integrate: %s lives on %s, the volume on %s" % (type(self).__name__, name, a.device, self.device))
        if keep is None:
            return a.contiguous()
        return keep(name, a).copy_(a)

    def _frame(self, color_im, depth_im, keep=None):
        """(colour, depth) on the device, checked for shape (keep: as _to_device's)"""
        depth = self._to_device(depth_im, (torch.float64, torch.float32), "depth_im", keep)
        color = self._to_device(color_im, (torch.uint8, torch.float32), "color_im", keep)
        if depth.dim() != 2 or tuple(color.shape) != (depth.shape[0], depth.shape[1], 3):
            raise RuntimeError("%s.integrate: expected depth (H,W) and colour (H,W,3), got %s and %s" % (
                type(self).__name__, tuple(depth.shape), tuple(color.shape)))
        return color, depth

    @staticmethod
    def _camera(cam_intr, cam_pose):
        """(float32 fx, fy, cx, cy, float64 inv(cam_pose)) as ctypes arrays, computed on the host as in the reference"""
        intr = np.asarray(cam_intr.cpu() if isinstance(cam_intr, torch.Tensor) else cam_intr).astype(np.float32)      # :197
        pose = np.asarray(cam_pose.cpu() if isinstance(cam_pose, torch.Tensor) else cam_pose)
        inv = np.ascontiguousarray(np.linalg.inv(pose), dtype=np.float64)              # :285, host logic as in the reference
        intr4 = (ctypes.c_float * 4)(float(intr[0, 0]), float(intr[1, 1]), float(intr[0, 2]), float(intr[1, 2]))
        inv16 = (ctypes.c_double * 16)(*[float(v) for v in inv.reshape(-1)])
        return intr4, inv16

    def _views(self, cam_intr, cam_poses, height, width):
        """render_tensors' arguments checked and packed: (views (V,16) float32 on the device -- fx fy cx cy, R row-major, t --,
        V, whether a single (4,4) pose was given, height, width).  Call inside the volume's device scope."""
        name = type(self).__name__
        intr = np.asarray(cam_intr.detach().cpu() if isinstance(cam_intr, torch.Tensor) else cam_intr)
        if intr.shape != (3, 3):
            raise RuntimeError("%s.render: cam_intr must be (3,3), got %s" % (name, intr.shape))
        intr4 = intr.astype(np.float32)[[0, 1, 0, 1], [0, 1, 2, 2]]                  # fx fy cx cy
        if not (np.all(np.isfinite(intr4)) and intr4[0] > 0 and intr4[1] > 0):
            raise RuntimeError("%s.render: focal lengths must be finite and > 0 and the principal point finite, got "
                               "fx %r fy %r cx %r cy %r" % ((name,) + tuple(float(v) for v in intr4)))
        height, width = int(height), int(width)
        if height <= 0 or width <= 0:
            raise RuntimeError("%s.render: bad image size %d x %d" % (name, height, width))
        poses = cam_poses
        if isinstance(poses, torch.Tensor) and poses.device.type == "cpu":
            poses = poses.detach().numpy()
        if not isinstance(poses, torch.Tensor):
            poses = np.asarray(poses)
        shape = tuple(poses.shape)
        single = shape == (4, 4)
        if not (single or (len(shape) == 3 and shape[0] > 0 and shape[1:] == (4, 4))):
            raise RuntimeError("%s.render: cam_poses must be (4,4) or (V,4,4), got %s" % (name, shape))
        n = 1 if single else shape[0]
        if isinstance(poses, torch.Tensor):
            if poses.device != self.device:
                raise RuntimeError("%s.render: cam_poses lives on %s, the volume on %s" % (name, poses.device, self.device))
            p = poses.detach().reshape(n, 4, 4)
            intr_dev = self._upload(torch.from_numpy(intr4.copy()), "intr")             # pinned: no stream synchronisation
            views = torch.cat([intr_dev.expand(n, 4), p[:, :3, :3].reshape(n, 9).to(torch.float32), p[:, :3, 3].to(torch.float32)],
                              dim=1).contiguous()
        else:
            p = poses.reshape(n, 4, 4).astype(np.float32)
            packed = np.concatenate([np.broadcast_to(intr4, (n, 4)), p[:, :3, :3].reshape(n, 9), p[:, :3, 3]], axis=1)
            views = self._upload(torch.from_numpy(np.ascontiguousarray(packed, dtype=np.float32)), "views")
        return views, n, single, height, width


class TSDFVolume(_FrameInputs):
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
    def integrate(self, color_im, depth_im, cam_intr, cam_pose, obs_weight=1.):
        """Integrate an RGB-D frame (:220-323).  color_im (H,W,3) RGB uint8 / float; depth_im (H,W) float32 / float64, 0 =
        invalid; cam_intr (3,3); cam_pose (4,4) camera-to-world; obs_weight: weight of this observation."""
        intr4, inv16 = self._camera(cam_intr, cam_pose)
        with torch.cuda.device(self.device):
            color, depth = self._frame(color_im, depth_im)
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
        with torch.cuda.device(self.device):
            views, n, single, height, width = self._views(cam_intr, cam_poses, height, width)
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


_CAPACITY_FLAGS = N.SPARSE_POOL_FULL | N.SPARSE_TABLE_FULL
# a frame a growable SparseTSDFVolume holds until its allocation is known to have found room: its ring slot (the device copies
# of its depth and colour, the pinned copy of the counters after its allocation and the event recorded after that copy), its
# number among the volume's integrate calls and integrate's arguments
_HeldFrame = collections.namedtuple("_HeldFrame", "slot index color depth intr4 inv16 obs_weight")


class SparseTSDFVolume(_FrameInputs):
    """TSDF fusion without bounds: a volume of 8 x 8 x 8-voxel blocks on the device (csrc/tsdf_sparse.cu, C ABI
    include/dvmvs_tsdf_sparse.h).  A frame allocates, through a hash table on the device, every block holding a voxel it can
    update (free space in front of the surface included) and integrates only the blocks it sees, so memory grows with the
    observed space and the work per frame with what the camera sees.  Voxel (i, j, k) of the signed global lattice sits at
    f32(f64(origin) + voxel_size * f64((i, j, k))) and is updated by the arithmetic of TSDFVolume.integrate: after any frames
    the volume holds, voxel for voxel, the tsdf, weight and colour a TSDFVolume whose origin is `origin` holds after the same
    frames.  `to_dense` exports it into a TSDFVolume; get_mesh / get_point_cloud / render compute what the export's would,
    on the blocks.

    Allocation runs on the device; integrate reads nothing back.  A pool of capacity_blocks blocks is allocated up front
    (device_bytes tells its size).  With max_capacity_blocks None (the default) the pool is fixed: when a frame needs more
    blocks than it holds, the blocks without room are not integrated and the next allocated_blocks / to_dense / get_mesh* /
    render* raises RuntimeError naming the capacity the frames need; the blocks that have room keep being integrated correctly.

    With max_capacity_blocks an integer (>= capacity_blocks, at most 2^29) the volume grows, up to that many blocks, when its
    frames need more.  A frame that finds the pool or the table full is not integrated, and neither is any later frame until
    the volume has grown (halt mode, include/dvmvs_tsdf_sparse_grow.h).  integrate keeps each frame's depth and colour in a
    ring of RING slots on the device until the host has seen, through a pinned copy of the counters, that its allocation found
    room; it never synchronises, except that with all RING slots held it waits for the oldest frame's allocation.  When a held
    frame turns out to have overflowed, and at the start of every read that synchronises (allocated_blocks, updated_voxels,
    to_dense, get_mesh*, render*), the volume settles: it synchronises, grows the pool to
    min(max_capacity_blocks, max(2 x capacity, blocks needed)) with the old pool's slots copied over and the hash table rebuilt
    on the device (dvmvs_tsdf_sparse_rehash), replays the held frames from the first that overflowed, and repeats while a
    frame still overflows.  **Contract**: after any frames, a growable volume holds, voxel for voxel, what a fixed volume
    large enough from the start holds after the same frames, and so what a TSDFVolume with the same origin holds;
    updated_voxels, to_dense, get_mesh* and render* return the same results too.  Only the order of the pool's slots differs
    (it was never deterministic: slots come from an atomic counter, and none of those results depend on it).  At
    max_capacity_blocks the frames from the one that overflowed on are not integrated (integrate then returns at once);
    allocated_blocks, to_dense, get_mesh*
    and render* then raise RuntimeError naming the blocks needed and the cap (updated_voxels still returns its count), and
    every block with a slot holds what it held after the frames before that one.  `capacity` is the current pool size and
    `growths` counts the growths so far."""
    BLOCK = 8
    # Frames a growable volume holds on the device.  A frame is held until the copy of the counters behind its allocation has
    # reached the host, a few launches after integrate enqueued it; 4 slots let the host run three frames ahead of the device
    # (a depth network producing frames while the previous ones fuse) before integrate waits, at a cost of 4 frames of depth
    # and colour in device memory (about 8.6 MB at 640 x 480 with float32 depth and uint8 colour).
    RING = 4

    @staticmethod
    def table_size(capacity_blocks):
        """hash-table entries for a pool of capacity_blocks blocks: the smallest power of two >= 2 * capacity_blocks"""
        return 1 << max(1, (2 * int(capacity_blocks) - 1).bit_length())

    @staticmethod
    def device_bytes(capacity_blocks):
        """device memory of a volume with capacity_blocks blocks: 512 voxels x 12 B, block coordinates and the visible list
        per block; 8 B key and 4 B slot per hash-table entry; the counters.  A growable volume (max_capacity_blocks) holds
        both pools for the length of a growth: its device memory peaks at device_bytes(old capacity) + device_bytes(new
        capacity), plus its ring of RING frames."""
        c = int(capacity_blocks)
        return c * (SparseTSDFVolume.BLOCK ** 3 * 12 + 12 + 4) + SparseTSDFVolume.table_size(c) * 12 + 16

    @staticmethod
    def _grown_capacity(capacity, need, max_capacity):
        """the pool a growth allocates: at least double the current one and at least the blocks needed, at most the cap"""
        return min(int(max_capacity), max(2 * int(capacity), int(need)))

    def __init__(self, voxel_size, origin=(0.0, 0.0, 0.0), capacity_blocks=32768, device=None, max_capacity_blocks=None):
        voxel_size = float(voxel_size)
        if not (np.isfinite(voxel_size) and voxel_size > 0):
            raise ValueError("SparseTSDFVolume: voxel_size must be finite and > 0, got %r" % voxel_size)
        origin = np.asarray(origin, dtype=np.float64)
        if origin.shape != (3,) or not np.all(np.isfinite(origin)):
            raise ValueError("SparseTSDFVolume: origin must be 3 finite numbers, got %r" % (origin,))
        if isinstance(capacity_blocks, bool) or int(capacity_blocks) != capacity_blocks or capacity_blocks < 1:
            raise ValueError("SparseTSDFVolume: capacity_blocks must be a positive integer, got %r" % (capacity_blocks,))
        capacity = int(capacity_blocks)
        if self.table_size(capacity) > 1 << 30:
            raise ValueError("SparseTSDFVolume: capacity_blocks %d exceeds 2^29" % capacity)
        if max_capacity_blocks is not None:
            if (isinstance(max_capacity_blocks, bool) or int(max_capacity_blocks) != max_capacity_blocks
                    or max_capacity_blocks < capacity):
                raise ValueError("SparseTSDFVolume: max_capacity_blocks must be None or an integer >= capacity_blocks %d, got %r"
                                 % (capacity, max_capacity_blocks))
            max_capacity_blocks = int(max_capacity_blocks)
            if self.table_size(max_capacity_blocks) > 1 << 30:
                raise ValueError("SparseTSDFVolume: max_capacity_blocks %d exceeds 2^29" % max_capacity_blocks)
        if not N.DRYRUN and not torch.cuda.is_available():
            raise RuntimeError("SparseTSDFVolume: needs a CUDA device (no CPU fallback)")
        self._voxel_size = voxel_size
        self._trunc_margin = 5 * voxel_size                                             # as TSDFVolume (:46)
        self._origin = origin.astype(np.float32)
        self._origin_c = (ctypes.c_float * 3)(*[float(v) for v in self._origin])
        self.capacity = capacity
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type == "cuda" and self.device.index is None and torch.cuda.is_available():
            self.device = torch.device("cuda", torch.cuda.current_device())
        dev, b = self.device, self.BLOCK
        table = self.table_size(capacity)
        self._keys = torch.full((table,), -1, dtype=torch.int64, device=dev)             # all bits set: empty
        self._slots = torch.full((table,), -1, dtype=torch.int32, device=dev)
        self._coords = torch.zeros((capacity, 3), dtype=torch.int32, device=dev)
        self._tsdf = torch.ones((capacity, b, b, b), dtype=torch.float32, device=dev)   # TSDFVolume's initial state (:57-61)
        self._weight = torch.zeros((capacity, b, b, b), dtype=torch.float32, device=dev)
        self._color = torch.zeros((capacity, b, b, b), dtype=torch.float32, device=dev)
        self._counters = torch.zeros(4, dtype=torch.int32, device=dev)                 # keys, flags, visible, halt mode
        self._visible = torch.zeros(capacity, dtype=torch.int32, device=dev)
        self._updated = torch.zeros(1, dtype=torch.int64, device=dev)
        self._scratch = {}
        self._staging = {}
        self.max_capacity_blocks = max_capacity_blocks
        self.growths = 0
        self._held = collections.deque()                 # growable: the frames not yet known to have found room, oldest first
        self._ring = [{} for _ in range(self.RING)]      # per ring slot: name -> device copy of that input
        self._ring_flags = self._ring_events = None      # pinned [RING][2] counters[0:2] after each slot's allocation; events
        self._next_slot = self._frames = 0
        self._halted_at = None                           # at max_capacity_blocks: the first frame not integrated
        if max_capacity_blocks is not None:
            self._counters[3] = N.SPARSE_HALT_ON_FULL

    def _device_scope(self):
        return torch.cuda.device(self.device) if self.device.type == "cuda" else contextlib.nullcontext()

    # ---- the hot path -------------------------------------------------------------------------------------------------
    def integrate(self, color_im, depth_im, cam_intr, cam_pose, obs_weight=1.):
        """Integrate an RGB-D frame: TSDFVolume.integrate's arguments, accepted types and arithmetic (:220-323), with the
        blocks the frame can update allocated first.  Focal lengths must be finite and > 0.  A growable volume copies the
        frame's depth and colour to its ring first: the caller may overwrite its tensors as soon as integrate returns."""
        intr4, inv16 = self._camera(cam_intr, cam_pose)
        if not (np.all(np.isfinite(list(intr4))) and intr4[0] > 0 and intr4[1] > 0):
            raise ValueError("SparseTSDFVolume.integrate: focal lengths must be finite and > 0 and the principal point finite, "
                             "got fx %r fy %r cx %r cy %r" % tuple(intr4))
        with self._device_scope():
            if self.max_capacity_blocks is None:
                color, depth = self._frame(color_im, depth_im)
                self._enqueue(color, depth, intr4, inv16, float(obs_weight))
                return
            if self._halted_at is not None:
                return                                                      # at the cap: no later frame is integrated
            if self._ring_events is None:
                self._ring_flags = torch.zeros((self.RING, 2), dtype=torch.int32).pin_memory()
                self._ring_events = [torch.cuda.Event() for _ in range(self.RING)]
            self._retire()
            if len(self._held) == self.RING:
                self._ring_events[self._held[0].slot].synchronize()        # integrate's one wait: RING frames in flight
                self._retire()
            slot = self._next_slot
            color, depth = self._frame(color_im, depth_im, keep=lambda name, a: self._ring_buffer(slot, name, a))
            frame = _HeldFrame(slot, self._frames, color, depth, intr4, inv16, float(obs_weight))
            # held only once the library has accepted the frame: a frame it refuses (a pose that is not an invertible finite
            # transform) raises here, before any launch, and takes no ring slot, so no replay ever meets it
            self._enqueue(color, depth, intr4, inv16, frame.obs_weight, slot)
            self._next_slot, self._frames = (slot + 1) % self.RING, self._frames + 1
            self._held.append(frame)

    def _enqueue(self, color, depth, intr4, inv16, obs_weight, slot=None):
        """allocate + integrate one frame on the current stream, inside the volume's device scope; with a ring slot, the
        counters after the allocation are copied to the slot's pinned entry and its event recorded"""
        h, w = int(depth.shape[0]), int(depth.shape[1])
        scratch = self._scratch.get((h, w))
        if scratch is None:
            nbytes = ctypes.c_longlong(0)
            N.check(N.lib().dvmvs_tsdf_sparse_scratch_bytes(h, w, ctypes.byref(nbytes)), "tsdf_sparse_scratch_bytes")
            scratch = self._scratch[(h, w)] = torch.empty(max(int(nbytes.value), 8), dtype=torch.uint8, device=self.device)
        depth_f64 = 1 if depth.dtype == torch.float64 else 0
        stream = _stream()
        N.check(N.lib().dvmvs_tsdf_sparse_allocate(
            self._keys.data_ptr(), self._slots.data_ptr(), int(self._keys.numel()), self._coords.data_ptr(), self.capacity,
            self._counters.data_ptr(), self._visible.data_ptr(), scratch.data_ptr(), scratch.numel(), self._origin_c,
            self._voxel_size, self._trunc_margin, depth.data_ptr(), depth_f64, h, w, intr4, inv16, stream), "tsdf_sparse_allocate")
        if slot is not None:
            self._ring_flags[slot].copy_(self._counters[:2], non_blocking=True)
            self._ring_events[slot].record()
        N.check(N.lib().dvmvs_tsdf_sparse_integrate(
            self._tsdf.data_ptr(), self._weight.data_ptr(), self._color.data_ptr(), self._coords.data_ptr(), self.capacity,
            self._counters.data_ptr(), self._visible.data_ptr(), self._origin_c, self._voxel_size, self._trunc_margin,
            color.data_ptr(), 1 if color.dtype == torch.uint8 else 0, depth.data_ptr(), depth_f64, h, w, intr4, inv16,
            float(obs_weight), self._updated.data_ptr(), stream), "tsdf_sparse_integrate")

    # ---- growth ---------------------------------------------------------------------------------------------------------
    def _ring_buffer(self, slot, name, a):
        """the ring slot's device buffer for input `name`, of a's shape and dtype"""
        t = self._ring[slot].get(name)
        if t is None or t.shape != a.shape or t.dtype != a.dtype:
            t = self._ring[slot][name] = torch.empty(a.shape, dtype=a.dtype, device=self.device)
        return t

    def _overflowed(self, frame):
        return bool(int(self._ring_flags[frame.slot, 1]) & _CAPACITY_FLAGS)

    def _retire(self):
        """lets go of the held frames whose allocation has completed, oldest first; one that found no room settles the volume
        (which replays it and every later frame, and lets go of them all)"""
        while self._held and self._ring_events[self._held[0].slot].query():
            if self._halted_at is None and self._overflowed(self._held[0]):
                self._settle()
            else:
                self._held.popleft()

    def _synchronize(self):
        if self.device.type == "cuda":
            torch.cuda.synchronize(self.device)

    def _settle(self):
        """Synchronises; then, while a frame has found no room and max_capacity_blocks allows, grows the volume and replays
        the held frames from the first that found none.  At the cap, records that frame.  Either way every held frame is then
        settled -- integrated after the last growth, or never to be -- and is let go."""
        if self.max_capacity_blocks is None or self._halted_at is not None:
            return
        with self._device_scope():
            self._synchronize()
            while True:
                n, flags = (int(v) for v in self._counters[:2].tolist())
                held = list(self._held)
                if not flags & _CAPACITY_FLAGS:
                    self._held.clear()
                    return
                first = next((i for i, f in enumerate(held) if self._overflowed(f)), 0)
                if self.capacity >= self.max_capacity_blocks:
                    self._halted_at = held[first].index if held else self._frames
                    self._held.clear()
                    return
                self._grow(self._grown_capacity(self.capacity, n, self.max_capacity_blocks), min(n, self.capacity))
                for f in held[first:]:
                    self._enqueue(f.color, f.depth, f.intr4, f.inv16, f.obs_weight, f.slot)
                self._synchronize()

    def _grow(self, capacity, n_blocks):
        """a pool of `capacity` blocks whose first slots are the old pool's, and a hash table of table_size(capacity) entries
        rebuilt on the device from its first n_blocks slots; clears the pool- and table-full flags"""
        dev, b, old = self.device, self.BLOCK, self.capacity
        table = self.table_size(capacity)
        grown = (torch.zeros((capacity, 3), dtype=torch.int32, device=dev), torch.ones((capacity, b, b, b), dtype=torch.float32, device=dev),
                 torch.zeros((capacity, b, b, b), dtype=torch.float32, device=dev), torch.zeros((capacity, b, b, b), dtype=torch.float32, device=dev))
        for new, cur in zip(grown, (self._coords, self._tsdf, self._weight, self._color)):
            new[:old].copy_(cur)
        self._coords, self._tsdf, self._weight, self._color = grown
        self._visible = torch.zeros(capacity, dtype=torch.int32, device=dev)
        self._keys = torch.full((table,), -1, dtype=torch.int64, device=dev)
        self._slots = torch.full((table,), -1, dtype=torch.int32, device=dev)
        N.check(N.lib().dvmvs_tsdf_sparse_rehash(self._keys.data_ptr(), self._slots.data_ptr(), table, self._coords.data_ptr(), n_blocks,
                                                  self._counters.data_ptr(), _stream()), "tsdf_sparse_rehash")
        self.capacity = capacity
        self.growths += 1

    # ---- read-back ----------------------------------------------------------------------------------------------------
    def allocated_blocks(self):
        """Number of blocks allocated so far (synchronises; a growable volume settles first).  RuntimeError when a frame
        found no room for a block (a growable volume: at max_capacity_blocks)."""
        self._settle()
        n, flags = (int(v) for v in self._counters[:2].cpu())
        if self._halted_at is not None and flags & _CAPACITY_FLAGS:
            raise RuntimeError("SparseTSDFVolume: the frames so far need %s blocks, more than max_capacity_blocks %d: frame %d "
                               "(counting the frames integrate accepted from 0), the one that overflowed the volume, and every later frame "
                               "were not integrated" % (("more than %d" if flags & N.SPARSE_TABLE_FULL else "%d") % n,
                                                        self.max_capacity_blocks, self._halted_at))
        if flags & N.SPARSE_TABLE_FULL:
            raise RuntimeError("SparseTSDFVolume: the hash table of %d entries is full; the frames so far need more than %d "
                               "blocks: construct the volume with a larger capacity_blocks" % (self._keys.numel(), n))
        if flags & N.SPARSE_POOL_FULL:
            raise RuntimeError("SparseTSDFVolume: the frames so far need %d blocks, the pool holds %d: construct the volume with "
                               "capacity_blocks >= %d" % (n, self.capacity, n))
        if flags & N.SPARSE_FRUSTUM:
            raise RuntimeError("SparseTSDFVolume: a frame was not integrated: its view frustum, to its largest depth, spans more "
                               "than 2^31 blocks or leaves the block coordinate range +-2^20")
        return n

    def updated_voxels(self):
        """Total number of voxel updates so far (synchronises; a growable volume settles first)."""
        self._settle()
        return int(self._updated.item())

    def _box(self, vol_bnds, what):
        """(allocated blocks, lower global voxel index k (3,) int64, vol_bnds (3,2) float64) of a lattice-aligned box, by default
        the bounding box of the allocated blocks.  RuntimeError as allocated_blocks; ValueError for a box off the lattice or no
        default box."""
        n = self.allocated_blocks()
        vs, origin = self._voxel_size, self._origin.astype(np.float64)
        if vol_bnds is None:
            if n == 0:
                raise ValueError("SparseTSDFVolume.%s: no block is allocated; give vol_bnds" % what)
            bounds = torch.empty(6, dtype=torch.int32, device=self.device)
            with self._device_scope():
                N.check(N.lib().dvmvs_tsdf_sparse_block_bounds(self._coords.data_ptr(), self.capacity, self._counters.data_ptr(),
                                                                bounds.data_ptr(), _stream()), "tsdf_sparse_block_bounds")
            b = bounds.cpu().numpy().astype(np.int64)
            k = b[:3] * self.BLOCK
            dims = (b[3:] - b[:3] + 1) * self.BLOCK
            lo = origin + k * vs
            vol_bnds = np.stack([lo, lo + (dims - 0.5) * vs], axis=1)                  # TSDFVolume's ceil gives dims exactly
        vol_bnds = np.array(vol_bnds, dtype=np.float64)
        if vol_bnds.shape != (3, 2) or not np.all(np.isfinite(vol_bnds)):
            raise ValueError("SparseTSDFVolume.%s: vol_bnds must be (3,2) finite bounds, got %r" % (what, vol_bnds))
        k = np.rint((vol_bnds[:, 0] - origin) / vs)
        off = np.abs(vol_bnds[:, 0] - (origin + k * vs))
        if np.any(off > 1e-3 * vs + 2.0 ** -23 * np.abs(vol_bnds[:, 0])) or np.any(np.abs(k) >= 2 ** 31):
            raise ValueError("SparseTSDFVolume.%s: the lower bounds %s are not on the voxel lattice origin %s + k * %r"
                             % (what, vol_bnds[:, 0].tolist(), origin.tolist(), vs))
        return n, k.astype(np.int64), vol_bnds

    def to_dense(self, vol_bnds=None):
        """The volume as a TSDFVolume over vol_bnds ((3,2) metres, as TSDFVolume's; the lower bounds on the voxel lattice
        origin + k * voxel_size, else ValueError), by default the bounding box of the allocated blocks.  Voxels of no allocated
        block hold TSDFVolume's initial 1 / 0 / 0.  RuntimeError as allocated_blocks."""
        _, k, vol_bnds = self._box(vol_bnds, "to_dense")
        dense = TSDFVolume(vol_bnds, self._voxel_size, device=self.device)
        dims = [int(d) for d in dense._vol_dim]
        if min(dims) > 0:
            tsdf, weight, color = dense.get_volume_tensors()
            with self._device_scope():
                N.check(N.lib().dvmvs_tsdf_sparse_export(
                    self._tsdf.data_ptr(), self._weight.data_ptr(), self._color.data_ptr(), self._coords.data_ptr(), self.capacity,
                    self._counters.data_ptr(), (ctypes.c_int * 3)(*[int(v) for v in k]), dims[0], dims[1], dims[2],
                    tsdf.data_ptr(), weight.data_ptr(), color.data_ptr(), _stream()), "tsdf_sparse_export")
        return dense

    # ---- mesh and rendering on the blocks (no dense box) ----------------------------------------------------------------
    def _view_box(self, vol_bnds, what):
        """_box plus the box's grid as TSDFVolume(vol_bnds) computes it: (n, k as a ctypes int64[3], dims, float32 origin as
        a ctypes float[3])."""
        n, k, vol_bnds = self._box(vol_bnds, what)
        dims = np.ceil((vol_bnds[:, 1] - vol_bnds[:, 0]) / self._voxel_size).astype(int)          # TSDFVolume's (:50, :52)
        origin = vol_bnds[:, 0].astype(np.float32)
        if np.any(dims >= 2 ** 31) or float(np.prod(np.maximum(dims, 0).astype(np.float64))) >= 2.0 ** 61:
            raise ValueError("SparseTSDFVolume.%s: a box of %s voxels is too large (each dimension < 2^31, at most 2^61 voxels)"
                             % (what, dims.tolist()))
        return (n, (ctypes.c_longlong * 3)(*[int(v) for v in k]), [int(d) for d in dims],
                (ctypes.c_float * 3)(*[float(v) for v in origin]))

    def _state(self):
        return (self._keys.data_ptr(), self._slots.data_ptr(), int(self._keys.numel()), self._coords.data_ptr(), self.capacity,
                self._counters.data_ptr())

    def get_mesh_tensors(self, vol_bnds=None):
        """Marching cubes over vol_bnds (to_dense's box, by default the allocated blocks' bounding box) on the blocks: exactly
        to_dense(vol_bnds).get_mesh_tensors() -- the same vertices, faces, normals and colours in the same order -- without the
        dense box.  Scratch and outputs scale with the allocated blocks and the mesh.  Synchronises to read the block count and,
        as TSDFVolume's, once between the count and the extract launches."""
        n, k, dims, origin = self._view_box(vol_bnds, "get_mesh")
        dev = self.device
        with self._device_scope():
            if n == 0 or min(dims) < 2:
                return (torch.empty((0, 3), dtype=torch.float32, device=dev), torch.empty((0, 3), dtype=torch.int32, device=dev),
                        torch.empty((0, 3), dtype=torch.float32, device=dev), torch.empty((0, 3), dtype=torch.uint8, device=dev))
            nbytes = ctypes.c_longlong(0)
            N.check(N.lib().dvmvs_tsdf_sparse_mesh_scratch_bytes(n, ctypes.byref(nbytes)), "tsdf_sparse_mesh_scratch_bytes")
            scratch = torch.empty(max(int(nbytes.value), 16), dtype=torch.uint8, device=dev)
            stream = _stream()
            N.check(N.lib().dvmvs_tsdf_sparse_mesh_count(*self._state(), self._tsdf.data_ptr(), n, k, dims[0], dims[1], dims[2],
                                                         scratch.data_ptr(), scratch.numel(), stream), "tsdf_sparse_mesh_count")
            n_verts, n_faces = (int(v) for v in scratch[:16].view(torch.int64).cpu())        # the one read between the passes
            if n_verts >= 2 ** 31 or 3 * n_faces >= 2 ** 31:
                raise RuntimeError("SparseTSDFVolume.get_mesh: a mesh of %d vertices and %d faces exceeds the int32 indices"
                                   % (n_verts, n_faces))
            verts = torch.empty((n_verts, 3), dtype=torch.float32, device=dev)
            norms = torch.empty((n_verts, 3), dtype=torch.float32, device=dev)
            colors = torch.empty((n_verts, 3), dtype=torch.uint8, device=dev)
            faces = torch.empty((n_faces, 3), dtype=torch.int32, device=dev)
            keys = torch.empty(max(n_verts + 3 * n_faces, 1), dtype=torch.int64, device=dev)
            N.check(N.lib().dvmvs_tsdf_sparse_mesh_extract(
                *self._state(), self._tsdf.data_ptr(), self._color.data_ptr(), n, k, dims[0], dims[1], dims[2], origin,
                self._voxel_size, scratch.data_ptr(), scratch.numel(), n_verts, n_faces, keys.data_ptr(), verts.data_ptr(),
                faces.data_ptr(), norms.data_ptr(), colors.data_ptr(), stream), "tsdf_sparse_mesh_extract")
        return verts, faces, norms, colors

    def get_mesh(self, vol_bnds=None):
        """get_mesh_tensors copied to the host: (verts, faces, norms, colors) numpy arrays, as TSDFVolume.get_mesh."""
        return tuple(t.cpu().numpy() for t in self.get_mesh_tensors(vol_bnds))

    def get_point_cloud(self, vol_bnds=None):
        """as TSDFVolume.get_point_cloud: (V,6) vertices and colours."""
        verts, _, _, colors = self.get_mesh(vol_bnds)
        return np.hstack([verts, colors])

    def render_tensors(self, cam_intr, cam_poses, height, width, vol_bnds=None):
        """Ray-cast over vol_bnds (to_dense's box, by default the allocated blocks' bounding box) on the blocks: exactly
        to_dense(vol_bnds).render_tensors(cam_intr, cam_poses, height, width) -- TSDFVolume.render_tensors' arguments, types,
        shapes and errors -- without the dense box.  One launch for all views, enqueued on torch's current stream;
        synchronises once, to read the block count."""
        with self._device_scope():
            _, k, dims, origin = self._view_box(vol_bnds, "render")
            views, n, single, height, width = self._views(cam_intr, cam_poses, height, width)
            depth = torch.empty((n, height, width), dtype=torch.float32, device=self.device)
            normals = torch.empty((n, height, width, 3), dtype=torch.float32, device=self.device)
            colors = torch.empty((n, height, width, 3), dtype=torch.uint8, device=self.device)
            N.check(N.lib().dvmvs_tsdf_sparse_raycast(
                *self._state(), self._tsdf.data_ptr(), self._color.data_ptr(), k, dims[0], dims[1], dims[2], origin,
                self._voxel_size, self._trunc_margin, views.data_ptr(), n, height, width, depth.data_ptr(), normals.data_ptr(),
                colors.data_ptr(), _stream()), "tsdf_sparse_raycast")
        if single:
            return depth[0], normals[0], colors[0]
        return depth, normals, colors

    def render(self, cam_intr, cam_poses, height, width, vol_bnds=None):
        """render_tensors copied to the host: (depth, normals, colors) numpy arrays."""
        return tuple(t.cpu().numpy() for t in self.render_tensors(cam_intr, cam_poses, height, width, vol_bnds))


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
