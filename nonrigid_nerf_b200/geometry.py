"""Triangle meshes of the scene: density grids through the fused field kernel and marching cubes on the GPU (csrc/mesh.cu).

The reference exports no geometry; these functions give the canonical mesh, the mesh of any frame in world space (the grid
points bent by that frame's latent code) and the rigidity painted onto the surface.

Grid.  `resolution` is an int or (nx, ny, nz), each at least 2.  Point (i, j, k) is (x_i, y_j, z_k) with, per axis and in
fp32, lo = float32(min), hi = float32(max), x_i = lo + (hi - lo) * (i / (n - 1)), each of the four operations rounded on its
own (no fused multiply-add), and x_{n-1} = hi exactly.  Grids are [nz, ny, nx]: x varies fastest.

Density.  sigma = relu(raw[..., 3]) of NeRF.forward in point mode at the grid point, with the model's test-time knobs
(the bender's rigidity_test_time_cutoff and test_time_scaling, the NeRF's test_time_nonrigid_object_removal_threshold).
With a ray bender and a latent code the points are bent by that latent (the frame's geometry in world space); with a bender
and latent=None the bender is off, as render_canonical turns it off (the canonical geometry).  A time-conditioned baseline
needs the latent; a view-dependent model (use_viewdirs=True) is refused.

Surface.  A grid point is occupied when sigma > threshold (NaN is not).  Each grid edge with exactly one occupied end gets
one vertex, p_a + ((t - s_a) / (s_b - s_a)) * (p_b - p_a) from its lower end a (NaN counts as 0 there), shared by every
cell around the edge.  Vertices are ordered by edge key (k, j, i, axis), faces by cell (k, j, i) and then by the cube
table's order (DESIGN.md describes its construction); face normals, by the right-hand rule, point out of the occupied region.
The result is bit-reproducible.

Memory.  The volume is meshed in z-slabs: three density planes and three planes of counts are resident, so device memory is
O(nx * ny) plus the mesh.  density_grid alone materialises the whole volume.  V and T must stay below 2^31.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
from typing import NamedTuple, Optional, Tuple

import numpy as np
import torch

from . import _lib, ops
from . import autograd as _ag

_ID_LIMIT = 2 ** 31
_ATTR_CHUNK = 1 << 22   # vertices per point-mode pass of the attributes


class Mesh(NamedTuple):
    vertices: torch.Tensor              # [V, 3] fp32
    faces: torch.Tensor                 # [T, 3] int32 vertex ids
    colors: Optional[torch.Tensor]      # [V, 3] uint8 to8b(sigmoid(raw[:3])) at each vertex
    rigidity: Optional[torch.Tensor]    # [V] fp32 the bender's rigidity at each vertex (None: no bender, or canonical)
    vertex_offsets: np.ndarray          # [nz + 1] int64: the vertices of z-plane k's edges are rows vertex_offsets[k]..[k+1]
    face_offsets: np.ndarray            # [nz] int64: the faces of cell layer k (between planes k, k + 1) start at face_offsets[k]; [-1] = T


def _resolution(resolution):
    r = (resolution,) * 3 if isinstance(resolution, (int, np.integer)) else tuple(resolution)
    if len(r) != 3 or any(not isinstance(n, (int, np.integer)) or isinstance(n, bool) for n in r):
        raise RuntimeError(f"nonrigid_nerf_b200: resolution must be an int or (nx, ny, nz), got {resolution!r}")
    if any(n < 2 for n in r):
        raise RuntimeError(f"nonrigid_nerf_b200: resolution must be at least 2 on every axis, got {r}")
    if any(n > 2 ** 24 for n in r) or r[0] * r[1] > 2 ** 28:
        raise RuntimeError(f"nonrigid_nerf_b200: resolution {r} too large (at most 2^24 per axis and nx * ny <= 2^28)")
    return tuple(int(n) for n in r)


def _extent(min_point, max_point):
    """The volume extent as the fp32 values the grid is built from (host arrays the C ABI reads)."""
    lo, hi = (np.ascontiguousarray(np.asarray(p, dtype=np.float64).reshape(-1).astype(np.float32)) for p in (min_point, max_point))
    if lo.shape != (3,) or hi.shape != (3,):
        raise RuntimeError("nonrigid_nerf_b200: min_point and max_point must hold 3 values each")
    if not (np.all(np.isfinite(lo)) and np.all(np.isfinite(hi)) and np.all(hi > lo)):
        raise RuntimeError(f"nonrigid_nerf_b200: max_point {hi.tolist()} must exceed min_point {lo.tolist()} on every axis "
                           "(finite, in fp32)")
    return lo, hi


class _PointField:
    """NeRF.forward in point mode at given points, with one latent code for every point (or none)."""

    def __init__(self, network_fn, latent):
        if getattr(network_fn, "use_viewdirs", False):
            raise RuntimeError("nonrigid_nerf_b200: meshes of a view-dependent model (use_viewdirs=True) are not implemented")
        tc = _ag._tc_net(network_fn)
        bender = network_fn.ray_bender[0]
        if tc is not None and latent is None:
            raise RuntimeError("nonrigid_nerf_b200: a time_conditioned_baseline model needs the latent code of a frame")
        if tc is None and bender is None and latent is not None:
            raise RuntimeError("nonrigid_nerf_b200: a latent code was given, but the model has no ray bender")
        self.net, self.tc = network_fn, tc
        self.bent = bender is not None and latent is not None
        self.dev = network_fn.output_linear.weight.device
        if self.dev.type != "cuda":
            raise RuntimeError("nonrigid_nerf_b200: the model must be on a CUDA device (there is no CPU path)")
        self.out_ch = network_fn.output_linear.weight.shape[0]
        self.knobs = _ag._knobs(network_fn) if self.bent else (None, None, None)
        with torch.no_grad():
            self.nerf_pack = ops.pack_nerf(network_fn)
            self.bender_pack = ops.pack_bender(bender) if self.bent else None
        self.latent = None
        if latent is not None:
            lat = torch.as_tensor(latent).detach().to(device=self.dev, dtype=torch.float32).reshape(-1)
            if lat.numel() != ops.LATENT:
                raise RuntimeError(f"nonrigid_nerf_b200: the latent code must hold {ops.LATENT} values, got {lat.numel()}")
            self.latent = lat.reshape(1, ops.LATENT).contiguous()

    def __call__(self, points: torch.Tensor, want_details: bool = False):
        """raw [P, out_ch] and the details (point mode) at points [P, 3]."""
        lat = None if self.latent is None else self.latent.expand(points.shape[0], ops.LATENT)
        raw, det = ops.field_forward_points(points, lat, self.nerf_pack, self.bender_pack, self.out_ch, *self.knobs,
                                            want_details=want_details, tc_net=self.tc)
        return raw.view(points.shape[0], self.out_ch), det


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _density_plane(field: _PointField, lo, hi, n3, k, points: torch.Tensor, out: torch.Tensor) -> None:
    """sigma of z-plane k into out [ny, nx] (points: a [ny * nx, 3] scratch buffer)."""
    lib = _lib.load()
    nx, ny, nz = n3
    _lib.check(lib.nrn_mesh_grid_points(lo.ctypes.data, hi.ctypes.data, nx, ny, nz, k, points.data_ptr(), _stream()), "mesh_grid_points")
    raw, _ = field(points)
    _lib.check(lib.nrn_mesh_sigma(raw.data_ptr(), nx * ny, field.out_ch, out.data_ptr(), _stream()), "mesh_sigma")


def density_grid(network_fn, min_point, max_point, resolution, latent=None) -> torch.Tensor:
    """sigma [nz, ny, nx] fp32 on the model's device: relu(raw[..., 3]) of NeRF.forward (point mode) at every grid point."""
    nx, ny, nz = _resolution(resolution)
    lo, hi = _extent(min_point, max_point)
    field = _PointField(network_fn, latent)
    with torch.cuda.device(field.dev), torch.no_grad():
        sigma = torch.empty(nz, ny, nx, dtype=torch.float32, device=field.dev)
        points = torch.empty(ny * nx, 3, dtype=torch.float32, device=field.dev)
        for k in range(nz):
            _density_plane(field, lo, hi, (nx, ny, nz), k, points, sigma[k])
    return sigma


def _grow(buf: torch.Tensor, used: int, need: int) -> torch.Tensor:
    if need <= buf.shape[0]:
        return buf
    new = torch.empty((max(need, 2 * buf.shape[0]),) + tuple(buf.shape[1:]), dtype=buf.dtype, device=buf.device)
    new[:used].copy_(buf[:used])
    return new


def _march(dev, n3, lo, hi, threshold: float, plane):
    """Marching cubes over the planes plane(0), plane(1), ... (each [ny, nx] fp32, asked for once and in order; a plane
    must stay valid until plane(k + 3) is asked for).  Returns (vertices, faces, vertex_offsets, face_offsets)."""
    lib = _lib.load()
    nx, ny, nz = n3
    t = float(np.float32(threshold))
    if t != t:
        raise RuntimeError("nonrigid_nerf_b200: threshold is NaN")
    ws = torch.empty(lib.nrn_mesh_workspace_bytes(nx, ny), dtype=torch.uint8, device=dev)
    totals = torch.zeros(3, 2, dtype=torch.int32, device=dev)
    totals_host = torch.zeros(3, 2, dtype=torch.int32).pin_memory()
    done = [torch.cuda.Event() for _ in range(3)]
    sig = {0: plane(0), 1: plane(1)}

    def args(k):
        a = _lib.NrnMeshSlabArgs()
        a.sigma0, a.sigma1 = sig[k].data_ptr(), (sig[k + 1].data_ptr() if k + 1 < nz else None)
        a.min_point, a.max_point = lo.ctypes.data, hi.ctypes.data
        a.threshold, a.nx, a.ny, a.nz, a.k = t, nx, ny, nz, k
        a.workspace, a.stream = ws.data_ptr(), _stream()
        return a

    def count(k):
        a = args(k)
        a.totals = totals[k % 3].data_ptr()
        _lib.check(lib.nrn_mesh_count(C.byref(a)), "mesh_count")
        totals_host[k % 3].copy_(totals[k % 3], non_blocking=True)
        done[k % 3].record()

    verts = torch.empty(max(1024, 2 * nx * ny), 3, dtype=torch.float32, device=dev)
    faces = torch.empty(max(1024, 4 * nx * ny), 3, dtype=torch.int32, device=dev)
    voff, foff, nf_prev = [0], [0], 0
    count(0)
    for k in range(nz):
        if k + 2 < nz:
            sig.pop(k - 1, None)
            sig[k + 2] = plane(k + 2)
        if k + 1 < nz:
            count(k + 1)          # enqueued before waiting for plane k's totals: the device keeps working meanwhile
        done[k % 3].synchronize()
        nv, nf = (int(x) for x in totals_host[k % 3].tolist())
        v_end, f_end = voff[k] + nv, foff[-1] + (nf_prev if k > 0 else 0)
        if v_end >= _ID_LIMIT or f_end >= _ID_LIMIT:
            raise RuntimeError(f"nonrigid_nerf_b200: the mesh would have {v_end} vertices and {f_end} faces by plane {k}; "
                               "V and T must stay below 2^31 (lower the resolution)")
        verts = _grow(verts, voff[k], v_end)
        faces = _grow(faces, foff[-1], f_end)
        a = args(k)
        a.vertex_base_prev, a.vertex_base = voff[k - 1] if k > 0 else 0, voff[k]
        a.face_base = foff[-1]
        a.vertices, a.faces = verts.data_ptr(), faces.data_ptr()
        _lib.check(lib.nrn_mesh_emit(C.byref(a)), "mesh_emit")
        voff.append(v_end)
        if k > 0:
            foff.append(f_end)
        nf_prev = nf
    v, f = voff[-1], foff[-1]
    verts = verts[:v] if verts.shape[0] == v else verts[:v].clone()
    faces = faces[:f] if faces.shape[0] == f else faces[:f].clone()
    return verts, faces, np.array(voff, dtype=np.int64), np.array(foff, dtype=np.int64)


def marching_cubes(sigma: torch.Tensor, min_point, max_point, threshold: float) -> Mesh:
    """The surface sigma = threshold of a density grid sigma [nz, ny, nx] (fp32 CUDA) whose points span min_point ..
    max_point as density_grid's do.  colors and rigidity are None."""
    if not isinstance(sigma, torch.Tensor) or not sigma.is_cuda:
        raise RuntimeError("nonrigid_nerf_b200: sigma must be a CUDA tensor (there is no CPU path)")
    if sigma.dim() != 3:
        raise RuntimeError(f"nonrigid_nerf_b200: sigma must be [nz, ny, nx], got {tuple(sigma.shape)}")
    nz, ny, nx = sigma.shape
    _resolution((nx, ny, nz))
    lo, hi = _extent(min_point, max_point)
    sigma = sigma.float().contiguous()
    with torch.cuda.device(sigma.device):
        v, f, vo, fo = _march(sigma.device, (nx, ny, nz), lo, hi, threshold, lambda k: sigma[k])
    return Mesh(v, f, None, None, vo, fo)


def extract_mesh(network_fn, min_point, max_point, resolution, threshold: float, latent=None, colors: bool = True,
                 rigidity: bool = True) -> Mesh:
    """The surface sigma = threshold of network_fn's density over the grid, without materialising the grid: equal to
    marching_cubes(density_grid(...), ...) bit for bit.  colors: to8b(sigmoid(raw[:3])) at each vertex; rigidity: the
    bender's rigidity at each vertex (None without a bender, and for the canonical mesh).  Both come from one more
    point-mode pass over the vertices with the same latent and knobs."""
    n3 = _resolution(resolution)
    nx, ny, nz = n3
    lo, hi = _extent(min_point, max_point)
    field = _PointField(network_fn, latent)
    dev = field.dev
    with torch.cuda.device(dev), torch.no_grad():
        points = torch.empty(ny * nx, 3, dtype=torch.float32, device=dev)
        ring = [torch.empty(ny, nx, dtype=torch.float32, device=dev) for _ in range(3)]

        def plane(k):
            _density_plane(field, lo, hi, n3, k, points, ring[k % 3])
            return ring[k % 3]

        v, f, vo, fo = _march(dev, n3, lo, hi, threshold, plane)
        col = torch.empty(v.shape[0], 3, dtype=torch.uint8, device=dev) if colors else None
        rig = torch.empty(v.shape[0], dtype=torch.float32, device=dev) if rigidity and field.bent else None
        if col is not None or rig is not None:
            for c0 in range(0, v.shape[0], _ATTR_CHUNK):
                c1 = min(c0 + _ATTR_CHUNK, v.shape[0])
                raw, det = field(v[c0:c1], want_details=rig is not None)
                if col is not None:
                    _lib.check(_lib.load().nrn_mesh_colors(raw.data_ptr(), c1 - c0, field.out_ch, col[c0:c1].data_ptr(), _stream()),
                               "mesh_colors")
                if rig is not None:
                    rig[c0:c1].copy_(det["rigidity_mask"].view(-1))
    return Mesh(v, f, col, rig, vo, fo)


# ---- occupancy grids ------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True, eq=False)
class OccupancyGrid:
    """Which cells of the canonical volume may hold density, for render(..., occupancy=grid).  nx * ny * nz cells over
    [min_point, max_point]; cell (i, j, k) is bit c % 32 of word c // 32 of `bits`, c = (k * ny + j) * nx + i.  A sample is
    evaluated when its (bent) point lies in an occupied cell, outside the box, or has a non-finite coordinate; its cell is
    min(floor(fl(fl(x - min) * scale)), n - 1) per axis with scale = fl(n / fl(max - min)), all in fp32.  Not a tuple, so
    the ray-sharded render wrapper hands it to every rank as it is."""
    bits: torch.Tensor                 # [ceil(nx * ny * nz / 32)] int32 on the model's device
    min_point: np.ndarray              # [3] float32
    max_point: np.ndarray              # [3] float32
    resolution: Tuple[int, int, int]   # (nx, ny, nz) cells

    def c_struct(self, device) -> "_lib.NrnOccupancyGrid":
        """The grid as the C ABI reads it; raises unless the bits are a contiguous int32 tensor of the right length on `device`."""
        nx, ny, nz = self.resolution
        words = _lib.load().nrn_occupancy_words(nx, ny, nz)
        b = self.bits
        if not (isinstance(b, torch.Tensor) and b.dtype == torch.int32 and b.dim() == 1 and b.is_contiguous() and b.numel() == words):
            raise RuntimeError(f"nonrigid_nerf_b200: occupancy bits must be a contiguous [{words}] int32 tensor for resolution "
                               f"{self.resolution}")
        if b.device != torch.device(device):
            raise RuntimeError(f"nonrigid_nerf_b200: the occupancy grid is on {b.device}, the rays on {device}")
        g = _lib.NrnOccupancyGrid()
        g.bits, g.nx, g.ny, g.nz = b.data_ptr(), nx, ny, nz
        g.min_point[:] = [float(v) for v in self.min_point]
        g.max_point[:] = [float(v) for v in self.max_point]
        return g

    def occupied_fraction(self) -> float:
        """The fraction of cells marked occupied (reads the bits back to the host)."""
        nx, ny, nz = self.resolution
        words = self.bits.cpu().numpy().view(np.uint8)
        return float(np.unpackbits(words, bitorder="little")[:nx * ny * nz].sum()) / (nx * ny * nz)


def _cells(resolution):
    r = (resolution,) * 3 if isinstance(resolution, (int, np.integer)) else tuple(resolution)
    if len(r) != 3 or any(not isinstance(n, (int, np.integer)) or isinstance(n, bool) for n in r):
        raise RuntimeError(f"nonrigid_nerf_b200: resolution must be an int or (nx, ny, nz) cells, got {resolution!r}")
    if any(n < 1 or n > 4096 for n in r):
        raise RuntimeError(f"nonrigid_nerf_b200: occupancy resolution must be 1..4096 cells on every axis, got {r}")
    return tuple(int(n) for n in r)


def occupancy_from_sigma(sigma: torch.Tensor, min_point, max_point, threshold: float, dilation: int = 1) -> OccupancyGrid:
    """The occupancy grid of densities sigma [nz + 1, ny + 1, nx + 1] (fp32 CUDA) at the corners of nx * ny * nz cells
    spanning min_point .. max_point, as density_grid lays them out: a cell is occupied when any of its 8 corners has
    sigma > threshold or NaN, and the occupied set is then dilated by `dilation` cells (Chebyshev distance)."""
    if not isinstance(sigma, torch.Tensor) or not sigma.is_cuda or sigma.dim() != 3:
        raise RuntimeError("nonrigid_nerf_b200: sigma must be a [nz + 1, ny + 1, nx + 1] CUDA tensor (there is no CPU path)")
    nx, ny, nz = _cells((sigma.shape[2] - 1, sigma.shape[1] - 1, sigma.shape[0] - 1))
    lo, hi = _extent(min_point, max_point)
    if isinstance(dilation, bool) or not isinstance(dilation, (int, np.integer)) or not 0 <= dilation <= 4096:
        raise RuntimeError(f"nonrigid_nerf_b200: dilation must be an int in 0..4096, got {dilation!r}")
    t = float(np.float32(threshold))
    if t != t:
        raise RuntimeError("nonrigid_nerf_b200: threshold is NaN")
    lib = _lib.load()
    sigma = sigma.float().contiguous()
    dev = sigma.device
    bits = torch.empty(lib.nrn_occupancy_words(nx, ny, nz), dtype=torch.int32, device=dev)
    ws = torch.empty(lib.nrn_occupancy_build_workspace_bytes(nx, ny, nz), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.nrn_occupancy_build(sigma.data_ptr(), nx, ny, nz, t, int(dilation), ws.data_ptr(), bits.data_ptr(), _stream()),
                   "occupancy_build")
    return OccupancyGrid(bits, lo, hi, (nx, ny, nz))


def occupancy_grid(network_fn, min_point, max_point, resolution, threshold: float, dilation: int = 1) -> OccupancyGrid:
    """The occupancy grid of network_fn's canonical density (the bender off, as render_canonical renders) on
    resolution = n or (nx, ny, nz) cells over min_point .. max_point (for example the scene's min_nerf_volume_point /
    max_nerf_volume_point): occupancy_from_sigma(density_grid(network_fn, min_point, max_point, (nx + 1, ny + 1, nz + 1)),
    ...).  The model's test-time knobs of the NeRF (object removal needs a bender, so it never applies here) are as in
    density_grid.  Not implemented for use_viewdirs=True and time_conditioned_baseline=True models."""
    if getattr(network_fn, "use_viewdirs", False):
        raise RuntimeError("nonrigid_nerf_b200: occupancy grids of a view-dependent model (use_viewdirs=True) are not implemented")
    if getattr(network_fn, "time_conditioned_baseline", False):
        raise RuntimeError("nonrigid_nerf_b200: occupancy grids of a time_conditioned_baseline=True model are not implemented")
    nx, ny, nz = _cells(resolution)
    sigma = density_grid(network_fn, min_point, max_point, (nx + 1, ny + 1, nz + 1), latent=None)
    return occupancy_from_sigma(sigma, min_point, max_point, threshold, dilation)


# ---- baked canonical radiance grids ---------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True, eq=False)
class RadianceGrid:
    """The canonical model's raw, baked for render(..., baked=BakedScene(grid, ...)).  nx * ny * nz vertices over
    [min_point, max_point]; values[k, j, i] holds raw[0:4] at density_grid's point (i, j, k) as fp16.  A sample whose (bent)
    point is finite and inside the box takes raw from the trilinear lookup (nrnerf_b200.h gives the fp32 rule), every
    other sample from the NeRF trunk."""
    values: torch.Tensor               # [nz, ny, nx, 4] fp16 on the model's device
    min_point: np.ndarray              # [3] float32
    max_point: np.ndarray              # [3] float32
    resolution: Tuple[int, int, int]   # (nx, ny, nz) vertices

    def c_struct(self, device) -> "_lib.NrnRadianceGrid":
        """The grid as the C ABI reads it; raises unless the values are a contiguous [nz, ny, nx, 4] fp16 tensor on `device`."""
        nx, ny, nz = self.resolution
        v = self.values
        if not (isinstance(v, torch.Tensor) and v.dtype == torch.float16 and tuple(v.shape) == (nz, ny, nx, 4) and v.is_contiguous()):
            raise RuntimeError(f"nonrigid_nerf_b200: radiance grid values must be a contiguous [{nz}, {ny}, {nx}, 4] float16 tensor "
                               f"for resolution {self.resolution}")
        if v.device != torch.device(device):
            raise RuntimeError(f"nonrigid_nerf_b200: the radiance grid is on {v.device}, the rays on {device}")
        g = _lib.NrnRadianceGrid()
        g.values, g.nx, g.ny, g.nz = v.data_ptr(), nx, ny, nz
        g.min_point[:] = [float(x) for x in self.min_point]
        g.max_point[:] = [float(x) for x in self.max_point]
        return g


@dataclasses.dataclass(frozen=True, eq=False)
class DeformationGrid:
    """The ray bender baked per frame by bake_deformation: F frames of nx * ny * nz vertices over [min_point, max_point];
    values[f, k, j, i] holds, as fp16, the bender's unmasked offset (channels 0..2) and rigidity (channel 3) at
    density_grid's point (i, j, k) with latent code latents[f], every test-time knob off.  frame(i) is what a render of
    frame i reads (BakedScene.deformation)."""
    values: torch.Tensor               # [F, nz, ny, nx, 4] fp16 on the bender's device
    min_point: np.ndarray              # [3] float32
    max_point: np.ndarray              # [3] float32
    resolution: Tuple[int, int, int]   # (nx, ny, nz) vertices
    latents: torch.Tensor              # [F, 32] fp32: the latent code of each frame

    @property
    def n_frames(self) -> int:
        return int(self.values.shape[0])

    def frame(self, i: int) -> "FrameDeformation":
        return FrameDeformation(self, i)


@dataclasses.dataclass(frozen=True, eq=False)
class FrameDeformation:
    """Frame `index` of a DeformationGrid, for render(..., baked=BakedScene(..., deformation=grid.frame(index))).  A ray whose
    every sample is finite and inside the grid's box takes its bends from the grid (trilinear lookup of offset and rigidity,
    then the bender's test-time knobs: nrnerf_b200.h gives the fp32 rule); any other ray is bent by the ray bender with its
    own latent, exactly as without the grid.  Render with frame `index`'s latent code as the rays' latents."""
    grid: DeformationGrid
    index: int

    def __post_init__(self):
        if not isinstance(self.grid, DeformationGrid):
            raise RuntimeError(f"nonrigid_nerf_b200: a FrameDeformation needs a geometry.DeformationGrid, got {type(self.grid).__name__}")
        v = self.grid.values
        if not (isinstance(v, torch.Tensor) and v.dim() == 5):   # before the index: F is values.shape[0]
            raise RuntimeError("nonrigid_nerf_b200: deformation grid values must be a contiguous [F, nz, ny, nx, 4] float16 tensor, "
                               f"got {type(v).__name__}" + (f" of shape {list(v.shape)}" if isinstance(v, torch.Tensor) else ""))
        i, n = self.index, self.grid.n_frames
        if not isinstance(i, (int, np.integer)) or isinstance(i, bool) or not 0 <= i < n:
            raise RuntimeError(f"nonrigid_nerf_b200: deformation frame {i!r} out of range ({n} frames)")

    def c_struct(self, device) -> "_lib.NrnDeformGrid":
        """The grid as the C ABI reads it; raises unless the values are a contiguous [F, nz, ny, nx, 4] fp16 tensor on
        `device`, the resolution is 2..1024 vertices per axis and the box has max > min."""
        g = self.grid
        nx, ny, nz = _vertices(g.resolution, "deformation grid")
        lo, hi = _extent(g.min_point, g.max_point)
        v = g.values
        if not (isinstance(v, torch.Tensor) and v.dtype == torch.float16 and v.dim() == 5 and tuple(v.shape[1:]) == (nz, ny, nx, 4)
                and v.is_contiguous()):
            raise RuntimeError(f"nonrigid_nerf_b200: deformation grid values must be a contiguous [F, {nz}, {ny}, {nx}, 4] float16 "
                               f"tensor for resolution {g.resolution}")
        if v.device != torch.device(device):
            raise RuntimeError(f"nonrigid_nerf_b200: the deformation grid is on {v.device}, the rays on {device}")
        c = _lib.NrnDeformGrid()
        c.values, c.nx, c.ny, c.nz, c.n_frames, c.frame = v.data_ptr(), nx, ny, nz, int(v.shape[0]), int(self.index)
        c.min_point[:] = [float(x) for x in lo]
        c.max_point[:] = [float(x) for x in hi]
        return c


@dataclasses.dataclass(frozen=True, eq=False)
class BakedScene:
    """The grids render(..., baked=scene) samples: `coarse` for the coarse pass, `fine` for the fine pass (needed when
    N_importance > 0; bake the model that pass runs), and optionally one frame's `deformation` (DeformationGrid.frame(i)),
    whose bends both passes look up in place of the ray bender.  Not a tuple, so the ray-sharded render wrapper hands it
    to every rank as it is."""
    coarse: RadianceGrid
    fine: Optional[RadianceGrid] = None
    deformation: Optional[FrameDeformation] = None


def _vertices(resolution, what="radiance grid"):
    r = (resolution,) * 3 if isinstance(resolution, (int, np.integer)) else resolution
    if not isinstance(r, (tuple, list)) or len(r) != 3 or any(not isinstance(n, (int, np.integer)) or isinstance(n, bool) for n in r):
        raise RuntimeError(f"nonrigid_nerf_b200: resolution must be an int or (nx, ny, nz) vertices, got {resolution!r}")
    if any(n < 2 or n > 1024 for n in r):
        raise RuntimeError(f"nonrigid_nerf_b200: {what} resolution must be 2..1024 vertices on every axis, got {r}")
    return tuple(int(n) for n in r)


def bake_check(network_fn) -> None:
    """Raise for a model whose raw depends on more than the canonical point: the view-dependent head and the
    time-conditioned baseline."""
    if getattr(network_fn, "use_viewdirs", False):
        raise RuntimeError("nonrigid_nerf_b200: a view-dependent model (use_viewdirs=True) cannot be baked: its raw depends on "
                           "the view direction")
    if getattr(network_fn, "time_conditioned_baseline", False):
        raise RuntimeError("nonrigid_nerf_b200: a time_conditioned_baseline=True model cannot be baked: its raw depends on the "
                           "latent code")


def bake_radiance(network_fn, min_point, max_point, resolution) -> RadianceGrid:
    """network_fn's canonical raw (the bender off, as render_canonical renders) on resolution = n or (nx, ny, nz) vertices
    (2..1024 per axis) over min_point .. max_point: the point-mode NeRF trunk at density_grid's points, z-plane by
    z-plane, stored as fp16 with round to nearest, finite values saturated to +-65504 and non-finite ones kept.  Bake the
    coarse and the fine model separately.  Not implemented for use_viewdirs=True and time_conditioned_baseline=True."""
    bake_check(network_fn)
    nx, ny, nz = _vertices(resolution)
    lo, hi = _extent(min_point, max_point)
    field = _PointField(network_fn, None)
    lib = _lib.load()
    with torch.cuda.device(field.dev), torch.no_grad():
        values = torch.empty(nz, ny, nx, 4, dtype=torch.float16, device=field.dev)
        points = torch.empty(ny * nx, 3, dtype=torch.float32, device=field.dev)
        for k in range(nz):
            _lib.check(lib.nrn_mesh_grid_points(lo.ctypes.data, hi.ctypes.data, nx, ny, nz, k, points.data_ptr(), _stream()),
                       "mesh_grid_points")
            raw, _ = field(points)
            _lib.check(lib.nrn_radiance_plane_f16(raw.data_ptr(), nx * ny, field.out_ch, values[k].data_ptr(), _stream()),
                       "radiance_plane_f16")
    return RadianceGrid(values, lo, hi, (nx, ny, nz))


def bake_deformation(ray_bender, latents, min_point, max_point, resolution) -> DeformationGrid:
    """The ray bender's unmasked offset and rigidity per frame, on resolution = n or (nx, ny, nz) vertices (2..1024 per
    axis) over min_point .. max_point (density_grid's points), for render(..., baked=BakedScene(..., deformation=
    grid.frame(i))).  latents: [F, 32] (or [32] for one frame) on the bender's device.  The bend pass of the field kernel
    runs in point mode, one z-plane and one frame at a time, with every test-time knob off (cut-off, scaling and object
    removal act at lookup, so one bake serves every setting); the values are stored as fp16 with round to nearest, finite
    values saturated to +-65504 and non-finite ones kept.  Takes 8 F nx ny nz bytes of device memory."""
    nx, ny, nz = _vertices(resolution, "deformation grid")
    lo, hi = _extent(min_point, max_point)
    params = list(ray_bender.parameters())
    dev = params[0].device if params else torch.device("cpu")
    if dev.type != "cuda":
        raise RuntimeError("nonrigid_nerf_b200: the ray bender must be on a CUDA device (there is no CPU path)")
    lat = latents.detach() if isinstance(latents, torch.Tensor) else torch.as_tensor(latents)
    if lat.dim() == 1:
        lat = lat.reshape(1, -1)
    if lat.dim() != 2 or lat.shape[1] != ops.LATENT or lat.shape[0] < 1:
        raise RuntimeError(f"nonrigid_nerf_b200: latents must be [F, {ops.LATENT}] or [{ops.LATENT}], got {list(lat.shape)}")
    if lat.device != dev:
        raise RuntimeError(f"nonrigid_nerf_b200: the latents are on {lat.device}, the ray bender on {dev}")
    lat = lat.to(torch.float32).contiguous().clone()
    lib = _lib.load()
    n_frames, n = lat.shape[0], nx * ny
    with torch.cuda.device(dev), torch.no_grad():
        bender_pack = ops.pack_bender(ray_bender)
        # ops.bend_points runs the bend pass alone, which reads no NeRF weights: a zero buffer stands in for the packed NeRF
        nerf_pack = torch.zeros(lib.nrn_packed_nerf_bytes(), dtype=torch.uint8, device=dev)
        values = torch.empty(n_frames, nz, ny, nx, 4, dtype=torch.float16, device=dev)
        points = torch.empty(n, 3, dtype=torch.float32, device=dev)
        offsets = torch.empty(n, 3, dtype=torch.float32, device=dev)
        rigidity = torch.empty(n, dtype=torch.float32, device=dev)
        workspace = torch.empty(lib.nrn_views_workspace_bytes(n, 1), dtype=torch.uint8, device=dev)
        for k in range(nz):
            _lib.check(lib.nrn_mesh_grid_points(lo.ctypes.data, hi.ctypes.data, nx, ny, nz, k, points.data_ptr(), _stream()),
                       "mesh_grid_points")
            for f in range(n_frames):
                ops.bend_points(points, lat[f:f + 1], bender_pack, nerf_pack, offsets, rigidity, workspace)
                _lib.check(lib.nrn_deformation_plane_f16(offsets.data_ptr(), rigidity.data_ptr(), n, values[f, k].data_ptr(), _stream()),
                           "deformation_plane_f16")
    return DeformationGrid(values, lo, hi, (nx, ny, nz), lat)


# ---- host-side writers --------------------------------------------------------------------------------------------------
def _host(mesh: Mesh):
    v = mesh.vertices.detach().cpu().numpy().astype("<f4", copy=False).reshape(-1, 3)
    f = mesh.faces.detach().cpu().numpy().astype("<i4", copy=False).reshape(-1, 3)
    col = None if mesh.colors is None else mesh.colors.detach().cpu().numpy().astype(np.uint8, copy=False).reshape(-1, 3)
    rig = None if mesh.rigidity is None else mesh.rigidity.detach().cpu().numpy().astype("<f4", copy=False).reshape(-1)
    return v, f, col, rig


def _host_normals(normals, n_vertices: int):
    if normals is None:
        return None
    nrm = normals.detach().cpu().numpy() if isinstance(normals, torch.Tensor) else np.asarray(normals)
    nrm = nrm.astype("<f4", copy=False).reshape(-1, 3)
    if nrm.shape[0] != n_vertices:
        raise RuntimeError(f"nonrigid_nerf_b200: normals must be [{n_vertices}, 3], got {tuple(nrm.shape)}")
    return nrm


def write_ply(path, mesh: Mesh, normals=None) -> None:
    """Binary little-endian PLY: float x, y, z (+ float nx, ny, nz when `normals` [V, 3] are given, + uchar red, green,
    blue when the mesh has colours, + float rigidity when it has rigidity) per vertex, and an int vertex_indices list of 3
    per face."""
    v, f, col, rig = _host(mesh)
    nrm = _host_normals(normals, len(v))
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    props = ["property float x", "property float y", "property float z"]
    if nrm is not None:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
        props += ["property float nx", "property float ny", "property float nz"]
    if col is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
        props += ["property uchar red", "property uchar green", "property uchar blue"]
    if rig is not None:
        fields.append(("rigidity", "<f4"))
        props.append("property float rigidity")
    vert = np.empty(len(v), dtype=fields)
    vert["x"], vert["y"], vert["z"] = v[:, 0], v[:, 1], v[:, 2]
    if nrm is not None:
        vert["nx"], vert["ny"], vert["nz"] = nrm[:, 0], nrm[:, 1], nrm[:, 2]
    if col is not None:
        vert["red"], vert["green"], vert["blue"] = col[:, 0], col[:, 1], col[:, 2]
    if rig is not None:
        vert["rigidity"] = rig
    face = np.empty(len(f), dtype=[("n", "u1"), ("v", "<i4", (3,))])
    face["n"], face["v"] = 3, f
    header = "\n".join(["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}"] + props +
                       [f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]) + "\n"
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vert.tobytes())
        fh.write(face.tobytes())


def write_obj(path, mesh: Mesh, normals=None) -> None:
    """Wavefront OBJ: 'v x y z' per vertex (+ ' r g b' in [0, 1] when the mesh has colours, c / 255), then, when `normals`
    [V, 3] are given, 'vn nx ny nz' per vertex, and 'f a b c' per face (1-based; 'f a//a b//b c//c' with normals, vertex
    i using normal i).  Numbers are written with 9 significant digits, which restore the fp32 values exactly."""
    v, f, col, _ = _host(mesh)
    nrm = _host_normals(normals, len(v))
    with open(path, "w") as fh:
        if col is None:
            np.savetxt(fh, v, fmt="v %.9g %.9g %.9g")
        else:
            np.savetxt(fh, np.concatenate([v.astype(np.float64), col / 255.0], 1), fmt="v %.9g %.9g %.9g %.9g %.9g %.9g")
        if nrm is None:
            np.savetxt(fh, f.astype(np.int64) + 1, fmt="f %d %d %d")
        else:
            np.savetxt(fh, nrm, fmt="vn %.9g %.9g %.9g")
            fi = np.repeat(f.astype(np.int64) + 1, 2, axis=1)
            np.savetxt(fh, fi, fmt="f %d//%d %d//%d %d//%d")


# ---- the inverse of the ray bender: canonical points and meshes into frames ----------------------------------------------
# Defaults of deform_points / deform_mesh (DESIGN.md, "Inverse bending", gives the measured convergence behind them)
DEFORM_ITERATIONS = 8
DEFORM_TOL = 1e-5


class Deformed(NamedTuple):
    points: torch.Tensor      # [P, 3] or [F, P, 3] fp32: x with b(x; z) = c
    residual: torch.Tensor    # [P] or [F, P] fp32: |b(x; z) - c|_2 at x
    converged: torch.Tensor   # [P] or [F, P] bool: residual <= tol
    rigidity: torch.Tensor    # [P] or [F, P] fp32: the bender's rigidity r~ at x (after the test-time cutoff)


class DeformedMesh(NamedTuple):
    mesh: Mesh                # the canonical mesh with its vertices moved into the frame, rigidity = r~ at them
    residual: torch.Tensor    # [V] fp32
    converged: torch.Tensor   # [V] bool


def deform_points(ray_bender, points: torch.Tensor, latents: torch.Tensor, iterations: int = DEFORM_ITERATIONS,
                  tol: float = DEFORM_TOL) -> Deformed:
    """Canonical points into frames: for every canonical point c (points [P, 3], CUDA) and every latent code z (latents
    [32], giving results [P, ...], or [F, 32], giving [F, P, ...]), the observed point x whose bend is c, b(x; z) = c, with
    b = ray_bender's forward including its test-time knobs (rigidity_test_time_cutoff, test_time_scaling).

    x_0 = c - s r~(c) o(c, z), then `iterations` (1..64) Newton steps on J = db/dx at fp32 accuracy (csrc/deform.cu); a point
    is frozen once |b(x) - c|_2 <= tol, and where J is singular the step is the fixed-point one.  Points that do not
    converge (the bending folds, or too few steps) keep their last x and report converged = False with their residual; a
    non-finite point or latent gives NaN.  The defaults, 8 steps and tol = 1e-5, come from the measured convergence on
    benders with offsets of 0.01 and 0.1 (DESIGN.md): tol is two orders above the fp32 evaluation error of b on the example
    volume, and 8 steps leave room over the iterations those benders need.

    Inference only: no autograd node is recorded; with parameters or inputs that require grad the call still runs, on
    detached values.  Runs on the current stream without host synchronisation (CUDA-graph capturable); a frame's results
    do not depend on the other frames of the call."""
    from .run_nerf_helpers import ray_bending
    if ray_bender is None or not isinstance(ray_bender, ray_bending):
        raise RuntimeError(f"nonrigid_nerf_b200: deform_points needs the model's ray_bending module, got {type(ray_bender).__name__}")
    if not isinstance(points, torch.Tensor) or not isinstance(latents, torch.Tensor):
        raise RuntimeError("nonrigid_nerf_b200: points and latents must be tensors")
    if points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError(f"nonrigid_nerf_b200: points must be [P, 3], got {tuple(points.shape)}")
    if latents.dim() not in (1, 2) or latents.shape[-1] != ops.LATENT:
        raise RuntimeError(f"nonrigid_nerf_b200: latents must be [{ops.LATENT}] or [F, {ops.LATENT}], got {tuple(latents.shape)}")
    if isinstance(iterations, bool) or not isinstance(iterations, (int, np.integer)) or not 1 <= iterations <= 64:
        raise RuntimeError(f"nonrigid_nerf_b200: iterations must be an int in 1..64, got {iterations!r}")
    if isinstance(tol, bool) or not isinstance(tol, (int, float, np.floating)) or not np.isfinite(tol) or tol < 0:
        raise RuntimeError(f"nonrigid_nerf_b200: tol must be a finite float >= 0, got {tol!r}")
    if not points.is_cuda or not latents.is_cuda:
        raise RuntimeError("nonrigid_nerf_b200: points and latents must be CUDA tensors (there is no CPU path)")
    dev = ray_bender.network[0].weight.device
    if points.device != dev or latents.device != dev:
        raise RuntimeError(f"nonrigid_nerf_b200: points ({points.device}) and latents ({latents.device}) must be on the bender's "
                           f"device ({dev})")
    cutoff = getattr(ray_bender, "rigidity_test_time_cutoff", None)
    scaling = getattr(ray_bender, "test_time_scaling", None)
    pts = points.detach().float().contiguous()
    lat = latents.detach().float().reshape(-1, ops.LATENT).contiguous()
    F, P = lat.shape[0], pts.shape[0]
    with torch.cuda.device(dev), torch.no_grad():
        out = torch.empty(F, P, 3, dtype=torch.float32, device=dev)
        residual = torch.empty(F, P, dtype=torch.float32, device=dev)
        converged = torch.empty(F, P, dtype=torch.bool, device=dev)
        rigidity = torch.empty(F, P, dtype=torch.float32, device=dev)
        if F > 0 and P > 0:
            pack = ops.pack_bender(ray_bender)
            a = _lib.NrnDeformArgs()
            a.points, a.n_points = pts.data_ptr(), P
            a.latents, a.n_latents, a.latent_stride = lat.data_ptr(), F, ops.LATENT
            a.bender_packed = pack.data_ptr()
            a.use_cutoff, a.rigidity_cutoff = int(cutoff is not None), float(cutoff) if cutoff is not None else 0.0
            a.use_scaling, a.scaling = int(scaling is not None), float(scaling) if scaling is not None else 1.0
            a.iterations, a.tol = int(iterations), float(tol)
            a.out, a.residual, a.converged, a.rigidity = out.data_ptr(), residual.data_ptr(), converged.data_ptr(), rigidity.data_ptr()
            a.stream = _stream()
            _lib.check(_lib.load().nrn_deform_points(C.byref(a)), "deform_points")
    if latents.dim() == 1:
        return Deformed(out[0], residual[0], converged[0], rigidity[0])
    return Deformed(out, residual, converged, rigidity)


def deform_mesh(ray_bender, mesh: Mesh, latent: torch.Tensor, iterations: int = DEFORM_ITERATIONS,
                tol: float = DEFORM_TOL) -> DeformedMesh:
    """The canonical mesh moved into the frame of `latent` ([32]): its vertices through deform_points, so every frame's
    mesh has the canonical faces and vertex order (one topology across the sequence).  faces, vertex_offsets, face_offsets
    and colors are the canonical mesh's (a canonical point's colour does not depend on the frame); rigidity is r~ at the
    moved vertices.  Vertices that did not converge keep their last iterate; `converged` tells them apart."""
    if latent is None or not isinstance(latent, torch.Tensor) or latent.dim() != 1:
        raise RuntimeError(f"nonrigid_nerf_b200: deform_mesh needs one latent code [{ops.LATENT}]")
    d = deform_points(ray_bender, mesh.vertices, latent, iterations, tol)
    return DeformedMesh(mesh._replace(vertices=d.points, rigidity=d.rigidity), d.residual, d.converged)


# ---- surface normals: the density gradient through the fused DGRAD chain (csrc/field_bwd.cu) -------------------------------
def _grad_latents(network_fn, latent, n: int, dev):
    """(latent rows [n or 1, 32] fp32, row stride) for the density gradient, after the refusals of _PointField."""
    tc = _ag._tc_net(network_fn)
    bender = network_fn.ray_bender[0]
    if tc is not None and latent is None:
        raise RuntimeError("nonrigid_nerf_b200: a time_conditioned_baseline model needs the latent code of a frame")
    if tc is None and bender is None and latent is not None:
        raise RuntimeError("nonrigid_nerf_b200: a latent code was given, but the model has no ray bender")
    if latent is None:
        return None, 0
    lat = torch.as_tensor(latent).detach().to(device=dev, dtype=torch.float32)
    if lat.dim() == 1 and lat.numel() == ops.LATENT:
        return lat.reshape(1, ops.LATENT).contiguous(), 0
    if lat.dim() == 2 and lat.shape == (n, ops.LATENT):
        return lat.contiguous(), ops.LATENT
    raise RuntimeError(f"nonrigid_nerf_b200: the latent code must be [{ops.LATENT}] or [P, {ops.LATENT}], got {tuple(lat.shape)}")


def density_gradient(network_fn, points: torch.Tensor, latent=None) -> torch.Tensor:
    """g [P, 3] fp32 = d raw[..., 3] / d x of NeRF.forward in point mode at points [P, 3] (CUDA): the gradient of the
    density before its ReLU, so points just outside the surface have one too.  With a ray bender and a latent code ([32]
    for every point, or [P, 32]) the gradient passes through the bend, bent = x + rigidity * unmasked (* scaling): the
    frame's world space.  With no latent, or no bender, it is the canonical one.  The test-time knobs apply as in point
    mode (rigidity cutoff, scaling, object removal, which zeroes g where it zeroes raw[..., 3]).  The time-conditioned
    baseline needs its latent; a view-dependent model's density is its trunk's alpha.

    One forward and one DGRAD kernel per chunk of nrn_density_gradient_chunk() points, on the current stream without host
    synchronisation (CUDA-graph capturable); the workspace is one chunk's (DESIGN.md gives its size).  Inference only: no
    autograd node is recorded.  A non-finite point gives a non-finite g."""
    return _density_gradient(network_fn, points, latent)


def _density_gradient(network_fn, points: torch.Tensor, latent=None, workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """density_gradient; `workspace` (uint8, at least nrn_density_gradient_workspace_bytes) replaces the call's own, so
    that a test can read back the last chunk's mask bits, encoding, offsets and rigidity (layout in nrnerf_b200.h)."""
    if not isinstance(points, torch.Tensor) or points.dim() != 2 or points.shape[1] != 3:
        raise RuntimeError(f"nonrigid_nerf_b200: points must be a [P, 3] tensor, got {getattr(points, 'shape', type(points))}")
    dev = network_fn.pts_linears[0].weight.device
    if dev.type != "cuda" or not points.is_cuda:
        raise RuntimeError("nonrigid_nerf_b200: the model and the points must be on a CUDA device (there is no CPU path)")
    if points.device != dev:
        raise RuntimeError(f"nonrigid_nerf_b200: points ({points.device}) must be on the model's device ({dev})")
    P = points.shape[0]
    lat, stride = _grad_latents(network_fn, latent, P, dev)
    tc = _ag._tc_net(network_fn)
    bent = network_fn.ray_bender[0] is not None and lat is not None
    cutoff, scaling, removal = _ag._knobs(network_fn) if bent else (None, None, None)
    pts = points.detach().float().contiguous()
    lib = _lib.load()
    with torch.cuda.device(dev), torch.no_grad():
        grad = torch.empty(P, 3, dtype=torch.float32, device=dev)
        if P == 0:
            return grad
        nerf_pack = ops.pack_nerf(network_fn)
        bender_pack = ops.pack_bender(network_fn.ray_bender[0]) if bent else None
        nbytes = int(lib.nrn_density_gradient_workspace_bytes(P, int(tc is not None and stride != 0)))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev) if workspace is None else workspace
        nbytes = ws.numel()
        a = _lib.NrnDensityGradArgs()
        a.points, a.n_points, a.points_stride = pts.data_ptr(), P, 3
        if lat is not None:
            a.latents, a.latent_stride = lat.data_ptr(), stride
        a.nerf_packed = nerf_pack.data_ptr()
        if bender_pack is not None:
            a.bender_packed = bender_pack.data_ptr()
        if tc is not None:
            tw = [tc.pts_linears[0].weight, tc.pts_linears[0].bias, tc.pts_linears[5].weight, tc.pts_linears[5].bias]
            for t in tw:
                if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                    raise RuntimeError("nonrigid_nerf_b200: NeRF parameters must be contiguous fp32 CUDA tensors")
            a.tc_w0, a.tc_b0, a.tc_w5, a.tc_b5 = (t.data_ptr() for t in tw)
        if cutoff is not None:
            a.use_cutoff, a.rigidity_cutoff = 1, float(cutoff)
        if scaling is not None:
            a.use_scaling, a.scaling = 1, float(scaling)
        if removal is not None:
            a.use_removal, a.removal_threshold = 1, float(removal)
        a.grad, a.workspace, a.workspace_bytes = grad.data_ptr(), ws.data_ptr(), nbytes
        a.stream = _stream()
        _lib.check(lib.nrn_field_density_gradient(C.byref(a)), "field_density_gradient")
    return grad


def normals_from_gradient(g: torch.Tensor) -> torch.Tensor:
    """Unit normals n = -g / |g| (out of the occupied region, like the mesh's face normals); n = 0 where |g| = 0 or g is
    not finite.  |g| = sqrt(gx^2 + gy^2 + gz^2) in fp32, n = -g / |g| elementwise."""
    gx, gy, gz = g[..., 0], g[..., 1], g[..., 2]
    norm = torch.sqrt(gx * gx + gy * gy + gz * gz)
    ok = torch.isfinite(norm) & (norm > 0)
    n = -g / torch.where(ok, norm, torch.ones_like(norm))[..., None]
    return torch.where(ok[..., None], n, torch.zeros_like(n))


def vertex_normals(network_fn, mesh: Mesh, latent=None) -> torch.Tensor:
    """Unit normals [V, 3] at the mesh's vertices: normals_from_gradient(density_gradient(network_fn, mesh.vertices,
    latent)).  Pass the latent the mesh was built with (extract_mesh's, or deform_mesh's for a frame's mesh)."""
    return normals_from_gradient(density_gradient(network_fn, mesh.vertices, latent))
