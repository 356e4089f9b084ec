"""Camera models and stitching tables for the cube-map observation transformers (CubeMap2Equirect, CubeMap2Fisheye,
Equirect2CubeMap).

Every camera maps output pixels to points on the unit sphere (`unproject`) and points on the sphere to the
normalised [-1, 1] image coordinates of grid_sample with align_corners=True (`project`), with a mask of the points it
sees.  A `Stitch` assigns every output pixel to the first input camera that sees it; an input that is not assigned a
pixel gets grid value 2 there, which bilinear sampling with zero padding turns into an exact 0 on any face of 3 pixels
or more.  Everything is computed once, on the CPU, in float32 torch ops in the order the reference's
habitat_baselines ProjectionConverter uses, so the grids and depth z-factors carry the same bits.

Depth: perspective cameras measure depth along their z axis, the others from the optical centre.  A perspective
input face is multiplied by 1 / z of each pixel's ray before sampling; a perspective output by the float32
reciprocal of that factor after sampling.
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import numpy as np
import torch


def _pixel_grid(h: int, w: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(row, column) int64 index planes of an h x w image."""
    return torch.meshgrid(torch.arange(h), torch.arange(w), indexing="ij")


class Camera:
    """A camera of h x w pixels; rot maps camera coordinates to world coordinates (world = rot @ cam)."""

    depth_along_z = False

    def __init__(self, h: int, w: int, rot: Optional[torch.Tensor] = None):
        self.h, self.w = int(h), int(w)
        self.rot = None if rot is None else rot.float()

    def to_world(self, pts: torch.Tensor) -> torch.Tensor:
        if self.rot is None:
            return pts
        return torch.matmul(pts.view(-1, 3), self.rot.T).view(*pts.shape)

    def to_camera(self, pts: torch.Tensor) -> torch.Tensor:
        if self.rot is None:
            return pts
        return torch.matmul(pts.view(-1, 3), self.rot).view(*pts.shape)

    def unproject(self, rotate: bool = True) -> Tuple[torch.Tensor, torch.Tensor]:
        """([h, w, 3] unit rays of the pixels, [h, w] bool mask of the pixels inside the field of view)"""
        raise NotImplementedError

    def project(self, world: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """([..., 2] normalised image coordinates (x, y), [...] bool mask of the points this camera sees)"""
        raise NotImplementedError


class Perspective(Camera):
    """Pinhole camera with focal length max(h, w) / 2 (a 90 degree field of view across the longer side)."""

    depth_along_z = True

    def __init__(self, h: int, w: int, rot: Optional[torch.Tensor] = None):
        super().__init__(h, w, rot)
        self.f = max(self.h, self.w) / 2

    def unproject(self, rotate: bool = True):
        rows, cols = _pixel_grid(self.h, self.w)
        x = (cols + 0.5) - self.w / 2
        y = (rows + 0.5) - self.h / 2
        z = torch.full_like(x, self.f, dtype=torch.float)
        rays = torch.stack([x, y, z], dim=-1)
        rays /= torch.linalg.norm(rays, dim=-1, keepdim=True)
        seen = torch.ones(rays.shape[:2], dtype=torch.bool)
        return (self.to_world(rays) if rotate else rays), seen

    def project(self, world):
        cam = self.to_camera(world)
        img = self.f * cam / torch.abs(cam[..., 2:3])
        u = img[..., 0] + self.w / 2
        v = img[..., 1] + self.h / 2
        grid = torch.stack([2 * u / self.w - 1.0, 2 * v / self.h - 1.0], dim=-1)
        seen = (torch.abs(grid).max(-1)[0] <= 1) & (img[..., 2] > 0)
        return grid, seen


class Equirect(Camera):
    """Equirectangular panorama: longitude across the width (-pi .. pi), latitude down the height."""

    def unproject(self, rotate: bool = True):
        rows, cols = _pixel_grid(self.h, self.w)
        lon = (cols + 0.5) * 2 * np.pi / self.w - np.pi
        lat = (rows + 0.5) * np.pi / self.h - np.pi / 2
        cos_lat = torch.cos(lat)
        rays = torch.stack([cos_lat * torch.sin(lon), torch.sin(lat), cos_lat * torch.cos(lon)], dim=-1)
        seen = torch.ones(rays.shape[:2], dtype=torch.bool)
        return (self.to_world(rays) if rotate else rays), seen

    def project(self, world):
        cam = self.to_camera(world)
        x, y, z = cam[..., 0], cam[..., 1], cam[..., 2]
        lon = torch.atan2(x, z)
        lat = torch.atan2(y, torch.sqrt(x * x + z * z))
        grid = torch.stack([lon / np.pi, lat / (np.pi / 2)], dim=-1)
        return grid, torch.ones(grid.shape[:2], dtype=torch.bool)


class DoubleSphere(Camera):
    """Double-sphere fisheye (Usenko, Demmel and Cremers, 3DV 2018): centre (cx, cy), focal lengths (fx, fy), model
    parameters xi and alpha, and a field of view of fov degrees.  Only unprojection is needed here: the fisheye is
    always the output."""

    def __init__(self, h: int, w: int, fov: float, cx: float, cy: float, fx: float, fy: float, xi: float,
                 alpha: float):
        super().__init__(h, w)
        self.cos_half_fov = np.cos(fov / 180 * np.pi / 2)
        self.cx, self.cy, self.fx, self.fy, self.xi, self.alpha = cx, cy, fx, fy, xi, alpha

    def unproject(self, rotate: bool = True):
        a, xi = self.alpha, self.xi
        rows, cols = _pixel_grid(self.h, self.w)   # integer pixel positions, not centres
        mx = (cols - self.cx) / self.fx
        my = (rows - self.cy) / self.fy
        r2 = mx * mx + my * my
        mz = (1 - a * a * r2) / (a * torch.sqrt(1 - (2 * a - 1) * r2) + 1 - a)
        mz2 = mz * mz
        k = (mz * xi + torch.sqrt(mz2 + (1 - xi * xi) * r2)) / (mz2 + r2)
        rays = k.unsqueeze(-1) * torch.stack([mx, my, mz], dim=-1)
        rays[..., 2] -= xi
        seen = rays[..., 2] >= self.cos_half_fov
        if a > 0.5:
            seen &= r2 <= (1 / (2 * a - 1))
        return rays, seen


# Face order Back, Down, Front, Left, Right, Up; world = R @ camera (rotations by 180 about y, -90 about x, none,
# -90 about y, 90 about y and 90 about x).
CUBE_FACES = ("BACK", "DOWN", "FRONT", "LEFT", "RIGHT", "UP")
_CUBE_ROTATIONS = (
    ((-1, 0, 0), (0, 1, 0), (0, 0, -1)),
    ((1, 0, 0), (0, 0, 1), (0, -1, 0)),
    ((1, 0, 0), (0, 1, 0), (0, 0, 1)),
    ((0, 0, -1), (0, 1, 0), (1, 0, 0)),
    ((0, 0, 1), (0, 1, 0), (-1, 0, 0)),
    ((1, 0, 0), (0, 0, -1), (0, 1, 0)),
)


def cube_cameras(h: int = 256, w: int = 256) -> List[Camera]:
    return [Perspective(h, w, torch.tensor(r)) for r in _CUBE_ROTATIONS]


def double_sphere_from_params(h: int, w: int, fov: float, params) -> DoubleSphere:
    """The CubeMap2Fisheye convention: params = (f, xi, alpha) with fx = fy = f * min(h, w), centre (w / 2, h / 2)."""
    if len(params) != 3:
        raise ValueError(f"fisheye params must be (f, xi, alpha), got {tuple(params)}")
    fx = params[0] * min(h, w)
    return DoubleSphere(h, w, fov, w / 2, h / 2, fx, fx, params[1], params[2])


class Stitch:
    """Resampling of `inputs` (all of one size) into `outputs` (all of one size).

    grids      [n_in, n_out, h, w, 2] float32: normalised sampling point of every output pixel in every input, 2 where
               that input is not the one assigned to the pixel
    face       [n_out, h, w] int64: the input assigned to each output pixel (the first that sees it), -1 for none
    in_zfactor [n_in, 1, Hi, Wi] or None: depth factor applied to input pixels before sampling
    out_zfactor [n_out, 1, h, w] or None: depth factor applied to output pixels after sampling
    """

    def __init__(self, inputs: List[Camera], outputs: List[Camera]):
        if len({(c.h, c.w) for c in inputs}) != 1 or len({(c.h, c.w) for c in outputs}) != 1:
            raise ValueError("all inputs, and all outputs, of a stitch must have one image size")
        self.inputs, self.outputs = list(inputs), list(outputs)
        self.in_hw = (inputs[0].h, inputs[0].w)
        self.out_hw = (outputs[0].h, outputs[0].w)
        self.in_zfactor = self._zfactor(self.inputs)
        out_z = self._zfactor(self.outputs)
        self.out_zfactor = None if out_z is None else 1 / out_z
        per_out = [self._assign(cam) for cam in self.outputs]
        self.grids = torch.stack([g for g, _ in per_out], dim=1)
        self.face = torch.stack([f for _, f in per_out], dim=0)

    def _assign(self, out_cam: Camera):
        rays, free = out_cam.unproject()
        face = torch.full(free.shape, -1, dtype=torch.int64)
        grids = []
        for i, cam in enumerate(self.inputs):
            grid, seen = cam.project(rays)
            mine = seen & free
            grid[~mine] = 2
            face[mine] = i
            free = free & ~mine
            grids.append(grid)
        return torch.stack(grids, dim=0), face

    @staticmethod
    def _zfactor(cams: List[Camera]) -> Optional[torch.Tensor]:
        """[n, 1, h, w]: 1 / z of each pixel's unit ray for z-depth cameras, 1 elsewhere; None when all are 1."""
        planes = []
        for cam in cams:
            if cam.depth_along_z:
                planes.append((1 / cam.unproject(rotate=False)[0][..., 2]).unsqueeze(0))
            else:
                planes.append(torch.full((1, cam.h, cam.w), 1.0, dtype=torch.float))
        z = torch.stack(planes)
        return None if bool((z == 1.0).all()) else z

    def table(self) -> torch.Tensor:
        """[n_out, h, w, 3] float32 (x, y, input) per output pixel: the assigned input's sampling point and its index
        (-1: no input, the pixel is 0)."""
        n_out = len(self.outputs)
        idx = self.face.clamp(min=0)                              # [n_out, h, w]
        g = self.grids.permute(1, 0, 2, 3, 4)                     # [n_out, n_in, h, w, 2]
        pt = torch.gather(g, 1, idx[:, None, :, :, None].expand(n_out, 1, *idx.shape[1:], 2))[:, 0]
        pt = torch.where((self.face >= 0)[..., None], pt, torch.zeros_like(pt))
        return torch.cat([pt, self.face.unsqueeze(-1).float()], dim=-1).contiguous()


def cube_to_equirect(h: int, w: int) -> Stitch:
    """Six 256 x 256 cube faces into an h x w panorama (the cube size is fixed; RGB faces of any size sample the
    same normalised grid)."""
    return Stitch(cube_cameras(), [Equirect(h, w)])


def cube_to_fisheye(h: int, w: int, fov: float, params) -> Stitch:
    """Six cube faces of the fisheye's size into an h x w double-sphere fisheye."""
    return Stitch(cube_cameras(h, w), [double_sphere_from_params(h, w, fov, params)])


def equirect_to_cube(h: int, w: int) -> Stitch:
    """A 256 x 512 panorama into six h x w cube faces."""
    return Stitch([Equirect(256, 512)], cube_cameras(h, w))
