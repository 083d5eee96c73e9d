"""Scene grids of joint-position control (DESIGN.md "Joint-position control", "Scene: obstacles and uneven ground"):
2D grids over the ground plane XZ (y is up) that JointControlSampleModel reads from y['obstacle_sdf'] and y['terrain']."""
import numpy as np
import torch


class SceneGrid:
    """A 2D grid over the ground plane: `values` [Gz, Gx] (shared by the batch) or [B, Gz, Gx] (one per sample), float
    and finite (kept as fp32), Gz, Gx >= 2; row i lies at z = z0 + i * cell and column k at x = x0 + k * cell, with
    `origin` = (x0, z0) and `cell` > 0.  The guidance samples it bilinearly: u = clamp((x - x0) / cell, 0, Gx - 1), v
    likewise in z, the cell (min(floor(v), Gz - 2), min(floor(u), Gx - 2)) and its gradient, 0 along a clamped axis.
    ValueError for anything else."""

    def __init__(self, values, origin, cell):
        if isinstance(values, np.ndarray):
            values = torch.from_numpy(values)
        if not torch.is_tensor(values) or not values.is_floating_point():
            raise ValueError("SceneGrid values must be a float tensor or array (got %r)" % type(values))
        if values.dim() not in (2, 3) or values.shape[-2] < 2 or values.shape[-1] < 2:
            raise ValueError("SceneGrid values must be [Gz, Gx] or [B, Gz, Gx] with Gz, Gx >= 2 (got %s)"
                             % (tuple(values.shape),))
        v = values.detach().to(torch.float32).contiguous()
        if not bool(torch.isfinite(v).all()):
            raise ValueError("SceneGrid values must be finite in fp32")
        o = np.asarray(origin, dtype=np.float64).reshape(-1)
        if o.shape != (2,) or not (np.abs(o) <= np.finfo(np.float32).max).all():
            raise ValueError("SceneGrid origin must be two finite numbers (x0, z0) (got %r)" % (origin,))
        c = float(cell)
        if not (np.finfo(np.float32).tiny <= c <= np.finfo(np.float32).max):
            raise ValueError("SceneGrid cell must be finite and > 0 (got %r)" % (cell,))
        self.values, self.origin, self.cell = v, (float(o[0]), float(o[1])), c

    @property
    def per_sample(self):
        """True for one grid per sample ([B, Gz, Gx])"""
        return self.values.dim() == 3

    @property
    def shape(self):
        """(Gz, Gx)"""
        return tuple(self.values.shape[-2:])

    def shard(self, lo, hi):
        """the grids of samples lo .. hi - 1 (a shared grid is returned as it is)"""
        return SceneGrid(self.values[lo:hi], self.origin, self.cell) if self.per_sample else self

    @classmethod
    def from_shapes(cls, shape, origin, cell, discs=(), boxes=()):
        """The 2D signed distance (positive outside) of a union of discs (cx, cz, radius) and axis-aligned boxes
        (xmin, zmin, xmax, zmax), sampled on a grid of `shape` (Gz, Gx) at `origin` with `cell`: shape_sdf in fp64 at
        every node, rounded to fp32."""
        gz, gx = int(shape[0]), int(shape[1])
        x = float(origin[0]) + float(cell) * np.arange(gx, dtype=np.float64)
        z = float(origin[1]) + float(cell) * np.arange(gz, dtype=np.float64)
        zz, xx = np.meshgrid(z, x, indexing="ij")
        return cls(torch.from_numpy(shape_sdf(xx, zz, discs, boxes)), origin, cell)


def shape_sdf(x, z, discs=(), boxes=()):
    """fp64 signed distance at points (x, z) (arrays of one shape) to the union of discs (cx, cz, radius) and axis-aligned
    boxes (xmin, zmin, xmax, zmax): the smallest of the shapes' signed distances.  That is the exact distance to the union
    outside every shape and inside shapes that do not overlap; inside an overlap its magnitude is the deepest single
    shape's, a lower bound on the distance to the union's boundary."""
    x, z = np.asarray(x, dtype=np.float64), np.asarray(z, dtype=np.float64)
    if not discs and not boxes:
        raise ValueError("shape_sdf needs at least one disc or box")
    d = np.full(np.broadcast(x, z).shape, np.inf)
    for cx, cz, r in discs:
        if not r > 0:
            raise ValueError("disc radius must be > 0 (got %r)" % (r,))
        d = np.minimum(d, np.hypot(x - cx, z - cz) - r)
    for x0, z0, x1, z1 in boxes:
        if not (x1 > x0 and z1 > z0):
            raise ValueError("box (%r, %r, %r, %r) needs xmin < xmax and zmin < zmax" % (x0, z0, x1, z1))
        qx = np.abs(x - 0.5 * (x0 + x1)) - 0.5 * (x1 - x0)
        qz = np.abs(z - 0.5 * (z0 + z1)) - 0.5 * (z1 - z0)
        d = np.minimum(d, np.hypot(np.maximum(qx, 0), np.maximum(qz, 0)) + np.minimum(np.maximum(qx, qz), 0))
    return d
