"""Searchlight shapes and configuration for ``brainiak_b200.fcma.mvpa_voxelselector.MVPAVoxelSelector``.

The shapes restate ``brainiak.searchlight.searchlight`` (Cube, Diamond, Ball): a boolean ``mask_`` of size
``(2r+1)^3`` that is true where the searchlight reaches.  ``Searchlight`` carries the parameters the selector reads
(``sl_rad``, ``shape``, ``min_active_voxels_proportion``); it has no MPI and no ``run_searchlight``: the selector
computes every centre itself.  A real ``brainiak.searchlight.Searchlight`` works in its place.
"""
import numpy as np

__all__ = ["Shape", "Cube", "Diamond", "Ball", "Searchlight"]


def _offsets(rad):
    """Integer offsets (di, dj, dk) from the centre of the (2r+1)^3 cube, each of shape (2r+1, 2r+1, 2r+1)."""
    ax = np.arange(2 * rad + 1) - rad
    return np.meshgrid(ax, ax, ax, indexing="ij")


class Shape:
    """A searchlight shape inside the cube of edge ``2*rad+1`` (``rad`` does not count the centre voxel)."""

    def __init__(self, rad):
        self.rad = rad


class Cube(Shape):
    """Every voxel of the cube."""

    def __init__(self, rad):
        super().__init__(rad)
        self.mask_ = np.ones((2 * rad + 1,) * 3, dtype=bool)


class Diamond(Shape):
    """The voxels at Manhattan (cityblock) distance <= rad from the centre."""

    def __init__(self, rad):
        super().__init__(rad)
        di, dj, dk = _offsets(rad)
        self.mask_ = (np.abs(di) + np.abs(dj) + np.abs(dk)) <= rad


class Ball(Shape):
    """The voxels at Euclidean distance <= rad from the centre (squared distances compared in integers)."""

    def __init__(self, rad):
        super().__init__(rad)
        di, dj, dk = _offsets(rad)
        self.mask_ = (di * di + dj * dj + dk * dk) <= rad * rad


class Searchlight:
    """Searchlight parameters, with the signature of ``brainiak.searchlight.Searchlight``.

    ``sl_rad``: radius of the cube, not counting the centre; ``shape``: a Shape class; a centre is processed only if
    the proportion of the cube that is inside both the brain mask and the shape is strictly greater than
    ``min_active_voxels_proportion`` (0 = no test).  ``max_blk_edge`` and ``pool_size`` are accepted for compatibility
    and unused.
    """

    def __init__(self, sl_rad=1, max_blk_edge=10, shape=Cube, min_active_voxels_proportion=0, pool_size=None):
        if sl_rad < 0:
            raise ValueError("sl_rad should not be negative")
        if max_blk_edge <= 0:
            raise ValueError("max_blk_edge should be positive")
        self.sl_rad = sl_rad
        self.max_blk_edge = max_blk_edge
        self.min_active_voxels_proportion = min_active_voxels_proportion
        self.shape = shape(sl_rad).mask_
        self.pool_size = pool_size
