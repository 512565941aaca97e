"""Axis-aligned boxes in objective space, and a queue of boxes kept in order of volume (IPRO-2D's open boxes).

Same attributes, methods and comparisons as the reference's ``Box`` (multi_policy/ipro/box.py).  ``BoxQueue`` replaces the
``sortedcontainers.SortedKeyList`` keyed by ``Box.volume`` that IPRO-2D keeps, with the same ordering of equal keys.
"""

from __future__ import annotations

import bisect

import numpy as np


class Box:
    """The box spanned by two corner points, in any dimension."""

    def __init__(self, point1, point2):
        self.dimensions = len(point1)
        self.bounds = np.array([point1, point2])
        self.nadir = np.min(self.bounds, axis=0)
        self.ideal = np.max(self.bounds, axis=0)
        self.midpoint = (self.nadir + self.ideal) / 2
        self.volume = self.compute_volume()
        self.max_dist = np.max(self.ideal - self.nadir)

    def compute_volume(self):
        """Product of the side lengths."""
        return abs(np.prod(self.ideal - self.nadir))

    def get_intersecting_box(self, box):
        """The intersection with ``box`` as a Box, or None when the interiors do not meet."""
        if not self.is_intersecting(box):
            return None
        return Box(np.max([self.nadir, box.nadir], axis=0), np.min([self.ideal, box.ideal], axis=0))

    def is_intersecting(self, box):
        """Whether the open boxes overlap: their ranges overlap strictly in every dimension."""
        return np.all((self.nadir < box.ideal) & (box.nadir < self.ideal))

    def is_intersecting_with_boundary(self, box):
        """Whether the closed ranges overlap in at least one dimension (the reference's test, kept as it is)."""
        return np.any((self.nadir <= box.ideal) & (box.nadir <= self.ideal))

    def projection_is_intersecting(self, box, dim):
        """Whether the open boxes overlap once dimension ``dim`` is dropped."""
        lo, hi, blo, bhi = (np.delete(v, dim) for v in (self.nadir, self.ideal, box.nadir, box.ideal))
        return np.all((lo < bhi) & (blo < hi))

    def contains(self, point):
        """Whether ``point`` lies in the closed box."""
        return np.all((self.nadir <= point) & (point <= self.ideal))

    def contains_inner(self, point):
        """Whether ``point`` lies in the open box."""
        return np.all((self.nadir < point) & (point < self.ideal))

    def vertices(self):
        """The 2^d corners as tuples; bit j of the corner's index picks the ideal (set) or the nadir (clear) in dimension j."""
        return [tuple(self.ideal[j] if (i >> j) & 1 else self.nadir[j] for j in range(self.dimensions)) for i in range(2**self.dimensions)]

    def __repr__(self):
        return f"Box({self.nadir}, {self.ideal})"


class BoxQueue:
    """Boxes in ascending order of volume.  ``add`` places a box after those of equal volume, so the box at ``[-1]`` is the largest and,
    among equal volumes, the latest added.  Supports ``pop(idx)``, indexing, ``len``, truthiness, iteration and ``copy.deepcopy``."""

    def __init__(self, boxes=()):
        self._boxes, self._keys = [], []
        for b in boxes:
            self.add(b)

    def add(self, box: Box):
        i = bisect.bisect_right(self._keys, box.volume)
        self._keys.insert(i, box.volume)
        self._boxes.insert(i, box)

    def pop(self, idx: int = -1) -> Box:
        self._keys.pop(idx)
        return self._boxes.pop(idx)

    def __getitem__(self, idx):
        return self._boxes[idx]

    def __len__(self):
        return len(self._boxes)

    def __iter__(self):
        return iter(self._boxes)

    def __repr__(self):
        return f"BoxQueue({self._boxes})"
