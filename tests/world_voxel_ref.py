"""The saved map as a voxel map (malio_world_voxel_*, include/malio_b200.h) restated in numpy float32: every accumulated dense
registered cloud {x, y, z, intensity} folded per voxel, in accumulation order.
  voxel of a point   (int)floorf(x * il) per axis with il = float32(1) / float32(leaf); non-finite points are skipped; an index
                     outside int refuses the whole cloud (CapacityError) and leaves the map as it was
  centroid           float32 sums from 0 continued point by point across clouds, an integer count, sum / float32(count)
  order              ascending (k, j, i) = (z, y, x) voxel index
VoxelMapRef.accumulate is the contract as a loop over points.  accumulate_fast gives the same bits with the loop turned
sideways (the d-th point of every voxel at once, d = 0, 1, ...): each voxel's sum still sees its points one by one in order."""
import numpy as np

F = np.float32
_LO, _HI = F(-2147483648.0), F(2147483648.0)


class CapacityError(ValueError):
    """A finite point whose voxel index falls outside int (MALIO_ERR_CAPACITY)."""


class LeafError(ValueError):
    """A leaf other than the map's (MALIO_ERR_INVALID_ARG)."""


def voxel_index(xyz, leaf):
    """float32 (n, 3) world points -> (int64 (n, 3) voxel index (k, j, i) = (z, y, x), finite mask, in-int mask)."""
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    il = F(1.0) / F(leaf)
    with np.errstate(invalid="ignore", over="ignore"):
        f = np.floor(xyz * il)
        finite = np.isfinite(xyz).all(axis=1)
        in_int = ((f >= _LO) & (f < _HI)).all(axis=1)
    ijk = np.zeros((xyz.shape[0], 3), np.int64)
    ok = finite & in_int
    ijk[ok] = f[ok][:, ::-1].astype(np.int64)
    return ijk, finite, in_int


class VoxelMapRef:
    def __init__(self):
        self.leaf = None
        self.sums = {}   # (k, j, i) -> float32[4]
        self.cnt = {}

    def _check(self, cloud, leaf):
        cloud = np.ascontiguousarray(cloud, F).reshape(-1, 4)
        if self.leaf is not None and F(leaf) != self.leaf:
            raise LeafError(f"leaf {leaf} differs from the map's {self.leaf}")
        ijk, finite, in_int = voxel_index(cloud[:, :3], leaf)
        if np.any(finite & ~in_int):
            raise CapacityError("voxel index outside int")
        return cloud, ijk, finite

    def accumulate(self, cloud, leaf) -> int:
        """Fold one dense cloud (float32 (n, 4) {x, y, z, intensity}) in, point by point.  Returns the voxel count."""
        cloud, ijk, finite = self._check(cloud, leaf)
        for p in range(cloud.shape[0]):
            if not finite[p]:
                continue
            key = tuple(int(v) for v in ijk[p])
            s = self.sums.get(key)
            if s is None:
                s = np.zeros(4, F)
                self.sums[key] = s
                self.cnt[key] = 0
            s += cloud[p]                      # four float32 additions
            self.cnt[key] += 1
        self.leaf = F(leaf)
        return len(self.sums)

    def accumulate_fast(self, cloud, leaf) -> int:
        """accumulate() with the same bits, vectorised over voxels."""
        cloud, ijk, finite = self._check(cloud, leaf)
        pts, keys = cloud[finite], ijk[finite]
        if pts.shape[0]:
            uk, inv = np.unique(keys, axis=0, return_inverse=True)
            inv = inv.reshape(-1)
            order = np.argsort(inv, kind="stable")            # point order inside every voxel
            counts = np.bincount(inv, minlength=uk.shape[0])
            starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
            tuples = [tuple(int(v) for v in k) for k in uk]
            S = np.stack([self.sums.get(t, np.zeros(4, F)) for t in tuples]).astype(F)
            sp = pts[order]
            for d in range(int(counts.max())):
                sel = np.nonzero(counts > d)[0]
                S[sel] += sp[starts[sel] + d]
            for t, s, c in zip(tuples, S, counts):
                self.sums[t] = s.copy()
                self.cnt[t] = self.cnt.get(t, 0) + int(c)
        self.leaf = F(leaf)
        return len(self.sums)

    def clear(self):
        self.__init__()

    def centroids(self) -> np.ndarray:
        """float32 (m, 4) in ascending (k, j, i) order."""
        keys = sorted(self.sums)
        if not keys:
            return np.zeros((0, 4), F)
        S = np.stack([self.sums[k] for k in keys])
        C = np.array([self.cnt[k] for k in keys], np.int64).astype(F)
        return (S / C[:, None]).astype(F)

    def keys(self) -> np.ndarray:
        return np.array(sorted(self.sums), np.int64).reshape(-1, 3)
