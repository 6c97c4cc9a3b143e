"""Keeping a saved map current (malio_world_voxel_seed* and the changes, include/malio_b200.h) restated on top of
tests/world_voxel_ref.py and tests/carve_ref.py:
  seed       an empty map folds the n points {x, y, z, intensity} in input order, in chunks of at most `chunk` points, exactly
             as one accumulate of the whole cloud; every voxel it creates is seeded and starts at hit = seed_hits, miss = 0
  changes    removed = the seeded voxels the keep rule drops, added = the voxels not seeded that it keeps, each as centroids in
             ascending (k, j, i) order
`variant` plants the mistakes the GPU comparison must catch: "carve_zeroes" (the first carve zeroes the counters again),
"added_all" (added = every kept voxel, seeded ones included), "reversed_chunks" (the chunks folded last to first) and
"removed_before_seed" (the keep rule for removed applied to the session's hits alone, without the seed's)."""
import numpy as np

import carve_ref as CR
import world_voxel_ref as V

F = np.float32
SEED_CHUNK = 1 << 22   # MALIO_SEED_CHUNK


class StateError(ValueError):
    """A seed into a map that is not empty (MALIO_ERR_STATE)."""


class SeedMapRef(CR.CarveMapRef):
    """CarveMapRef with a seeded set."""

    def __init__(self, variant=""):
        super().__init__()
        self.variant = variant
        self.seeded = set()
        self.seed_hits = 0
        self.carved = False

    def seed(self, xyzi, leaf, seed_hits, chunk=SEED_CHUNK) -> int:
        if self.sums or self.leaf is not None:
            raise StateError("the voxel map is not empty")
        xyzi = np.ascontiguousarray(xyzi, F).reshape(-1, 4)
        if not (np.isfinite(F(leaf)) and F(leaf) > 0) or xyzi.shape[0] == 0:
            raise ValueError("leaf or n")
        _, finite, in_int = V.voxel_index(xyzi[:, :3], leaf)
        if np.any(finite & ~in_int):                   # refused before any chunk: the map stays empty
            raise V.CapacityError("voxel index outside int")
        parts = [xyzi[a:a + chunk] for a in range(0, xyzi.shape[0], chunk)]
        if self.variant == "reversed_chunks":
            parts = parts[::-1]
        for p in parts:
            self.accumulate_fast(p, leaf)
        self.leaf = F(leaf)
        self.seeded = set(self.sums)
        self.seed_hits = int(seed_hits)
        for k in self.seeded:
            self.hit[k], self.miss[k] = self.seed_hits, 0
        return len(self.sums)

    def accumulate(self, cloud, leaf) -> int:
        n = self.accumulate_fast(cloud, leaf)
        for k in self.sums:
            self.hit.setdefault(k, 0)
            self.miss.setdefault(k, 0)
        return n

    def accumulate_carve(self, cloud, slot_sizes, origins, leaf, max_range, end_margin, variant="") -> int:
        if self.variant == "carve_zeroes" and not self.carved:
            for k in self.sums:
                self.hit[k], self.miss[k] = 0, 0
        self.carved = True
        return super().accumulate_carve(cloud, slot_sizes, origins, leaf, max_range, end_margin, variant)

    def clear(self):
        self.__init__(self.variant)

    def change_masks(self, min_miss, max_miss_per_hit):
        """(seeded, kept, removed, added) as bool arrays in ascending (k, j, i) order."""
        keys = sorted(self.sums)
        seeded = np.array([k in self.seeded for k in keys], bool)
        kept = self.kept_mask(min_miss, max_miss_per_hit).reshape(-1)
        if self.variant == "removed_before_seed":
            gone = np.array([CR.dropped(self.hit[k] - (self.seed_hits if k in self.seeded else 0), self.miss[k], min_miss,
                                        max_miss_per_hit) for k in keys], bool)
            removed = seeded & gone
        else:
            removed = seeded & ~kept
        added = kept.copy() if self.variant == "added_all" else ~seeded & kept
        return seeded, kept, removed, added

    def changes(self, min_miss, max_miss_per_hit):
        """(removed, added) centroids float32 (m, 4) in ascending (k, j, i) order."""
        _, _, removed, added = self.change_masks(min_miss, max_miss_per_hit)
        c = self.centroids()
        return c[removed], c[added]
