"""Clearing moving objects out of the voxel map (malio_world_voxel_accumulate_carve and the keep rule, include/malio_b200.h)
restated in numpy, step by step:
  ray        one per finite dense point: origin o = the slot's origin (body_to_world of (0, 0, 0)), end w = the point's world
             bits; u = o * il, e = w * il as float32 products (il = float32(1) / float32(leaf)), start cell floor(u), end cell
             floor(e)
  walk       exactly |di| + |dj| + |dk| steps; each along the axis with steps left whose next face
             ((double)c + (step > 0) - (double)u) * inv, inv = 1.0 / ((double)e - (double)u), is smallest; ties x, y, z
  passed     a visited cell other than floor(e) whose entry parameter t (0 for the start cell) has t * len < lim, with
             len = sqrt(dx*dx + dy*dy + dz*dz), d = (double)w - (double)o, lim = min(max_range, len - end_margin)
  counters   per scan: hit += 1 on every voxel a finite point lands in; miss += 1 on every voxel of the map after the fold
             that no point of the scan lands in and at least one ray passes
  keep rule  dropped when miss >= min_miss and (double)miss > (double)max_miss_per_hit * (double)hit
`variant` plants the mistakes the GPU comparison must catch: "tie_zyx" (ties broken z, y, x), "le" (t * len <= lim), "float"
(the walk in float32) and "per_ray" (a miss per passing ray instead of per scan)."""
import numpy as np

import world_voxel_ref as V

F = np.float32


def scaled(xyz, leaf):
    """float32 world coordinates -> float32 scaled coordinates, the products of the voxel key."""
    return (np.asarray(xyz, F).reshape(-1, 3) * (F(1.0) / F(leaf))).astype(F)


def walk(o, w, leaf, variant=""):
    """Every cell each ray visits, in order.  o, w float32 (n, 3).  Returns (ray, cell int64 (m, 3) as (x, y, z), t, last),
    sorted by ray then step; t is the entry parameter, last marks the end cell floor(e)."""
    T = F if variant == "float" else np.float64
    u, e = scaled(o, leaf), scaled(w, leaf)
    cell = np.floor(u).astype(np.int64)
    end = np.floor(e).astype(np.int64)
    step = np.where(end > cell, 1, -1)
    rem = np.abs(end - cell)
    up = np.where(step > 0, T(1), T(0)).astype(T)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = (T(1) / (e.astype(T) - u.astype(T))).astype(T)
    ut = u.astype(T)

    def face(c):
        with np.errstate(invalid="ignore"):
            return ((c.astype(T) + up) - ut) * inv

    tmax = np.where(rem > 0, face(cell), T(0)).astype(T)
    t = np.zeros(o.shape[0], T)
    order = [2, 1, 0] if variant == "tie_zyx" else [0, 1, 2]
    rays, cells, ts, last = [], [], [], []
    idx = np.arange(o.shape[0])
    while True:
        left = rem.sum(axis=1)
        rays.append(idx.copy()); cells.append(cell.copy()); ts.append(t.copy()); last.append(left == 0)
        act = left > 0
        if not act.any():
            break
        idx, cell, rem, tmax, t, step, up, ut, inv = (a[act] for a in (idx, cell, rem, tmax, t, step, up, ut, inv))
        a = np.full(idx.shape[0], -1)
        ta = np.zeros(idx.shape[0], T)
        for ax in order:
            take = (rem[:, ax] > 0) & ((a < 0) | (tmax[:, ax] < ta))
            a = np.where(take, ax, a)
            ta = np.where(take, tmax[:, ax], ta)
        t = ta.astype(T)
        r = np.arange(idx.shape[0])
        cell[r, a] += step[r, a]
        rem[r, a] -= 1
        tmax[r, a] = face(cell)[r, a]
    ray = np.concatenate(rays)
    srt = np.argsort(ray, kind="stable")
    return ray[srt], np.concatenate(cells)[srt], np.concatenate(ts)[srt], np.concatenate(last)[srt]


def passed(o, w, leaf, max_range, end_margin, variant=""):
    """The passed cells of each ray: (ray, cell (x, y, z))."""
    T = F if variant == "float" else np.float64
    o, w = np.asarray(o, F).reshape(-1, 3), np.asarray(w, F).reshape(-1, 3)
    d = w.astype(T) - o.astype(T)
    ln = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
    lim = np.minimum(T(max_range), ln - T(end_margin))
    ray, cell, t, last = walk(o, w, leaf, variant)
    tl = t * ln[ray]
    ok = ~last & ((tl <= lim[ray]) if variant == "le" else (tl < lim[ray]))
    return ray[ok], cell[ok]


def dropped(hit, miss, min_miss, max_miss_per_hit) -> bool:
    return miss >= min_miss and float(miss) > float(F(max_miss_per_hit)) * float(hit)


class CarveMapRef(V.VoxelMapRef):
    """VoxelMapRef with the two counters per voxel."""

    def __init__(self):
        super().__init__()
        self.hit, self.miss = {}, {}

    def accumulate(self, cloud, leaf) -> int:
        n = self.accumulate_fast(cloud, leaf)
        for k in self.sums:
            self.hit.setdefault(k, 0)
            self.miss.setdefault(k, 0)
        return n

    def accumulate_carve(self, cloud, slot_sizes, origins, leaf, max_range, end_margin, variant="") -> int:
        """cloud float32 (n, 4): the dense registered points of slots 0..L-1 concatenated; slot_sizes: their counts; origins
        float32 (L, 3): each slot's origin.  Refusals as the library's (CapacityError / LeafError), before anything changes."""
        cloud = np.ascontiguousarray(cloud, F).reshape(-1, 4)
        origins = np.asarray(origins, F).reshape(-1, 3)
        sizes = np.asarray(slot_sizes, np.int64)
        with np.errstate(invalid="ignore", over="ignore"):
            f = np.floor(scaled(origins[sizes > 0], leaf))
            if not ((f >= V._LO) & (f < V._HI)).all():
                raise V.CapacityError("ray origin outside int")
        n = self.accumulate(cloud, leaf)          # the fold (raises before changing anything)
        fin = np.isfinite(cloud[:, :3]).all(axis=1)
        o = np.repeat(origins, sizes, axis=0)[fin]
        w = cloud[fin, :3]
        hits = {tuple(int(v) for v in k) for k in V.voxel_index(w, leaf)[0]}
        for k in hits:
            self.hit[k] += 1
        ray, cell = passed(o, w, leaf, max_range, end_margin, variant)
        keys = cell[:, ::-1]
        if variant == "per_ray":
            keys = np.unique(np.concatenate([ray[:, None], keys], axis=1), axis=0)[:, 1:]
        else:
            keys = np.unique(keys, axis=0)
        for k in (tuple(int(v) for v in r) for r in keys):
            if k in self.sums and k not in hits:
                self.miss[k] += 1
        return n

    def clear(self):
        self.__init__()

    def evidence(self) -> np.ndarray:
        """uint32 (m, 2) (hit, miss) in ascending (k, j, i) order."""
        keys = sorted(self.sums)
        return np.array([(self.hit[k], self.miss[k]) for k in keys], np.uint32).reshape(-1, 2)

    def kept_mask(self, min_miss, max_miss_per_hit) -> np.ndarray:
        return np.array([not dropped(self.hit[k], self.miss[k], min_miss, max_miss_per_hit) for k in sorted(self.sums)], bool)
