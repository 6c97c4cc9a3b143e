"""numpy restatement of the 2-D occupancy grid (malio_grid_build_device, include/malio_b200.h, "a 2-D occupancy grid for
navigation"), step by step in float32 and the order-preserving u32 key, so that the device raster and ground compare byte for
byte.  No thread order enters: every step is a min, a count or a flag per cell."""
import numpy as np

F = np.float32
FREE, OCCUPIED, UNKNOWN = 0, 100, 255
EMPTY = np.uint32(0xFFFFFFFF)
GROUND_NAN = np.uint32(0x7FC00000)
MAX_BOUND = 1 << 24


class ArgumentError(ValueError):
    pass


def zkey(z):
    """Order-preserving u32 key of float32 values (-0.0 < +0.0)."""
    b = np.ascontiguousarray(z, F).view(np.uint32)
    return np.where(b & 0x80000000, ~b, b | 0x80000000).astype(np.uint32)


def zkey_inv(k):
    k = np.asarray(k, np.uint32)
    return np.where(k & 0x80000000, k & 0x7FFFFFFF, ~k).astype(np.uint32).view(F)


def columns(xyz, res):
    """Step 2: fi = floorf(x * ir), fj = floorf(y * ir), ir = 1.0f / res in float32; and the finite mask (step 1)."""
    p = np.asarray(xyz, F).reshape(-1, 4)[:, :3]
    ir = F(1.0) / F(res)
    finite = np.all(np.isfinite(p), axis=1)
    with np.errstate(over="ignore", invalid="ignore"):
        fi = np.floor(p[:, 0] * ir).astype(F)
        fj = np.floor(p[:, 1] * ir).astype(F)
    return fi, fj, finite


def check(res, i0, j0, nx, ny, w, h_lo, h_hi, min_pts):
    """The argument refusals of the header (MALIO_ERR_INVALID_ARG)."""
    res, h_lo, h_hi = F(res), F(h_lo), F(h_hi)
    if not (np.isfinite(res) and res > 0):
        raise ArgumentError("res")
    if nx == 0 or ny == 0:
        raise ArgumentError("nx, ny")
    if not (np.isfinite(h_lo) and np.isfinite(h_hi) and 0 < h_lo <= h_hi):
        raise ArgumentError("band")
    if min_pts == 0:
        raise ArgumentError("min_obstacle_points")
    for b in (i0 - w, i0 + nx + w, j0 - w, j0 + ny + w):
        if abs(b) > MAX_BOUND:
            raise ArgumentError("bound")


def grid(pts, res, i0, j0, nx, ny, w, h_lo, h_hi, min_pts):
    """(cls u8 (ny, nx), ground float32 (ny, nx), report dict) of the rows pts (n, 4) float32, as the header defines them."""
    check(res, i0, j0, nx, ny, w, h_lo, h_hi, min_pts)
    pts = np.asarray(pts, F).reshape(-1, 4)
    fi, fj, finite = columns(pts, res)
    z = pts[:, 2]
    pad = finite & (fi >= F(i0 - w)) & (fi < F(i0 + nx + w)) & (fj >= F(j0 - w)) & (fj < F(j0 + ny + w))
    px, py = nx + 2 * w, ny + 2 * w
    zr = np.full(px * py, EMPTY, np.uint32)                                          # step 4
    ci = (fi[pad].astype(np.int64) - (i0 - w)) + (fj[pad].astype(np.int64) - (j0 - w)) * px
    np.minimum.at(zr, ci, zkey(z[pad]))
    zr = zr.reshape(py, px)
    half = np.full((py, nx), EMPTY, np.uint32)                                       # step 5, along x then y
    for a in range(2 * w + 1):
        half = np.minimum(half, zr[:, a:a + nx])
    gk = np.full((ny, nx), EMPTY, np.uint32)
    for b in range(2 * w + 1):
        gk = np.minimum(gk, half[b:b + ny, :])
    ground = np.where(gk == EMPTY, GROUND_NAN, zkey_inv(gk).view(np.uint32)).view(F)
    reg = pad & (fi >= F(i0)) & (fi < F(i0 + nx)) & (fj >= F(j0)) & (fj < F(j0 + ny))    # step 6
    ri = fi[reg].astype(np.int64) - i0
    rj = fj[reg].astype(np.int64) - j0
    d = (z[reg] - ground[rj, ri]).astype(F)
    band = (d >= F(h_lo)) & (d <= F(h_hi))
    floor = d < F(h_lo)
    cnt = np.zeros((ny, nx), np.int64)
    np.add.at(cnt, (rj[band], ri[band]), 1)
    fl = np.zeros((ny, nx), bool)
    fl[rj[floor], ri[floor]] = True
    cls = np.where(cnt >= min_pts, OCCUPIED, np.where(fl, FREE, UNKNOWN)).astype(np.uint8)    # step 7
    rep = dict(n_used=int(pad.sum()), n_nonfinite=int((~finite).sum()), n_outside=int((finite & ~pad).sum()),
               n_occupied=int((cls == OCCUPIED).sum()), n_free=int((cls == FREE).sum()), n_unknown=int((cls == UNKNOWN).sum()),
               device_bytes=4 * (px * py + nx * py + nx * ny) + 64)
    return cls, ground, rep


def extent(pts, res):
    """(imin, jmin, imax, jmax) of the finite rows' columns, (0, 0, -1, -1) without one; ValueError beyond 2^24."""
    fi, fj, finite = columns(pts, res)
    if not finite.any():
        return (0, 0, -1, -1)
    fi, fj = fi[finite], fj[finite]
    if np.any(np.abs(fi) > MAX_BOUND) or np.any(np.abs(fj) > MAX_BOUND):
        raise ValueError("a column index beyond 2^24")
    return (int(fi.min()), int(fj.min()), int(fi.max()), int(fj.max()))


def pgm_values(cls):
    """map_saver's trinary values of a class raster, rows flipped so that the first row is the largest y."""
    v = np.where(cls == OCCUPIED, 0, np.where(cls == FREE, 254, 205)).astype(np.uint8)
    return v[::-1]


def decode(pgm, occupied_thresh=0.65, free_thresh=0.196):
    """map_server's trinary load of PGM values (file row order): p = (255 - v) / 255; back to the class raster's row order."""
    p = (255.0 - pgm.astype(np.float64)) / 255.0
    cls = np.where(p > occupied_thresh, OCCUPIED, np.where(p < free_thresh, FREE, UNKNOWN)).astype(np.uint8)
    return cls[::-1]


def footprint(lo, hi, res, i0, j0, nx, ny, inset=0.15):
    """Region cells whose centres lie in the box [lo + inset, hi - inset) in x and y."""
    cx = (np.arange(nx) + i0 + 0.5) * res
    cy = (np.arange(ny) + j0 + 0.5) * res
    return (((cy >= lo[1] + inset) & (cy < hi[1] - inset))[:, None]) & (((cx >= lo[0] + inset) & (cx < hi[0] - inset))[None, :])


def street_fractions(st, cls, res, i0, j0, nx, ny, n_scans=20):
    """What a navigation stack needs of synth.Street's grid: parked = the share of the parked boxes' footprints (inset 0.15 m)
    occupied; road = the share of observed road cells (between the right façade's kerb at y = -7 m and the parked row, away from
    every position of the car by 0.3 m) that are free; lane_free / lane_occupied = the shares of the car's footprints over its
    first 11 scans (a trail the drive has long passed) that are free / occupied.  Boxes within 10 m of the drive only."""
    x_lo, x_hi = st.ego(0)[0] - 10.0, st.ego(n_scans - 1)[0] + 10.0
    box = lambda lo, hi, inset=0.15: footprint(lo, hi, res, i0, j0, nx, ny, inset)
    parked = np.zeros(cls.shape, bool)
    for lo, hi in st.parked():
        if lo[0] >= x_lo and hi[0] <= x_hi:
            parked |= box(lo, hi)
    cars = np.zeros(cls.shape, bool)
    for k in range(n_scans):
        lo, hi = st.car(k)
        cars |= box(lo - 0.3, hi + 0.3, 0.0)
    lane = np.zeros(cls.shape, bool)
    for k in range(11):
        lo, hi = st.car(k)
        if lo[0] >= x_lo and hi[0] <= x_hi:
            lane |= box(lo, hi)
    road = box(np.array([x_lo, -st.half_width + 1.0]), np.array([x_hi, 4.0]), 0.0) & ~cars & (cls != UNKNOWN)
    return dict(parked=float(np.mean(cls[parked] == OCCUPIED)), road=float(np.mean(cls[road] == FREE)),
                lane_free=float(np.mean(cls[lane] == FREE)), lane_occupied=float(np.mean(cls[lane] == OCCUPIED)))
