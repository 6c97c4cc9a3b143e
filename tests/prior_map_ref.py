"""numpy restatement of lasermap_fov_segment (laserMapping.cpp:171-224) and of the prior-map window's contract
(malio_prior_map_window, include/malio_b200.h), with the reference's types:
  - first call: vertex_min = (float)(pos - cube_len / 2.0), vertex_max = (float)(pos + cube_len / 2.0)      (:177-185)
  - dist_to_map_edge = (float)fabs(pos - (double)vertex), MOV_THRESHOLD * DET_RANGE a float product          (:191-193)
  - mov_dist = (float)max((cube_len - 2.0 * MOV_THRESHOLD * DET_RANGE) * 0.5 * 0.9, (double)(DET_RANGE * (MOV_THRESHOLD - 1)))
  - the new vertices and the cub_needrm slabs are float subtractions / additions of mov_dist                  (:202-218)
  - boxes are half-open, min <= p < max per axis (Delete_by_range, ikd_Tree.cpp:807)
The live set the window must hold after every call is prior ∩ cube.  `variant` switches in one deliberate deviation
("strict": < for <= at :193, "double_mov": mov_dist and the vertices kept in double, "closed": boxes with p <= max) so that a
test can show it sees the difference."""
import numpy as np

F = np.float32
MOV_THRESHOLD = F(1.5)


def init_cube(pos, cube_len):
    p = np.asarray(pos, np.float64)
    return np.concatenate([(p - cube_len / 2.0).astype(F), (p + cube_len / 2.0).astype(F)])


def mov_dist(cube_len, det_range, variant=None):
    det = F(det_range)
    a = (float(cube_len) - 2.0 * float(MOV_THRESHOLD) * float(det)) * 0.5 * 0.9
    b = float(F(det * (MOV_THRESHOLD - F(1))))
    m = max(a, b)
    return m if variant == "double_mov" else F(m)


def segment(cube, pos, cube_len, det_range, variant=None):
    """One later call.  Returns (moved, new cube float32[6], slabs float32[k, 6])."""
    cube = np.asarray(cube, F)
    p = np.asarray(pos, np.float64)
    thr = F(MOV_THRESHOLD * F(det_range))
    dist = np.zeros((3, 2), F)
    need = False
    le = (lambda a, b: a < b) if variant == "strict" else (lambda a, b: a <= b)
    for i in range(3):
        dist[i, 0] = F(abs(p[i] - np.float64(cube[i])))
        dist[i, 1] = F(abs(p[i] - np.float64(cube[3 + i])))
        if le(dist[i, 0], thr) or le(dist[i, 1], thr):
            need = True
    if not need:
        return False, cube.copy(), np.zeros((0, 6), F)
    md = mov_dist(cube_len, det_range, variant)
    sub = (lambda a, b: F(np.float64(a) - b)) if variant == "double_mov" else (lambda a, b: F(a - b))
    add = (lambda a, b: F(np.float64(a) + b)) if variant == "double_mov" else (lambda a, b: F(a + b))
    new = cube.copy()
    boxes = []
    for i in range(3):
        tb = cube.copy()
        if le(dist[i, 0], thr):
            new[3 + i] = sub(new[3 + i], md); new[i] = sub(new[i], md)
            tb[i] = sub(cube[3 + i], md)
            boxes.append(tb)
        elif le(dist[i, 1], thr):
            new[3 + i] = add(new[3 + i], md); new[i] = add(new[i], md)
            tb[3 + i] = add(cube[i], md)
            boxes.append(tb)
    return True, new, np.array(boxes, F).reshape(-1, 6)


def in_box(xyz, box, variant=None):
    xyz = np.asarray(xyz, F).reshape(-1, 3)
    b = np.asarray(box, F)
    hi = (lambda v, m: v <= m) if variant == "closed" else (lambda v, m: v < m)
    return np.all((b[:3] <= xyz) & hi(xyz, b[3:]), axis=1)


def in_any(xyz, boxes, variant=None):
    m = np.zeros(np.asarray(xyz).reshape(-1, 3).shape[0], bool)
    for b in np.asarray(boxes, F).reshape(-1, 6):
        m |= in_box(xyz, b, variant)
    return m


class Window:
    """The window over a prior: the cube and the ids of prior ∩ cube after every call."""

    def __init__(self, xyz, cube_len, det_range, variant=None):
        self.xyz = np.asarray(xyz, F).reshape(-1, 3)
        self.cube_len, self.det_range, self.variant = float(cube_len), float(det_range), variant
        self.cube = None

    def step(self, pos):
        """Returns (initialized, moved, slabs)."""
        if self.cube is None:
            self.cube = init_cube(pos, self.cube_len)
            return True, False, np.zeros((0, 6), F)
        moved, self.cube, slabs = segment(self.cube, pos, self.cube_len, self.det_range, self.variant)
        return False, moved, slabs

    def live(self):
        return np.flatnonzero(in_box(self.xyz, self.cube, self.variant))


# A scripted drive for a 40 m cube with DET_RANGE 5 m (threshold 7.5 m, mov_dist 11.25 m): each entry is an offset from the
# centre of the cube the window holds before the step (from `origin` on the first step).  +-15 lies 5 m inside a face (the cube
# moves), +-25 lies 5 m past a face (it moves too: the reference tests the distance, not the side), 200 lies past the cube and
# away from every face (nothing moves), 0 keeps the cube.
DRIVE = [(0, 0, 0), (0, 0, 0), (-15, 0, 0), (15, 0, 0), (0, -15, 0), (0, 15, 0), (0, 0, 15), (0, 0, -15), (15, 15, 0),
         (-15, 15, 0), (-15, -15, -15), (14, -14, 14), (0, 0, 0), (200, 0, 0), (25, 0, 0), (0, -25, 0), (0, 0, 0)]


def drive_pos(w, off, origin=(0.0, 0.0, 0.0)):
    """The position of a DRIVE step for window w (before its step)."""
    c = np.asarray(origin, np.float64) if w.cube is None else (w.cube[:3].astype(np.float64) + w.cube[3:]) / 2
    return c + np.asarray(off, np.float64)
