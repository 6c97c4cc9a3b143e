"""The seed and the changes restated (tests/world_seed_ref.py), without a GPU: the seed is one accumulate of the seed cloud,
chunking does not change it, the kept / removed / added partition holds, and each planted mistake changes what the GPU tests
compare.  Also the two-session street scene behind plugin.SEED_HITS and the default street's parked boxes."""
import numpy as np
import pytest

import world_ref as W
import world_seed_ref as SR
import world_voxel_ref as V
from malio_b200 import plugin, synth

F = np.float32
LEAF = 0.5
KEEP = (plugin.KEEP_MIN_MISS, plugin.KEEP_MAX_MISS_PER_HIT)


def _cloud(n=4000, seed=0):
    """Runs of points in one voxel (so chunk boundaries fall inside them), scattered points, non-finite rows."""
    rng = np.random.default_rng(seed)
    centre = rng.uniform(-20, 20, (n // 10, 3)).astype(F)
    xyz = np.repeat(centre, 10, axis=0) + rng.uniform(-0.2, 0.2, (n // 10 * 10, 3)).astype(F)
    xyz = np.concatenate([xyz, rng.uniform(-20, 20, (n // 4, 3)).astype(F)])
    c = np.concatenate([xyz, rng.uniform(0, 100, (xyz.shape[0], 1)).astype(F)], axis=1).astype(F)
    c[5, 0], c[17, 2], c[-3, 1] = np.nan, np.inf, -np.inf
    return c


def _same(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape and a.tobytes() == b.tobytes(), what


def test_seed_is_one_accumulate_of_the_seed_cloud():
    c = _cloud()
    ref = SR.SeedMapRef()
    n = ref.seed(c, LEAF, 3)
    acc = V.VoxelMapRef()
    assert n == acc.accumulate(c, LEAF)                       # the point-by-point loop of the contract
    _same(ref.centroids(), acc.centroids(), "centroids")
    _same(ref.keys(), acc.keys(), "keys")
    ev = ref.evidence()
    assert np.all(ev[:, 0] == 3) and np.all(ev[:, 1] == 0) and len(ref.seeded) == n


@pytest.mark.parametrize("chunk", [1, 7, 10, 333, 1234])
def test_chunks_equal_one_shot(chunk):
    c = _cloud()
    one, parts = SR.SeedMapRef(), SR.SeedMapRef()
    one.seed(c, LEAF, 1)
    parts.seed(c, LEAF, 1, chunk=chunk)
    # the runs of 10 points in one voxel straddle chunk boundaries for every chunk size but 10
    if chunk not in (1, 10):
        ijk = V.voxel_index(c[:, :3], LEAF)[0]
        assert any((ijk[a - 1] == ijk[a]).all() for a in range(chunk, c.shape[0], chunk))
    _same(parts.centroids(), one.centroids(), chunk)
    _same(parts.evidence(), one.evidence(), chunk)


def test_refusals():
    ref = SR.SeedMapRef()
    ref.seed(_cloud(100), LEAF, 1)
    with pytest.raises(SR.StateError):
        ref.seed(_cloud(100), LEAF, 1)
    far = _cloud(100)
    far[50, :3] = 3.0e9
    with pytest.raises(V.CapacityError):
        SR.SeedMapRef().seed(far, 0.5, 1, chunk=10)


def _session(street, ref, seed, n=20, plain=True):
    """A carved session of n scans on the truth states (plain: every 7th scan folded with the plain accumulate); returns the
    labels (street_cast's) of the voxels the scans hit."""
    labels = {}
    for k in range(n):
        s = synth.street_scan(street, k, seed=seed)
        cloud = W.register_world(s["state"], None, s["body"][0], 0, 0.0)
        org = W.register_world(s["state"], None, np.zeros((1, 3), F), 0, 0.0)[:, :3]
        if plain and k % 7 == 3:
            ref.accumulate(cloud, LEAF)
        else:
            ref.accumulate_carve(cloud, [cloud.shape[0]], org, LEAF, plugin.CARVE_MAX_RANGE, plugin.CARVE_END_MARGIN)
        for key, wh in zip(map(tuple, V.voxel_index(cloud[:, :3], LEAF)[0].tolist()), s["what"][0]):
            labels.setdefault(key, set()).add(int(wh))
    return labels


GONE = 2                                            # the parked box at x = 6 .. 10 leaves
NEW = ((12.0, -6.4, 0.0), (16.0, -4.6, 1.4))        # a box appears on the other side


def _two_sessions(variant="", seed_hits=plugin.SEED_HITS, n=20, plain=True):
    r1 = SR.SeedMapRef()
    _session(synth.Street(), r1, 0, n, plain)
    kept = r1.centroids()[r1.kept_mask(*KEEP)]
    r2 = SR.SeedMapRef(variant)
    r2.seed(kept, LEAF, seed_hits)
    lab = _session(synth.Street(gone=(GONE,), extra=(NEW,)), r2, 1, n, plain)
    return r1, r2, lab


def test_partition_holds_after_a_carved_session():
    _, r2, _ = _two_sessions(n=8)
    seeded, kept, removed, added = r2.change_masks(*KEEP)
    assert removed.any() and added.any()
    assert not (removed & added).any()
    _same(kept, (seeded & ~removed) | added, "kept = (seeded - removed) + added")


def test_planted_mistakes_change_the_outputs():
    c = _cloud(3000, seed=4)
    good = SR.SeedMapRef()
    good.seed(c, LEAF, 2, chunk=100)
    bad = SR.SeedMapRef("reversed_chunks")
    bad.seed(c, LEAF, 2, chunk=100)
    assert good.centroids().tobytes() != bad.centroids().tobytes()
    _, ref, _ = _two_sessions(n=8)
    rem, add = ref.changes(*KEEP)
    ev = ref.evidence()
    for variant in ("carve_zeroes", "added_all", "removed_before_seed"):
        _, r, _ = _two_sessions(variant, n=8)
        r_rem, r_add = r.changes(*KEEP)
        differs = (r.evidence().tobytes() != ev.tobytes(), r_rem.tobytes() != rem.tobytes(), r_add.tobytes() != add.tobytes())
        assert any(differs), variant


def test_street_scene_behind_the_seed_hits_default():
    """Two sessions of 20 scans at 0.5 m with the library's carve and keep defaults; session 2 seeds from session 1's kept map
    and drives the same street with parked box GONE gone and the box NEW added.  At SEED_HITS (2): of the 34 gone-box voxels
    above the ground layer 23 (68 %) are removed (the others face the façade 1.6 m behind the box: the rays that pass them end
    within the 4 m margin); 48 of the 57 new-box voxels are added; 108 of 13 544 static voxels (0.8 %) are removed.  With 0
    seeded hits 3.1 % of the static voxels go, with 3 the gone box keeps 38 % of its voxels."""
    r1, r2, lab = _two_sessions(plain=False)
    lo, hi = synth.Street().parked()[GONE]
    keys = sorted(r2.sums)
    seeded, _, removed, added = r2.change_masks(*KEEP)
    c = r2.centroids()
    gone = seeded & np.all((c[:, :3] >= lo) & (c[:, :3] < hi), axis=1) & (c[:, 2] >= LEAF)
    new = np.array([lab.get(k) == {2} for k in keys]) & np.all((c[:, :3] >= np.array(NEW[0]) - 0.1) &
                                                              (c[:, :3] < np.array(NEW[1]) + 0.1), axis=1)
    lab1 = {}
    for k in range(20):
        s = synth.street_scan(synth.Street(), k, seed=0)
        cloud = W.register_world(s["state"], None, s["body"][0], 0, 0.0)
        for key, wh in zip(map(tuple, V.voxel_index(cloud[:, :3], LEAF)[0].tolist()), s["what"][0]):
            lab1.setdefault(key, set()).add(int(wh))
    static = seeded & np.array([k in lab1 and lab1[k] <= {0, 1} for k in keys])
    assert gone.sum() >= 30 and removed[gone].mean() >= 0.6, (gone.sum(), removed[gone].mean())
    assert new.sum() >= 50 and added[new].mean() >= 0.8, (new.sum(), added[new].mean())
    assert static.sum() > 13000 and removed[static].mean() <= 0.01, removed[static].mean()


def test_street_defaults_are_unchanged_and_the_new_fields_apply():
    st = synth.Street()
    boxes = st.parked()
    assert len(boxes) == 7
    for (lo, hi), x in zip(boxes, np.arange(-12.0, 48.0, 9.0)):
        assert lo.tolist() == [x, 4.6, 0.0] and hi.tolist() == [x + 4.0, 6.4, 1.4]
    two = synth.Street(gone=(GONE,), extra=(NEW,)).parked()
    assert len(two) == 7 and all(np.array_equal(a[0], b[0]) for a, b in zip(two[:6], boxes[:GONE] + boxes[GONE + 1:]))
    assert two[-1][0].tolist() == list(NEW[0])
    a = synth.street_scan(synth.Street(), 5)
    b = synth.street_scan(synth.Street(gone=(), extra=()), 5)
    assert a["body"][0].tobytes() == b["body"][0].tobytes()


def test_python_surface():
    assert plugin.SEED_HITS == 2
    for name in ("voxel_map_seed", "voxel_map_seed_tensor", "voxel_map_changes", "voxel_map_save_changes"):
        assert callable(getattr(plugin.MeasurementModel, name))
