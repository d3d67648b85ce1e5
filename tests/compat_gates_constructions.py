"""Frame scripts that put (candidate, track) pairs on the boundaries of the tracker's compatibility gate
(SortAttributes::compatible: epoch delta <= max_idle_epochs, then SpatioTemporalConstraints::validate(delta,
dist_in_2r)), shared by tests/test_gpu_compat_gates.py and tests/test_compat_gates_cpu.py.

A track fed the same box every frame predicts that box bit for bit (zero velocity, zero innovation), so its centre and
radius are known exactly.  Every track j gets a last epoch (its idle delta at the probe frame) and one probe candidate:
  tie     dist_in_2r == the applicable max_dist exactly (found by bisection over f32 offsets)    compatible
  above   the next f32 offset past the tie (dist_in_2r > max_dist)                                 cut
  inside  half the max_dist                                                                        compatible
  outside one and a half times the max_dist                                                        cut
  dup     the tie of the duplicate epoch's second, dropped entry                                   cut
  free    delta past every constraint epoch: any distance                                          compatible
  nan_cand / nan_track: the candidate's / the track's centre is NaN: cut under a constraint, else compatible
Delta > max_idle_epochs is cut whatever the distance.  Visual scripts give candidate j the feature of track j, every
other pair far apart in feature space, and offsets whose IoU stays below the tracker's threshold, so the visual stage
alone decides the pair; positional scripts use max_dists small enough that the positional metric accepts every
compatible probe.  The expected outcome of candidate j is then: it continues track j exactly when the pair is
compatible."""
import numpy as np

F32 = np.float32
EPS = F32(0.00001)
NAN = float("nan")

# (epoch, max_dist) lists: unsorted, one duplicate epoch (the first entry of an epoch wins), max_idle_epochs = 6
VISUAL_CONSTRAINTS = [(3, 0.9), (1, 0.25), (3, 2.0), (5, 1.5), (2, 0.5)]
IOU_CONSTRAINTS = [(3, 0.3), (1, 0.1), (3, 0.45), (5, 0.35), (2, 0.2)]
MAHA_CONSTRAINTS = [(3, 0.06), (1, 0.02), (3, 0.2), (5, 0.07), (2, 0.04)]
MAX_IDLE = 6
FRAMES = 8          # frames before the probe; a scene may skip epochs between the last of them and the probe


def constraints_for(kind, pos):
    return VISUAL_CONSTRAINTS if kind >= 2 else (IOU_CONSTRAINTS if pos == 1 else MAHA_CONSTRAINTS)


def sorted_unique(cons):
    out = []
    for e, m in sorted(cons, key=lambda c: c[0]):
        if not out or out[-1][0] != e:
            out.append((e, m))
    return out


def applicable(cons, delta):
    """max_dist of the constraint validate() applies to delta (None: no constraint applies)."""
    for e, m in sorted_unique(cons):
        if e >= delta:
            return m
    return None


# ------------------------------------------------------------------------------------------------ f32 replica
def radius(aspect, height):
    """Universal2DBox::get_radius in f32 (sb_math.cuh box_radius)."""
    aspect, height = np.asarray(aspect, F32), np.asarray(height, F32)
    hw = aspect * height / F32(2.0)
    hh = height / F32(2.0)
    return np.sqrt(hw * hw + hh * hh)


def dist_in_2r(xl, yl, rl, xr, yr, rr):
    """Universal2DBox::dist_in_2r in f32 (sb_math.cuh dist_in_2r)."""
    xl, yl, rl, xr, yr, rr = (np.asarray(v, F32) for v in (xl, yl, rl, xr, yr, rr))
    rd = rl + rr
    x = xl - xr
    y = yl - yr
    with np.errstate(invalid="ignore"):
        return np.sqrt(x * x + y * y) / np.sqrt(rd * rd + EPS)


def _bits(x):
    return np.asarray(x, F32).view(np.uint32).astype(np.int64)


def _f32_of(b):
    return np.asarray(b).astype(np.uint32).view(F32)


def _bisect(d, lo, hi, target):
    """Over the f32 bit patterns (positive floats: ordered like their values) of a monotone d: with d(lo) on one side
    of the target and d(hi) on the other, returns (lo, hi) adjacent, d(hi) on hi's side (<= target when d increases
    from hi to lo, else d(lo) <= target)."""
    while np.any(hi - lo > 1):
        mid = (lo + hi) // 2
        up = d(mid) > target
        lo, hi = np.where(up == (d(lo) > target), mid, lo), np.where(up == (d(lo) > target), hi, mid)
    return lo, hi


def tie_offsets(tx, ty, aspect, height, target, exact, rng, tries=64):
    """Candidate centres (cx, cy), cx = tx + a small perturbation and cy >= ty, and box heights: the candidate and its
    track share aspect and height.  Each pair's cy is the largest f32 with dist_in_2r <= target.  Where `exact`, the
    height is then moved, by bisection over its f32 values (dist_in_2r falls as the radius grows), to the smallest one
    with dist_in_2r <= target, and a pair whose distance there is not the target exactly draws a new perturbation."""
    tx, ty, a, h0, target = (np.asarray(v, F32).copy() for v in (tx, ty, aspect, height, target))
    n = len(tx)
    cx, cy, h = np.zeros(n, F32), np.zeros(n, F32), h0.copy()
    todo = np.arange(n)
    for _ in range(tries):
        if len(todo) == 0:
            return cx, cy, h
        t = todo
        px = (tx[t] + F32(rng.uniform(-0.5, 0.5, len(t)))).astype(F32)
        r = radius(a[t], h0[t])
        d_y = lambda b: dist_in_2r(px, _f32_of(b), r, tx[t], ty[t], r)  # noqa: E731
        lo, hi = _bits(ty[t]), _bits(ty[t] + F32(4.0) * target[t] * F32(2.0) * r)
        assert np.all(d_y(hi) > target[t]) and np.all(d_y(lo) <= target[t])
        lo, _ = _bisect(d_y, lo, hi, target[t])
        py = _f32_of(lo)
        cx[t], cy[t] = px, py
        ex = exact[t]
        if not np.any(ex):
            return cx, cy, h
        te = t[ex]
        d_h = lambda b: dist_in_2r(px[ex], py[ex], radius(a[te], _f32_of(b)), tx[te], ty[te],  # noqa: E731
                                   radius(a[te], _f32_of(b)))
        hlo, hhi = _bits(h0[te] * F32(0.98)), _bits(h0[te])
        assert np.all(d_h(hlo) > target[te]) and np.all(d_h(hhi) <= target[te])
        _, hhi = _bisect(d_h, hlo, hhi, target[te])
        hit = d_h(hhi) == target[te]
        h[te[hit]] = _f32_of(hhi[hit])
        todo = te[~hit]
    raise AssertionError(f"{len(todo)} ties not found")


def next_up(x):
    return np.nextafter(np.asarray(x, F32), F32(np.inf))


# ------------------------------------------------------------------------------------------------ scripts
class Script:
    """One tracker's frames: `steps` is a list of ("frame", request) and ("skip", scene_id, n); the last frame is the
    probe.  Per track (index into `tracks`): its scene, the frame of its first and last detection, its case and whether
    its probe candidate is compatible.  `probe_cand[j]` is the row of track j's candidate in the probe request."""

    def __init__(self, kind, pos, K, d, scenes, seed, vis=0, fillers=None):
        """scenes: list of (scene_id, skip, [(delta, case), ...]) -- one track per entry, in store order.  fillers:
        {scene_id: {frame: count}} -- detections that each start a track of their own in that frame, far from every
        probe (their row in `tracks` is -1), so that a scene holds more tracks at the probe than the culled scan takes."""
        self.kind, self.pos, self.K, self.d, self.vis = kind, pos, K, d, vis
        rng = np.random.default_rng(seed)
        cons = constraints_for(kind, pos)
        self.constraints = cons
        visual = kind >= 2
        rows = []
        for sid, skip, cases in scenes:
            for delta, case in cases:
                rows.append((sid, skip, delta, case))
        n = len(rows)
        self.scene = np.array([r[0] for r in rows], np.uint64)
        skip = np.array([r[1] for r in rows])
        self.delta = np.array([r[2] for r in rows])
        self.case = [r[3] for r in rows]
        # probe epoch of a scene = FRAMES + skip + 1; the track's last detection is at epoch probe - delta
        self.last = FRAMES + skip + 1 - self.delta
        assert np.all((self.last >= 1) & (self.last <= FRAMES)), "a delta the scene's schedule cannot reach"
        self.first = np.where([c == "nan_track" for c in self.case], self.last, 1)
        # boxes: a grid 400 apart, heights 40..80, aspects 0.4..0.6 (IoU of the probes below the trackers' thresholds)
        side = int(np.ceil(np.sqrt(n)))
        idx = np.arange(n)
        h = F32(rng.uniform(40, 80, n))
        a = F32(rng.uniform(0.4, 0.6, n))
        tx = F32(1000.0 + 400.0 * (idx % side) + rng.uniform(-5, 5, n))
        ty = F32(1000.0 + 400.0 * (idx // side) + rng.uniform(-5, 5, n))
        self.boxes = np.stack([tx, ty, np.full(n, NAN, F32), a, h, np.full(n, F32(0.9))], 1).astype(F32)
        for j, c in enumerate(self.case):
            if c == "nan_track":
                self.boxes[j, 0] = NAN
        r = radius(a, h)
        # probe offsets
        far = 1.1 * max(m for _, m in cons) if visual else (0.38 if pos == 1 else 0.075)
        target, compat = np.zeros(n, F32), np.zeros(n, bool)
        for j, (dl, c) in enumerate(zip(self.delta, self.case)):
            m = applicable(cons, dl)
            if dl > MAX_IDLE:
                target[j], compat[j] = F32(0.5 * (m or min(mm for _, mm in cons))), False
            elif c in ("nan_cand", "nan_track"):
                target[j], compat[j] = F32(0.5 * (m or far)), m is None
            elif m is None:
                assert c == "free", (dl, c)
                target[j], compat[j] = F32(far), True
            elif c == "tie" or c == "above":
                target[j], compat[j] = F32(m), c == "tie"
            elif c == "inside":
                target[j], compat[j] = F32(0.5 * m), True
            elif c == "outside":
                target[j], compat[j] = F32(1.5 * m), False
            elif c == "dup":
                dropped = [mm for e, mm in cons if e == dl][1:]
                assert dropped and dropped[0] > m
                target[j], compat[j] = F32(dropped[0]), False
            else:
                raise ValueError(c)
        self.target, self.compat = target, compat
        # the probe continues its track when the pair is compatible -- except a NaN candidate: its Kalman prediction is
        # NaN in every component (0 * NaN in the update), so its box area is NaN and its feature is never used
        self.expect = compat & np.array([c != "nan_cand" for c in self.case])
        exact = np.array([c in ("tie", "above", "dup") and dl <= MAX_IDLE for dl, c in zip(self.delta, self.case)])
        cx, cy, h = tie_offsets(tx, ty, a, h, target, exact, rng)
        self.boxes[:, 4] = h
        r = radius(a, h)
        above = np.array([c == "above" for c in self.case])
        cy[above] = next_up(cy[above])
        cand = self.boxes.copy()
        cand[:, 0], cand[:, 1] = cx, cy
        for j, c in enumerate(self.case):
            if c == "nan_cand":
                cand[j, 0] = NAN
            if c == "nan_track":
                cand[j, 0] = tx[j]
        self.cand = cand
        # the exact distances the gate sees (NaN centres give NaN)
        self.dist = dist_in_2r(cand[:, 0], cand[:, 1], r, self.boxes[:, 0], self.boxes[:, 1], r)
        if visual:
            f = rng.standard_normal((n, d)).astype(F32)
            self.feats = (f / np.linalg.norm(f, axis=1, keepdims=True)).astype(F32)
        else:
            self.feats = None
        # frames
        sids = list(dict.fromkeys(int(s) for s in self.scene))
        skips = {int(sid): int(sk) for sid, sk, _ in scenes}
        self.steps = []
        perm = rng.permutation(n)   # candidate rows in an order unrelated to the store order
        fillers = fillers or {}
        assert not (visual and fillers)
        n_fill = 0
        for fr in range(1, FRAMES + 2):
            probe = fr == FRAMES + 1
            if probe:
                for sid in sids:
                    if skips[sid]:
                        self.steps.append(("skip", sid, skips[sid]))
            rows_by_scene, fill_boxes = [], []
            for sid in sids:
                if probe:
                    sel = [j for j in perm if int(self.scene[j]) == sid]
                else:
                    sel = [j for j in range(n) if int(self.scene[j]) == sid and self.first[j] <= fr <= self.last[j]]
                k = fillers.get(sid, {}).get(fr, 0)
                # 150 apart (boxes of height 20) on a grid from x = 20000, far from the probes and from each other
                g = np.arange(n_fill, n_fill + k)
                n_fill += k
                fill_boxes.append(np.stack([20000.0 + 150.0 * (g % 64), 1000.0 + 150.0 * (g // 64), np.full(k, NAN),
                                            np.full(k, 0.5), np.full(k, 20.0), np.full(k, 0.9)], 1).astype(F32))
                rows_by_scene.append(sel + [-1] * k)
            order = [j for sel in rows_by_scene for j in sel]
            offs = np.concatenate([[0], np.cumsum([len(s) for s in rows_by_scene])]).astype(np.int32)
            src = self.cand if probe else self.boxes
            b = np.concatenate([np.concatenate([src[[j for j in sel if j >= 0]], fb]) for sel, fb in
                                zip(rows_by_scene, fill_boxes)]) if order else np.zeros((0, 6), F32)
            req = {"scene_ids": np.array(sids, np.uint64), "det_offsets": offs, "boxes": np.ascontiguousarray(b, F32),
                   "features": np.ascontiguousarray(self.feats[order]) if visual else None, "tracks": order}
            self.steps.append(("frame", req))

    def options(self, vis_threshold=None, **kw):
        visual = self.kind >= 2
        o = dict(kind=self.kind, positional_kind=self.pos, iou_threshold=0.8 if visual else 0.3,
                 max_idle_epochs=MAX_IDLE, constraints=self.constraints, min_confidence=0.05)
        if visual:
            thr = vis_threshold if vis_threshold is not None else (0.5 if self.vis == 0 else 0.8)
            o.update(visual_kind=self.vis, visual_threshold=thr, feature_dim=self.d, visual_max_observations=self.K,
                     visual_min_votes=1, visual_minimal_track_length=1, visual_minimal_area=0.0)
        o.update(kw)
        return o


def run(tracker, script, check=None):
    """Runs the script; returns (outputs per frame, the track id of every track, the probe outcome per track:
    True when the probe candidate continued its own track).  check(fr, out) is called after every frame."""
    track_id = np.zeros(len(script.delta), np.uint64)
    outs = []
    fr = 0
    for st in script.steps:
        if st[0] == "skip":
            tracker.skip_epochs(st[2], st[1])
            continue
        req = st[1]
        out = tracker.predict_batch(req["scene_ids"], req["det_offsets"], req["boxes"], features=req["features"])
        outs.append(out)
        if check:
            check(fr, out)
        fr += 1
        for row, j in enumerate(req["tracks"]):
            if j >= 0 and fr < FRAMES + 1 and fr == script.first[j]:   # the track's first detection creates it
                track_id[j] = out["ids"][row]
    probe = outs[-1]
    got = np.zeros(len(script.delta), bool)
    for row, j in enumerate(script.steps[-1][1]["tracks"]):
        got[j] = probe["ids"][row] == track_id[j]
    return outs, track_id, got


def cases_mix(rng, n, lo, cases=("tie", "above", "inside", "outside")):
    """n (delta, case) pairs in random order (so the outcome varies with the row and the column): deltas lo..
    MAX_IDLE + 1, each constrained delta with every case.  The three constraint lists share their epochs."""
    deltas = list(range(lo, MAX_IDLE + 2))
    pairs = []
    for dl in deltas:
        if applicable(VISUAL_CONSTRAINTS, dl) is None:
            pairs.append((dl, "free" if dl <= MAX_IDLE else "tie"))
        else:
            pairs += [(dl, c) for c in cases]
    out = [pairs[k % len(pairs)] for k in range(n)]
    rng.shuffle(out)
    return out


NAN_CASES = [(2, "nan_cand"), (MAX_IDLE, "nan_cand"), (2, "nan_track"), (MAX_IDLE, "nan_track")]


# Filler tracks per frame that take one scene past 4096 tracks at the probe, so that the positional cost of the probe
# frame runs in the dense tiled kernel.  A frame is limited by the shared memory of the assignment solver, which holds
# the scene's candidates and tracks (about 44 bytes per track and 38 per candidate at this size), so the fillers come
# in early and large, and the probe frame has few candidates.  They start at frame FRAMES - 4, so every filler is still
# under a constraint (delta <= 5) at the probe, and none is compatible with a probe.
BIG_FILLERS = {4: 2636, 5: 941, 6: 336, 7: 120, 8: 43}
BIG_PROBES = 24


def positional_script(kind, pos, seed, n=120, big=False):
    """Sort: one scene.  BatchSort: three scenes whose epochs differ (0, 2 and 1 skipped epochs before the probe).
    big: the first scene has BIG_PROBES probes and more than 4096 tracks at the probe (the others stay small)."""
    rng = np.random.default_rng(seed)
    n = BIG_PROBES if big else n
    if kind == 0:
        scenes = [(0, 0, cases_mix(rng, n, 1))]
    else:
        scenes = [(5, 0, cases_mix(rng, n if big else n // 2, 1)), (9, 2, cases_mix(rng, 12 if big else 40, 3)),
                  (2, 1, cases_mix(rng, 10 if big else 30, 2))]
    fillers = {scenes[0][0]: BIG_FILLERS} if big else None
    return Script(kind, pos, 1, 0, scenes, seed, fillers=fillers)


def visual_script(kind, vis, K, seed, n=300, d=64, nan=False):
    """The first scene has n candidates and n * K feature columns (both past 256) and the duplicate epoch's dropped
    entry (and with `nan` the NaN centres); BatchVisualSort adds two scenes at other epochs."""
    rng = np.random.default_rng(seed)
    first = cases_mix(rng, n - 8, 1) + [(3, "dup"), (3, "dup")] + (NAN_CASES if nan else [])
    rng.shuffle(first)
    scenes = [(0 if kind == 2 else 3, 0, first)]
    if kind == 3:
        scenes += [(11, 2, cases_mix(rng, 40, 3) + [(3, "dup")]), (4, 1, cases_mix(rng, 24, 2))]
    return Script(kind, 1, K, d, scenes, seed, vis=vis)
