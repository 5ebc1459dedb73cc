"""Seeded synthetic inputs for the projection-guided matchers and the DBoW2 transform (SURVEY.md §8(f) ranks 2-3).

A *grid* is the image side of a matcher (Frame or KeyFrame: undistorted keypoints, octaves, angles, descriptors and the
64-ish x 48 lookup grid geometry); *queries* are map points after the caller's projection prelude (valid flag, projected
pixel, search radius, predicted level, descriptor).  Plain dicts of numpy arrays: the product binding
(ccm_slam_b200.frontend) and the test-side checker each build their own C structs from them.
"""
from __future__ import annotations

import numpy as np

SCALE_FACTORS = (np.float32(1.2) ** np.arange(8)).astype(np.float32)          # ORBextractor scale table
LEVEL_SIGMA2 = (SCALE_FACTORS * SCALE_FACTORS).astype(np.float32)
INV_LEVEL_SIGMA2 = (np.float32(1.0) / LEVEL_SIGMA2).astype(np.float32)
_QUOTA = np.array([217, 181, 151, 126, 105, 87, 73, 60], np.float64)


def flip_bits(desc, nbits, rng):
    """copies of `desc` (n x 32 u8) with `nbits[i]` random bits flipped in row i"""
    out = desc.copy()
    for i in range(out.shape[0]):
        if nbits[i] <= 0:
            continue
        pos = rng.choice(256, size=int(nbits[i]), replace=False)
        np.bitwise_xor.at(out[i], pos // 8, (1 << (pos % 8)).astype(np.uint8))
    return out


def make_grid(n=1000, seed=0, bounds=(-10.5, -8.25, 761.0, 489.5), cols=75, rows=48, clustered=True):
    """Features of one image.  A few keypoints lie outside the bounds (undistortion can do that; PosInGrid drops them)."""
    rng = np.random.default_rng(seed)
    x0, y0, x1, y1 = bounds
    if clustered:  # textured regions: many features per window so that best/second-best and ties matter
        centres = rng.uniform([x0 + 30, y0 + 30], [x1 - 30, y1 - 30], size=(max(4, n // 25), 2))
        xy = centres[rng.integers(0, len(centres), n)] + rng.normal(0, 9.0, size=(n, 2))
    else:
        xy = rng.uniform([x0, y0], [x1, y1], size=(n, 2))
    n_out = max(1, n // 50)
    xy[:n_out] = rng.uniform([x0 - 20, y0 - 20], [x0 - 1, y0 - 1], size=(n_out, 2))   # out of the grid
    xy[n_out:2 * n_out, 0] = x1 + rng.uniform(0.0, 3.0, n_out)                        # right at / past the right edge
    xy = np.round(xy * 4) / 4                                                          # quarter-pixel positions: exact ties in |dx| < r
    octave = rng.choice(8, size=n, p=_QUOTA / _QUOTA.sum()).astype(np.int32)
    angle = rng.uniform(0, 360, n).astype(np.float32)
    desc = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    # near-duplicate descriptors inside clusters (repetitive texture): forces the ratio test and first-wins ties
    for i in range(0, n - 1, 7):
        desc[i + 1] = flip_bits(desc[i:i + 1], [rng.integers(0, 3)], rng)[0]
    return dict(desc=desc, kp_xy=xy.astype(np.float32), octave=octave, angle=angle, bounds=bounds, cols=cols, rows=rows)


def make_queries(grid, m=1500, seed=1, th=3.0, noise_px=2.0, invalid_frac=0.1, max_flip=70, dup_frac=0.15):
    """Map points projected into `grid`'s image.  Most are noisy copies of a feature (true matches); some are duplicates of
    an earlier query (two points competing for one feature); some are random (no match); some are invalid."""
    rng = np.random.default_rng(seed)
    n = grid["desc"].shape[0]
    src = rng.integers(0, n, m)
    dup = rng.random(m) < dup_frac
    for i in range(1, m):
        if dup[i]:
            src[i] = src[rng.integers(0, i)]
    uv = grid["kp_xy"][src] + rng.normal(0, noise_px, size=(m, 2)).astype(np.float32)
    uv = (np.round(uv * 4) / 4).astype(np.float32)
    level = np.clip(grid["octave"][src] + rng.choice([0, 0, 0, 1, 1, -1, 2], size=m), 0, 7).astype(np.int32)
    nflip = rng.integers(0, max_flip, m)
    desc = flip_bits(grid["desc"][src], nflip, rng)
    rnd = rng.random(m) < 0.1
    desc[rnd] = rng.integers(0, 256, size=(int(rnd.sum()), 32), dtype=np.uint8)
    radius = (np.float32(th) * SCALE_FACTORS[level]).astype(np.float32)
    valid = (rng.random(m) >= invalid_frac).astype(np.uint8)
    angle = ((grid["angle"][src] + rng.normal(0, 4.0, m) + np.where(rng.random(m) < 0.1, rng.uniform(0, 360, m), 0.0)) % 360).astype(np.float32)
    return dict(valid=valid, uv=uv, radius=radius, level=level, desc=desc, angle=angle, src=src)


def tie_storm(grid, queries=None, pool=6, seed=0):
    """Replace every descriptor by one of `pool` patterns that lie 8..30 bits from a common base (copies of the inputs are returned).
    Every window then holds many candidates at exactly the same distance, below the acceptance thresholds: what is selected is decided
    by the visiting order alone (first minimum, second best on the same level, who keeps a contested feature)."""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, size=(1, 32), dtype=np.uint8)
    pats = np.concatenate([flip_bits(base, [int(rng.integers(8, 31))], rng) for _ in range(pool)])
    g = dict(grid); g["desc"] = pats[rng.integers(0, pool, grid["desc"].shape[0])]
    if queries is None:
        return g
    q = dict(queries); q["desc"] = pats[rng.integers(0, pool, queries["desc"].shape[0])]
    return g, q


def make_vocabulary(k=10, L=3, seed=0, scoring=0, weighting=0, early_leaf_frac=0.05, tie_frac=0.05, stop_frac=0.02):
    """A DBoW2-style vocabulary tree as the rows of its text file (row 0 = root): parent, leaf flag, descriptor, weight.
    Hierarchical: children are perturbed copies of their parent, so descents are decisive at the top and close at the
    bottom; some siblings are exact duplicates (first-minimum-wins ties); some inner nodes stop early (ragged depth);
    a few words have weight 0 (stopped words)."""
    rng = np.random.default_rng(seed)
    parent, is_leaf, desc, weight = [0], [0], [np.zeros(32, np.uint8)], [0.0]

    def grow(pid, pdesc, level):
        flips = max(6, 110 >> (level - 1))
        prev = None
        for c in range(k):
            nid = len(parent)
            d = flip_bits(pdesc[None, :], [flips], rng)[0] if level > 1 else rng.integers(0, 256, 32, dtype=np.uint8)
            if prev is not None and rng.random() < tie_frac:
                d = prev.copy()
            prev = d
            leaf = level == L or (level > 1 and rng.random() < early_leaf_frac)
            parent.append(pid); is_leaf.append(1 if leaf else 0); desc.append(d)
            weight.append(0.0 if (not leaf or rng.random() < stop_frac) else float(rng.uniform(0.5, 12.0)))
            if not leaf:
                grow(nid, d, level + 1)

    grow(0, desc[0], 1)
    return dict(k=k, L=L, scoring=scoring, weighting=weighting, parent=np.array(parent, np.int32), is_leaf=np.array(is_leaf, np.uint8),
                desc=np.stack(desc).astype(np.uint8), weight=np.array(weight, np.float64))


def make_voc_features(voc, n=1000, seed=0):
    """descriptors near random leaves of `voc` (plus some uniformly random ones)"""
    rng = np.random.default_rng(seed)
    leaves = np.flatnonzero(voc["is_leaf"])
    pick = leaves[rng.integers(0, len(leaves), n)]
    d = flip_bits(voc["desc"][pick], rng.integers(0, 40, n), rng)
    rnd = rng.random(n) < 0.1
    d[rnd] = rng.integers(0, 256, size=(int(rnd.sum()), 32), dtype=np.uint8)
    return d


def make_init_pair(n=1000, seed=0, window=100.0, shift=(6.0, -4.0)):
    """Two frames for SearchForInitialization: F2 holds shifted, slightly perturbed copies of most of F1's keypoints.  Returns
    (grid of F2, queries = one per keypoint of F1 with level = its octave, uv = its own position (vbPrevMatched at the first call),
    radius = windowSize)."""
    rng = np.random.default_rng(seed)
    g1 = make_grid(n=n, seed=seed + 100)
    g1["octave"][: n // 2] = 0                      # the matcher only looks at octave 0
    g2 = make_grid(n=n, seed=seed + 200)
    keep = rng.permutation(n)[: (3 * n) // 4]
    g2["kp_xy"][keep] = g1["kp_xy"][keep] + np.float32(shift) + rng.normal(0, 0.75, (len(keep), 2)).astype(np.float32)
    g2["octave"][keep] = g1["octave"][keep]
    g2["angle"][keep] = (g1["angle"][keep] + rng.normal(0, 3.0, len(keep))).astype(np.float32) % np.float32(360)
    g2["desc"][keep] = flip_bits(g1["desc"][keep], rng.integers(0, 45, len(keep)), rng)
    q = dict(valid=np.ones(n, np.uint8), uv=g1["kp_xy"].copy(), radius=np.full(n, window, np.float32), level=g1["octave"].copy(),
             desc=g1["desc"], angle=g1["angle"])
    return g2, q


def make_place_db(n_clients=4, kf_per_client=60, n_words=20000, local_words=160, bg_words=60, pool=400, revisit=0.3, cross=0.3,
                  n_dups=4, seed=0):
    """A server-shaped keyframe database with BowVectors synthesised directly (no vocabulary tree): `n_clients` agents walk along
    trajectories of places; a keyframe draws `local_words` words from its place's pool (and its neighbour's) and `bg_words` from a
    Zipf background over the whole vocabulary, so that common words have long inverted lists.  A fraction `revisit` of each
    trajectory returns to the agent's earlier places (loop candidates) and a fraction `cross` visits another agent's places
    (map-match candidates).  `n_dups` keyframes copy another keyframe's BowVector exactly: equal scores, ties in the accumulation.
    Covisibility top-10 lists (GetBestCovisibilityKeyFrames(10)) rank the keyframes of the same agent within 8 steps by shared
    words (ties: older first).  Values are L1-normalised.
    Returns dict(n_words, uid, client, place, bow_ptr, bow_word, bow_val, covis_ptr, covis_uid) with uid = mUniqueId (1-based,
    agents interleaved in time as the server receives them)."""
    rng = np.random.default_rng(seed)
    n_places = max(4, kf_per_client // 3)
    pools = [rng.choice(n_words, size=pool, replace=False) for _ in range(n_clients * n_places)]
    zipf = 1.0 / np.arange(1, n_words + 1) ** 1.1
    zipf /= zipf.sum()
    zperm = rng.permutation(n_words)
    place_of = []
    for c in range(n_clients):
        t = np.minimum(np.arange(kf_per_client) // 3, n_places - 1) + c * n_places
        for i in range(kf_per_client):
            u = rng.random()
            if i > 6 and u < revisit:
                t[i] = t[rng.integers(0, i - 5)]
            elif u < revisit + cross:
                t[i] = rng.integers(0, n_clients * n_places)
        place_of.append(t)
    K = n_clients * kf_per_client
    order = np.arange(K).reshape(n_clients, kf_per_client).T.reshape(-1)      # time-interleaved arrival
    uid = np.arange(1, K + 1, dtype=np.uint64)
    client = (order // kf_per_client).astype(np.uint32)
    place = np.array([place_of[c][i] for c, i in zip(order // kf_per_client, order % kf_per_client)], np.int64)
    bows = []
    for k in range(K):
        p = place[k]
        loc = rng.choice(pools[p], size=local_words, replace=False)
        nb = rng.choice(pools[min(p + 1, len(pools) - 1)], size=local_words // 4, replace=False)
        bg = zperm[rng.choice(n_words, size=bg_words, p=zipf)]
        w = np.unique(np.concatenate([loc, nb, bg])).astype(np.uint32)
        v = rng.uniform(0.2, 3.0, len(w))
        bows.append((w, v / np.abs(v).sum()))
    for j in range(n_dups):                                                      # exact copies -> equal scores
        a, b = rng.choice(K, size=2, replace=False)
        bows[b] = (bows[a][0].copy(), bows[a][1].copy())
    covis = []
    sets = [set(w.tolist()) for w, _ in bows]
    for k in range(K):
        same = [j for j in range(max(0, k - 8 * n_clients), min(K, k + 8 * n_clients + 1)) if j != k and client[j] == client[k]]
        same.sort(key=lambda j: (-len(sets[k] & sets[j]), j))
        covis.append(uid[same[:10]])
    bow_ptr = np.concatenate([[0], np.cumsum([len(w) for w, _ in bows])]).astype(np.int64)
    covis_ptr = np.concatenate([[0], np.cumsum([len(c) for c in covis])]).astype(np.int64)
    return dict(n_words=n_words, uid=uid, client=client, place=place, bow_ptr=bow_ptr,
                bow_word=np.concatenate([w for w, _ in bows]).astype(np.uint32), bow_val=np.concatenate([v for _, v in bows]),
                covis_ptr=covis_ptr, covis_uid=np.concatenate(covis).astype(np.uint64) if K else np.zeros(0, np.uint64))


def place_db_bow(db, k):
    """BowVector (word, value) of keyframe row k of make_place_db()"""
    a, b = db["bow_ptr"][k], db["bow_ptr"][k + 1]
    return db["bow_word"][a:b], db["bow_val"][a:b]


def place_db_covis(db, k):
    return db["covis_uid"][db["covis_ptr"][k]:db["covis_ptr"][k + 1]]


# ---- a keyframe and its covisible neighbours for LocalMapping::CreateNewMapPoints ------------------------------------------------
def _rot(rv):
    th = np.linalg.norm(rv)
    if th < 1e-12:
        return np.eye(3)
    k = rv / th
    K = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def new_points_prelude(cur, v):
    """F12 and the epipole of neighbour `v` against `cur`, in f32, the way ComputeF12 (cslam/src/Mapping.cpp:549-566) and
    SearchForTriangulation's head (cslam/src/ORBmatcher.cpp:707-714) form them."""
    f = np.float32
    R1w, t1w = cur["Tcw"][:, :3].astype(f), cur["Tcw"][:, 3].astype(f)
    R2w, t2w = v["Tcw"][:, :3].astype(f), v["Tcw"][:, 3].astype(f)
    R12 = (R1w @ R2w.T).astype(f)
    t12 = (-(R1w @ R2w.T) @ t2w + t1w).astype(f)
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]], f)

    def K(i):
        fx, fy, cx, cy = i
        return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], f)
    F12 = (np.linalg.inv(K(cur["intr"]).T).astype(f) @ tx @ R12 @ np.linalg.inv(K(v["intr"])).astype(f)).astype(f)
    C2 = (R2w @ cur["Ow"].astype(f) + t2w).astype(f)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        invz = f(1.0) / C2[2]
        ex = f(v["intr"][0]) * C2[0] * invz + f(v["intr"][2])
        ey = f(v["intr"][1]) * C2[1] * invz + f(v["intr"][3])
    return F12, f(ex), f(ey)


def make_new_points_scene(n_nb=20, n=1000, seed=0, n_nodes=None, has_mp_frac=0.4, noise_px=0.4, outlier_frac=0.04, outlier_px=5.0,
                          octave_jump_frac=0.05, cross_frac=0.05, forward_every=5, decoy_frac=0.06, twin_frac=0.03, tie_frac=0.03, zero_baseline_nb=None, no_shared_nb=None,
                          all_have_mp=False):
    """A current keyframe and `n_nb` neighbours looking at one seeded point cloud.  Poses have a real baseline; mvKeysUn are projections
    plus pixel noise; octaves follow depth (so the scale gate passes for true matches); descriptors are a per-point base with bits
    flipped per observation; a feature's vocabulary node follows its point.  What forces each outcome to occur:
      zero_baseline_nb   that neighbour sits 1 mm from the current keyframe: every pair fails the parallax gate
      outlier_frac       pixels displaced by outlier_px
      cross_frac         neighbour features moved 3 to 6.5 px off the epipolar line and put on the coarsest level, where the line gate
                         is wide, against a fine-level feature of the current keyframe: the reprojection gates
      forward_every      every such neighbour moves along the optical axis, so the epipole lies in the image and decoys fall on both
                         sides of it: points in front of one camera and behind the other
      octave_jump_frac   neighbour octaves moved by four levels: the scale gate
      decoy_frac         copies of a current feature's descriptor placed along its epipolar line in the neighbour: points behind a
                         camera, low parallax, wrong scale
      has_mp_frac        features already carrying map points, in either view
      twin_frac          a second feature of the current keyframe on the same point: two idx1 sharing one idx2
      tie_frac           a second, identical feature in the neighbour a quarter pixel away: equal distances inside a node
      no_shared_nb       that neighbour's node ids are disjoint from the current keyframe's
      all_have_mp        every feature of the current keyframe carries a map point: nothing to search
    Every neighbour sees most of the cloud, so a feature is matchable in several of them (claims).
    Returns dict(cur=view, neighbours=[view + F12, ex, ey]); a view is what api.new_map_points reads."""
    rng = np.random.default_rng(seed)
    f = np.float32
    intr = (f(458.654), f(457.296), f(367.215), f(248.375))
    W, H = 752.0, 480.0
    P = n
    n_nodes = n_nodes or max(4, n // 10)
    X = np.stack([rng.uniform(-5, 5, P), rng.uniform(-3.2, 3.2, P), rng.uniform(4.0, 12.0, P)], 1)
    base_desc = rng.integers(0, 256, size=(P, 32), dtype=np.uint8)
    base_oct = rng.integers(0, 4, P)
    node_of_point = rng.integers(0, n_nodes, P) * 7 + 3

    def make_view(R, t, disjoint=False):
        Xc = X @ R.T + t
        z = Xc[:, 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            u = intr[0] * Xc[:, 0] / z + intr[2]
            v = intr[1] * Xc[:, 1] / z + intr[3]
        vis = np.flatnonzero((z > 0.5) & (u > 0) & (u < W) & (v > 0) & (v < H) & (rng.random(P) < 0.85))
        vis = rng.permutation(vis)[: n - n // 8]
        m = len(vis)
        xy = np.stack([u[vis], v[vis]], 1) + rng.normal(0, noise_px, (m, 2))
        out = rng.random(m) < outlier_frac
        xy[out] += rng.normal(0, outlier_px, (int(out.sum()), 2))
        d = np.linalg.norm(Xc[vis], axis=1)
        octave = np.clip(np.round(np.log(12.0 / d) / np.log(1.2)).astype(np.int64) + base_oct[vis], 0, 7)
        desc = flip_bits(base_desc[vis], rng.integers(0, 22, m), rng)
        node = node_of_point[vis].copy()
        point = vis.copy()
        k = n - m                                                   # clutter: features of nothing in the cloud
        xy = np.concatenate([xy, rng.uniform([0, 0], [W, H], (k, 2))])
        octave = np.concatenate([octave, rng.integers(0, 8, k)])
        desc = np.concatenate([desc, rng.integers(0, 256, (k, 32), dtype=np.uint8)])
        node = np.concatenate([node, rng.integers(0, n_nodes, k) * 7 + 3])
        point = np.concatenate([point, np.full(k, -1)])
        if disjoint:
            node = node + 1
        Tcw = np.concatenate([R, t[:, None]], 1).astype(f)
        Ow = (-(Tcw[:, :3].T @ Tcw[:, 3])).astype(f)
        has = (rng.random(n) < has_mp_frac).astype(np.uint8)
        return dict(desc=desc, has_mp=has, kp_xy=xy.astype(f), octave=octave.astype(np.int32),
                    angle=rng.uniform(0, 360, n).astype(f), node=node.astype(np.int64), point=point, intr=intr, Tcw=Tcw, Ow=Ow,
                    level_sigma2=LEVEL_SIGMA2.copy(), scale_factors=SCALE_FACTORS.copy(), scale_factor=f(1.2), n_seen=m)

    cur = make_view(np.eye(3), np.zeros(3))
    free = cur["n_seen"]
    # twins: clutter slots of the current keyframe become second features on points it already sees
    for s in range(free, min(n, free + int(twin_frac * n))):
        src = int(rng.integers(0, free))
        cur["kp_xy"][s] = cur["kp_xy"][src] + f(0.25)
        cur["octave"][s] = cur["octave"][src]
        cur["desc"][s] = flip_bits(cur["desc"][src:src + 1], [1], rng)[0]
        cur["node"][s] = cur["node"][src]; cur["point"][s] = cur["point"][src]; cur["has_mp"][s] = 0; cur["has_mp"][src] = 0
    if all_have_mp:
        cur["has_mp"][:] = 1
    nbs = []
    for b in range(n_nb):
        base = 1e-3 if b == zero_baseline_nb else rng.uniform(0.25, 1.1)
        c = rng.normal(0, 1, 3); c[2] *= 0.4
        if forward_every and b % forward_every == forward_every - 1:
            c = np.array([rng.normal(0, 0.08), rng.normal(0, 0.08), rng.choice([-1.0, 1.0])])
        c = c / np.linalg.norm(c) * base
        R = _rot(rng.normal(0, 0.04, 3) * (0.0 if b == zero_baseline_nb else 1.0))
        v = make_view(R, -R @ c, disjoint=(b == no_shared_nb))
        v.update(dict(zip(("F12", "ex", "ey"), new_points_prelude(cur, v))))
        m = v["n_seen"]
        slots = list(range(m, n))
        jump = rng.random(m) < octave_jump_frac
        v["octave"][:m][jump] = np.clip(v["octave"][:m][jump] + rng.choice([-4, 4], int(jump.sum())), 0, 7)
        row = {int(q): i for i, q in enumerate(cur["point"][:free])}
        for j in np.flatnonzero(rng.random(m) < cross_frac):
            i = row.get(int(v["point"][j]))
            if i is None or cur["octave"][i] > 2:
                continue
            x1, y1 = cur["kp_xy"][i].astype(np.float64)
            F = v["F12"].astype(np.float64)
            la, lb = x1 * F[0, 0] + y1 * F[1, 0] + F[2, 0], x1 * F[0, 1] + y1 * F[1, 1] + F[2, 1]
            nrm = np.hypot(la, lb)
            if not nrm > 0:
                continue
            v["kp_xy"][j] += (np.array([la, lb]) / nrm * rng.uniform(3.0, 6.5) * rng.choice([-1, 1])).astype(f)
            v["octave"][j] = 7
        n_tie, n_decoy = int(tie_frac * n), int(decoy_frac * n)
        for s in slots[:n_tie]:                                    # an identical feature a quarter pixel away, later in the node
            src = int(rng.integers(0, m))
            v["kp_xy"][s] = v["kp_xy"][src] + f(0.25)
            for k in ("octave", "desc", "node", "point"):
                v[k][s] = v[k][src]
            v["has_mp"][s] = v["has_mp"][src] = 0
        for s in slots[n_tie:n_tie + n_decoy]:                     # a copy of a current feature somewhere on its epipolar line
            i = int(rng.integers(0, free))
            x1, y1 = cur["kp_xy"][i].astype(np.float64)
            F = v["F12"].astype(np.float64)
            la, lb, lc = x1 * F[0, 0] + y1 * F[1, 0] + F[2, 0], x1 * F[0, 1] + y1 * F[1, 1] + F[2, 1], x1 * F[0, 2] + y1 * F[1, 2] + F[2, 2]
            if abs(lb) > abs(la):
                x2 = rng.uniform(0, W); y2 = -(la * x2 + lc) / lb
            else:
                y2 = rng.uniform(0, H); x2 = -(lb * y2 + lc) / la
            if not (np.isfinite(x2) and np.isfinite(y2)):
                continue
            v["kp_xy"][s] = (x2, y2)
            v["desc"][s] = flip_bits(cur["desc"][i:i + 1], [int(rng.integers(0, 4))], rng)[0]
            v["node"][s] = cur["node"][i] + (1 if b == no_shared_nb else 0)
            v["octave"][s] = cur["octave"][i]; v["has_mp"][s] = 0; v["point"][s] = -2
        nbs.append(v)
    return dict(cur=cur, neighbours=nbs)


# ---- a keyframe and its fuse targets for LocalMapping::SearchInNeighbors --------------------------------------------------------
def fuse_dist3d(X, Ow):
    """dist3D of Fuse's prelude: f32 difference, squares summed in f64, rounded to f32"""
    PO = (np.asarray(X, np.float32) - np.asarray(Ow, np.float32)).astype(np.float64)
    return np.sqrt((PO * PO).sum(-1)).astype(np.float32)


def make_fuse_scene(n_first=20, n_second=5, n=1000, seed=0, dup_frac=0.5, same_frac=0.15, has_mp_frac=0.8, dnr_frac=0.03, bad_frac=0.03,
                    behind=8, outside=8, off_cone=8, boundary=24, repeat_second=True, third_pairs=40):
    """A current keyframe, `n_first` first neighbours and up to `n_second` second neighbours each, looking at one seeded point cloud.
    Every keyframe's features are projections of the cloud plus pixel noise, octaves follow depth, descriptors a per-point base with bits
    flipped per observation.  The map points (one row each in `points`) and the knobs that force each outcome:
      dup_frac       a target's feature on a cloud point the current keyframe also holds carries a second point (a duplicate): the
                     searches pair the two both ways (MapPoint::Replace in the member)
      same_frac      ... or carries the very point the current slot holds (already in the target: skipped live by the member)
      has_mp_frac    share of features that carry a point at all
      dnr_frac       points with mbDoNotReplace; bad_frac  points already bad (skip = 1, kept in the slots)
      repeat_second  a second neighbour may be listed under several first neighbours (entries repeat a row)
      behind / outside / off_cone   extra points in the current slots and the candidates: behind the cameras, projecting outside the
                     image, or with the normal turned away (outside the 60-degree cone)
      third_pairs    duplicate pairs also observed, at different indices, by a third keyframe that is no target (third_point)
      boundary       points whose mfMaxDistance / dist3D sits within a few ulps of 1.2^k for the current keyframe (candidates) or for
                     target 0 (current slots): PredictScale's level hangs on the last bit of logf
    Returns dict(cur, targets (distinct keyframes), entries (target rows in list order), target_point (per target, the point row of
    each slot or -1), points, cur_point, cand, conn (ordered connections: [0] the current keyframe's as target rows, [1 + t] target
    t's, -1 = the current keyframe), third_point, boundary_rows); cand is the first-seen union of the targets' points over entries that are not bad."""
    rng = np.random.default_rng(seed)
    f = np.float32
    intr = (f(458.654), f(457.296), f(367.215), f(248.375))
    W, H = 752, 480
    lsf = f(np.log(f(1.2)))
    P0 = int(n * 1.4)
    X = np.stack([rng.uniform(-5, 5, P0), rng.uniform(-3.2, 3.2, P0), rng.uniform(4.0, 12.0, P0)], 1).astype(f)
    base_desc = rng.integers(0, 256, size=(P0, 32), dtype=np.uint8)
    d_ref = np.linalg.norm(X.astype(np.float64), axis=1)
    l0 = rng.integers(0, 4, P0)
    maxd = (d_ref * SCALE_FACTORS[l0]).astype(f)
    mind = (maxd / SCALE_FACTORS[7]).astype(f)
    pts = dict(pos=[], normal=[], max_d=[], min_d=[], desc=[], skip=[])
    dup_of = {}

    def add_point(x, nrm, mx, mn, desc, skip=0):
        pts["pos"].append(np.asarray(x, f)); pts["normal"].append(np.asarray(nrm, f)); pts["max_d"].append(f(mx)); pts["min_d"].append(f(mn))
        pts["desc"].append(np.asarray(desc, np.uint8)); pts["skip"].append(int(skip))
        return len(pts["skip"]) - 1

    def unit(v):
        v = np.asarray(v, np.float64)
        return (v / np.linalg.norm(v)).astype(f)

    def make_kf(R, t):
        Xc = X.astype(np.float64) @ R.T + t
        z = Xc[:, 2]
        u = intr[0] * Xc[:, 0] / z + intr[2]
        v = intr[1] * Xc[:, 1] / z + intr[3]
        vis = np.flatnonzero((z > 0.5) & (u > 0) & (u < W) & (v > 0) & (v < H) & (rng.random(P0) < 0.85))
        vis = rng.permutation(vis)[: n - n // 8]
        m = len(vis)
        xy = np.stack([u[vis], v[vis]], 1) + rng.normal(0, 0.5, (m, 2))
        Tcw = np.concatenate([R, t[:, None]], 1).astype(f)
        Ow = (-(Tcw[:, :3].T @ Tcw[:, 3])).astype(f)
        dist = fuse_dist3d(X[vis], Ow).astype(np.float64)
        octave = np.clip(np.ceil(np.log(maxd[vis] / dist) / np.log(1.2)), 0, 7).astype(np.int64)
        octave = np.where(rng.random(m) < 0.2, np.maximum(octave - 1, 0), octave)
        desc = flip_bits(base_desc[vis], rng.integers(0, 20, m), rng)
        k = n - m
        xy = np.concatenate([xy, rng.uniform([0, 0], [W, H], (k, 2))]).astype(f)
        octave = np.concatenate([octave, rng.integers(0, 8, k)]).astype(np.int32)
        desc = np.concatenate([desc, rng.integers(0, 256, (k, 32), dtype=np.uint8)])
        return dict(desc=desc, kp_xy=xy, octave=octave, angle=np.zeros(n, f), bounds=(0, 0, W, H), cols=64, rows=48, intr=intr, Tcw=Tcw,
                    Ow=Ow, scale_factors=SCALE_FACTORS.copy(), inv_level_sigma2=INV_LEVEL_SIGMA2.copy(), log_scale_factor=lsf,
                    world=np.concatenate([vis, np.full(k, -1)]))

    cur = make_kf(np.eye(3), np.zeros(3))
    n_pool = n_first + max(0, n_second * n_first // 3)
    targets = []
    for b in range(n_pool):
        c = rng.normal(0, 1, 3); c[2] *= 0.4
        c = c / np.linalg.norm(c) * rng.uniform(0.2, 1.0)
        R = _rot(rng.normal(0, 0.04, 3))
        targets.append(make_kf(R, -R @ c))
    # the current keyframe's points
    cur_row = {}
    cur_point = np.full(n, -1, np.int32)
    for i, w in enumerate(cur["world"]):
        if w < 0 or rng.random() >= has_mp_frac:
            continue
        r = add_point(X[w], unit(X[w] - cur["Ow"]), maxd[w], mind[w], flip_bits(base_desc[w:w + 1], [rng.integers(0, 10)], rng)[0],
                      rng.random() < dnr_frac + bad_frac)
        cur_row[int(w)] = r
        cur_point[i] = r
    # the targets' points: the current keyframe's own, duplicates of them, or points of their own
    target_point = []
    for k in targets:
        tp = np.full(n, -1, np.int32)
        for j, w in enumerate(k["world"]):
            if w < 0 or rng.random() >= has_mp_frac:
                continue
            a = rng.random()
            if int(w) in cur_row and a < same_frac:
                tp[j] = cur_row[int(w)]
                continue
            if int(w) not in cur_row or a < same_frac + dup_frac:
                xw = X[w] + rng.normal(0, 0.002, 3).astype(f)
                tp[j] = add_point(xw, unit(xw - k["Ow"]), maxd[w], mind[w], flip_bits(base_desc[w:w + 1], [rng.integers(0, 10)], rng)[0],
                                  rng.random() < dnr_frac + bad_frac)
                if int(w) in cur_row:
                    dup_of[int(tp[j])] = cur_row[int(w)]
        target_point.append(tp)
    # the entry list: each first neighbour, then up to n_second second neighbours from the rest of the pool
    entries, seconds = [], []
    for b in range(n_first):
        entries.append(b)
        pool = np.arange(n_first, n_pool) if n_pool > n_first else np.arange(0)
        pick = []
        if len(pool):
            pick = [int(p) for p in rng.choice(pool, size=min(n_second, len(pool)), replace=False)]
            if not repeat_second:
                pick = [p for p in pick if p not in entries]
            entries.extend(pick)
        seconds.append(pick)
    used = sorted(set(entries))
    remap = {r: i for i, r in enumerate(used)}
    targets = [targets[r] for r in used]
    target_point = [target_point[r] for r in used]
    entries = [remap[r] for r in entries]
    # each keyframe's ordered connections for the stand-in objects (-1: the current keyframe, which the member skips as a second)
    conn = [[remap[b] for b in range(n_first)]] + [[] for _ in targets]
    for b in range(n_first):
        c = [remap[p] for p in seconds[b]]
        c.insert(int(rng.integers(0, len(c) + 1)), -1)
        conn[1 + remap[b]] = c
    skip = np.asarray(pts["skip"], np.uint8)
    bad = skip & (rng.random(len(skip)) < bad_frac / max(dnr_frac + bad_frac, 1e-9)).astype(np.uint8)
    cand, seen = [], set()
    for e in entries:
        for r in target_point[e]:
            if r >= 0 and not bad[r] and r not in seen:
                seen.add(int(r)); cand.append(int(r))
    # the knob points, each in a free slot of the current keyframe and at the end of the candidates
    free = list(np.flatnonzero(cur_point < 0))
    rng.shuffle(free)

    def knob(x, nrm, mx, mn, desc):
        r = add_point(x, nrm, mx, mn, desc)
        if free:
            cur_point[free.pop()] = r
        cand.append(r)
    seen_w = [int(w) for w in cur["world"] if w >= 0]
    for _ in range(behind):
        w = seen_w[rng.integers(len(seen_w))]
        x = X[w] * f(-1.0)
        knob(x, unit(x), maxd[w], mind[w], base_desc[w])
    for _ in range(outside):
        w = seen_w[rng.integers(len(seen_w))]
        x = X[w] + np.array([rng.choice([-1, 1]) * 40.0, 0, 0], f)
        knob(x, unit(x), maxd[w] * 4, mind[w], base_desc[w])
    for _ in range(off_cone):
        w = seen_w[rng.integers(len(seen_w))]
        knob(X[w], -unit(X[w]), maxd[w], mind[w], base_desc[w])
    boundary_rows = []
    for b in range(boundary):
        w = seen_w[rng.integers(len(seen_w))]
        fwd = b % 2 == 0 and len(targets) > 0
        Ow = targets[0]["Ow"] if fwd else cur["Ow"]
        d = fuse_dist3d(X[w], Ow)
        mx = np.float32(np.float64(d) * 1.2 ** int(rng.integers(1, 5)))
        off = int(rng.integers(0, 9)) - 4                           # a few ulps either side of the boundary
        for _ in range(abs(off)):
            mx = np.nextafter(mx, np.float32(np.inf if off > 0 else -np.inf), dtype=np.float32)
        r = add_point(X[w], unit(X[w] - Ow), mx, mx / SCALE_FACTORS[7], base_desc[w])
        boundary_rows.append(r)
        if fwd:
            if free:
                cur_point[free.pop()] = r
        else:
            cand.append(r)
    points = {k: np.asarray(v) for k, v in pts.items()}
    points["skip"] = points["skip"].astype(np.uint8)
    points["bad"] = np.zeros(len(points["skip"]), np.uint8); points["bad"][:len(bad)] = bad
    # a third keyframe observing duplicate pairs (a current point and its duplicate in a target) at different indices: Replace's
    # id-mismatch branch when the pair fuses
    pairs = [(a, b) for b, a in dup_of.items() if cur_point.tolist().count(a) == 1][:third_pairs]
    third = np.full(n, -1, np.int32)
    for q, (a, b) in enumerate(pairs):
        third[2 * q], third[2 * q + 1] = a, b
    return dict(cur=cur, targets=targets, entries=entries, target_point=target_point, points=points, cur_point=cur_point,
                cand=np.asarray(cand, np.int32), conn=conn, third_point=third, boundary_rows=np.asarray(boundary_rows, np.int64))


def fuse_scene_arrays(sc):
    """The parts of a make_fuse_scene dict that api.fuse_neighbours reads, as flat named arrays (for np.savez)"""
    out = dict(cur_point=sc["cur_point"], cand=sc["cand"], n_targets=np.int64(len(sc["targets"])))
    for k, v in sc["points"].items():
        out["points_" + k] = np.asarray(v)
    for i, kf in enumerate([sc["cur"]] + list(sc["targets"])):
        for k in ("desc", "kp_xy", "octave", "angle", "bounds", "cols", "rows", "intr", "Tcw", "Ow", "scale_factors", "inv_level_sigma2",
                  "log_scale_factor"):
            out["kf%d_%s" % (i, k)] = np.asarray(kf[k])
    return out


def fuse_scene_from_arrays(z):
    """inverse of fuse_scene_arrays"""
    kfs = []
    for i in range(1 + int(z["n_targets"])):
        kf = {k: z["kf%d_%s" % (i, k)] for k in ("desc", "kp_xy", "octave", "angle", "intr", "Tcw", "Ow", "scale_factors", "inv_level_sigma2")}
        kf["bounds"] = tuple(float(b) for b in z["kf%d_bounds" % i])
        kf["cols"], kf["rows"] = int(z["kf%d_cols" % i]), int(z["kf%d_rows" % i])
        kf["log_scale_factor"] = np.float32(z["kf%d_log_scale_factor" % i])
        kfs.append(kf)
    points = {k[len("points_"):]: z[k] for k in z.files if k.startswith("points_")}
    return dict(cur=kfs[0], targets=kfs[1:], points=points, cur_point=z["cur_point"], cand=z["cand"])


# ---- the corrected keyframes and the loop points of LoopFinder / MapMerger::SearchAndFuse ------------------------------------
def split_scw(S):
    """Fuse(Scw)'s split (S/ORBmatcher.cpp:1004-1008) over the f32 4x4 Scw, rounded as its cv::Mat expressions round: scw = sqrt of the
    f64 dot of row 0 of sRcw, rounded to f32; Rcw = sRcw/scw and tcw = t/scw each an f64 quotient rounded to f32; Ow = -Rcw^T tcw with
    cv::gemm's f32 products summed left to right.  Returns (Tcw (3,4) f32, Ow (3,) f32)."""
    S = np.asarray(S, np.float32)
    d = 0.0
    for c in range(3):
        d += float(S[0, c]) * float(S[0, c])
    scw = np.float32(np.sqrt(d))
    R = (S[:3, :3].astype(np.float64) / np.float64(scw)).astype(np.float32)
    t = (S[:3, 3].astype(np.float64) / np.float64(scw)).astype(np.float32)
    return np.concatenate([R, t[:, None]], 1), _neg_rt_t(R, t)


def _neg_rt_t(R, t):
    """-R^T t as the reference computes it: (-R).t() * t, f32 products summed left to right"""
    Ow = np.empty(3, np.float32)
    for r in range(3):
        s = np.float32(-R[0, r]) * t[0]
        s = np.float32(s + np.float32(-R[1, r]) * t[1])
        Ow[r] = np.float32(s + np.float32(-R[2, r]) * t[2])
    return Ow


def _libm_logf():
    """glibc's logf, which PredictScale's log(float) is"""
    import ctypes
    f = ctypes.CDLL("libm.so.6").logf
    f.restype = ctypes.c_float
    f.argtypes = [ctypes.c_float]
    return f


def _sim3_of(R, t, s):
    """g2o::Sim3(R, t, s) as qx qy qz qw tx ty tz s (f64)"""
    from scipy.spatial.transform import Rotation
    return np.concatenate([Rotation.from_matrix(R).as_quat(), t, [s]]).astype(np.float64)


def _orb_levels():
    """mvScaleFactors as ORBextractor builds them (each level the previous times 1.2f), mvInvLevelSigma2 and mfLogScaleFactor"""
    sf = np.empty(8, np.float32); sf[0] = 1
    for i in range(1, 8):
        sf[i] = np.float32(sf[i - 1] * np.float32(1.2))
    return sf, (np.float32(1) / (sf * sf)).astype(np.float32), np.float32(np.log(np.float32(1.2)))


def make_search_and_fuse_scene(kind="loop", n_kf=6, n=500, n_loop=None, seed=0, held_frac=0.1, occupied_frac=0.4, dup=20, bad_frac=0.03,
                               dnr_frac=0.03, behind=8, outside=8, off_cone=8, boundary=24, far_frac=0.05, camera_probe=16):
    """The corrected keyframes of a loop closure (kind "loop", s = 1) or a map merge (kind "merge", s != 1 per keyframe) and the loop
    points vpLoopMapPoints, all looking at one seeded cloud.  Each keyframe's features are projections of the cloud through its pose plus
    pixel noise, octaves follow depth, descriptors a per-point base with bits flipped.  The corrected Sim3 of keyframe k is
    Scw = Sim3(R, s*t, s) of its pose [R | t]; its ccm_fuse_kf camera (Tcw, Ow) is Fuse(Scw)'s split of the f32 Scw (split_scw), and
    Tcw_pose / Ow_pose hold the [R t/s] pose the keyframe itself stores, which differs from the split in rounding; sim3 is the g2o Sim3
    itself (qx qy qz qw tx ty tz s).
    The loop points (one row each in `points`) and the knobs:
      held_frac       a keyframe's feature on a loop point's cloud point holds that very loop point (in spAlreadyFound)
      occupied_frac   ... or holds a point of its own (kf_slot -2: an occupant that Replace would merge)
      dup             pairs of loop points on one cloud point: both claim the same keypoint
      bad_frac        points already bad (skip = 1); dnr_frac  points with mbDoNotReplace (dnr = 1, searched all the same)
      behind / outside / off_cone   points behind the cameras, projecting outside the image, or with the normal turned away
      boundary        points whose mfMaxDistance / dist3D sits within a few ulps of 1.2^k for keyframe 0's split centre: PredictScale's
                      level hangs on the last bit of logf
      far_frac        features placed 3.1 to 3.9 scale units from their projection (found with th = 4 only, and only without the
                      chi-square gate of Fuse(kf, points))
      camera_probe    points on keyframe 0 whose PredictScale level differs between the split centre and the [R t/s] pose's centre,
                      at a level where their keypoint is searched under one of the two only
    Returns dict(kind, kfs, points (pos, normal, max_d, min_d, desc, skip, dnr, world), kf_slot (per keyframe, per feature: the loop
    row held, -2 an occupant, -1 empty), boundary_rows)."""
    rng = np.random.default_rng(seed)
    f = np.float32
    n_loop = int(n_loop or 3 * n)
    intr = (f(458.654), f(457.296), f(367.215), f(248.375))
    W, H = 752, 480
    sf, ils2, lsf = _orb_levels()
    P0 = int(n_loop * 1.1)
    X = np.stack([rng.uniform(-5, 5, P0), rng.uniform(-3.2, 3.2, P0), rng.uniform(4.0, 12.0, P0)], 1).astype(f)
    base_desc = rng.integers(0, 256, size=(P0, 32), dtype=np.uint8)
    d_ref = np.linalg.norm(X.astype(np.float64), axis=1)
    l0 = rng.integers(0, 4, P0)
    maxd = (d_ref * sf[l0]).astype(f)
    mind = (maxd / sf[7]).astype(f)

    def unit(v):
        v = np.asarray(v, np.float64)
        return (v / np.linalg.norm(v)).astype(f)

    # the loop points: most of the cloud, a few twice (dup), then the knob points
    world = list(rng.permutation(P0)[:n_loop - dup - behind - outside - off_cone - boundary])
    world += [int(w) for w in rng.choice(world, size=dup, replace=False)]
    m = len(world)
    pts = dict(pos=(X[world] + rng.normal(0, 0.002, (m, 3))).astype(f), normal=np.stack([unit(X[w]) for w in world]).astype(f),
               max_d=maxd[world].copy(), min_d=mind[world].copy(), desc=flip_bits(base_desc[world], rng.integers(0, 10, m), rng))
    kfs = []
    for k in range(n_kf):
        c = rng.normal(0, 1, 3); c[2] *= 0.4
        c = c / np.linalg.norm(c) * rng.uniform(0.2, 1.0)
        R = _rot(rng.normal(0, 0.04, 3))
        t = -R @ c
        s = 1.0 if kind == "loop" else float(rng.uniform(0.6, 1.6))
        S = np.eye(4); S[:3, :3] = s * R; S[:3, 3] = s * t
        S = S.astype(f)                                                         # Converter::toCvMat(g2oScw)
        Tcw, Ow = split_scw(S)
        Rp = R.astype(f); tp = (s * t / s).astype(f)                            # the keyframe's pose [R t/s]
        Xc = X.astype(np.float64) @ R.T + t
        z = Xc[:, 2]
        u = intr[0] * Xc[:, 0] / z + intr[2]
        v = intr[1] * Xc[:, 1] / z + intr[3]
        vis = np.flatnonzero((z > 0.5) & (u > 0) & (u < W) & (v > 0) & (v < H) & (rng.random(P0) < 0.85))
        vis = rng.permutation(vis)[: n - n // 8]
        mv = len(vis)
        xy = np.stack([u[vis], v[vis]], 1) + rng.normal(0, 0.5, (mv, 2))
        dist = fuse_dist3d(X[vis], Ow).astype(np.float64)
        octave = np.clip(np.ceil(np.log(maxd[vis] / dist) / np.log(1.2)), 0, 7).astype(np.int64)
        octave = np.where(rng.random(mv) < 0.2, np.maximum(octave - 1, 0), octave)
        far = rng.random(mv) < far_frac                 # 3 to 4 radii out: inside th = 4, outside th = 3 and the chi-square gate
        xy[far, 0] += rng.choice([-1, 1], far.sum()) * rng.uniform(3.1, 3.9, far.sum()) * sf[octave[far]]
        desc = flip_bits(base_desc[vis], rng.integers(0, 20, mv), rng)
        r = n - mv
        kfs.append(dict(desc=np.concatenate([desc, rng.integers(0, 256, (r, 32), dtype=np.uint8)]),
                        kp_xy=np.concatenate([xy, rng.uniform([0, 0], [W, H], (r, 2))]).astype(f),
                        octave=np.concatenate([octave, rng.integers(0, 8, r)]).astype(np.int32), angle=np.zeros(n, f), bounds=(0, 0, W, H),
                        cols=64, rows=48, intr=intr, sim3=_sim3_of(R, s * t, s), Scw=S, Tcw=Tcw, Ow=Ow, Tcw_pose=np.concatenate([Rp, tp[:, None]], 1),
                        Ow_pose=_neg_rt_t(Rp, tp), scale_factors=sf.copy(), inv_level_sigma2=ils2.copy(), log_scale_factor=lsf,
                        world=np.concatenate([vis, np.full(r, -1)])))
    # the knob points
    seen = [int(w) for w in kfs[0]["world"] if w >= 0]
    knobs = dict(pos=[], normal=[], max_d=[], min_d=[], desc=[], world=[])

    def knob(x, nrm, mx, mn, w):
        knobs["pos"].append(np.asarray(x, f)); knobs["normal"].append(np.asarray(nrm, f)); knobs["max_d"].append(f(mx))
        knobs["min_d"].append(f(mn)); knobs["desc"].append(base_desc[w]); knobs["world"].append(w)
    for _ in range(behind):
        w = seen[rng.integers(len(seen))]
        knob(X[w] * f(-1.0), unit(X[w] * -1.0), maxd[w], mind[w], w)
    for _ in range(outside):
        w = seen[rng.integers(len(seen))]
        x = X[w] + np.array([rng.choice([-1, 1]) * 40.0, 0, 0], f)
        knob(x, unit(x), maxd[w] * 4, mind[w], w)
    for _ in range(off_cone):
        w = seen[rng.integers(len(seen))]
        knob(X[w], -unit(X[w]), maxd[w], mind[w], w)
    Ow0 = kfs[0]["Ow"]
    for _ in range(boundary):
        w = seen[rng.integers(len(seen))]
        d = fuse_dist3d(X[w], Ow0)
        mx = np.float32(np.float64(d) * 1.2 ** int(rng.integers(1, 5)))
        off = int(rng.integers(0, 9)) - 4                           # a few ulps either side of the boundary
        for _ in range(abs(off)):
            mx = np.nextafter(mx, np.float32(np.inf if off > 0 else -np.inf), dtype=np.float32)
        knob(X[w], unit(X[w] - Ow0), mx, mx / sf[7], w)
    logf = _libm_logf()
    j_of = {int(w): j for j, w in enumerate(kfs[0]["world"]) if w >= 0}
    made = 0
    for w in rng.permutation(seen):
        if made >= camera_probe:
            break
        x = X[w]
        ds, dp = fuse_dist3d(x, Ow0), fuse_dist3d(x, kfs[0]["Ow_pose"])
        if ds == dp:
            continue
        o = int(kfs[0]["octave"][j_of[int(w)]])
        if o > 5:
            continue
        mx = np.float32(np.float64(ds) * 1.2 ** (o + 1))
        mx = np.nextafter(mx, np.float32(-np.inf), dtype=np.float32)
        for _ in range(24):
            mx = np.nextafter(mx, np.float32(np.inf), dtype=np.float32)
            ls = int(np.ceil(np.float32(logf(np.float32(mx / ds)) / lsf)))
            lp = int(np.ceil(np.float32(logf(np.float32(mx / dp)) / lsf)))
            if ls != lp:
                knob(x, unit(x - Ow0), mx, mx / sf[7], w)
                made += 1
                break
    for key in ("pos", "normal", "max_d", "min_d", "desc"):
        pts[key] = np.concatenate([pts[key], np.asarray(knobs[key]).reshape((-1,) + pts[key].shape[1:]).astype(pts[key].dtype)])
    pts["world"] = np.asarray(world + knobs["world"], np.int64)
    P = len(pts["world"])
    boundary_rows = np.arange(P - boundary - made, P - made)
    flag = rng.random(P)
    pts["skip"] = (flag < bad_frac).astype(np.uint8)
    pts["dnr"] = ((flag >= bad_frac) & (flag < bad_frac + dnr_frac)).astype(np.uint8)
    # what each keyframe holds: a loop point on the feature's cloud point, an occupant of its own, or nothing
    row_of = {}
    for i, w in enumerate(world):
        row_of.setdefault(int(w), i)
    kf_slot = []
    for kf in kfs:
        sl = np.full(n, -1, np.int32)
        for j, w in enumerate(kf["world"]):
            a = rng.random()
            if w >= 0 and int(w) in row_of and a < held_frac:
                sl[j] = row_of[int(w)]
            elif a < held_frac + occupied_frac:
                sl[j] = -2
        kf_slot.append(sl)
    return dict(kind=kind, kfs=kfs, points=pts, kf_slot=kf_slot, boundary_rows=boundary_rows)


_SF_KF_KEYS = ("desc", "kp_xy", "octave", "angle", "bounds", "cols", "rows", "intr", "Scw", "Tcw", "Ow", "Tcw_pose", "Ow_pose", "scale_factors",
               "inv_level_sigma2", "log_scale_factor")


def search_and_fuse_scene_arrays(sc):
    """The parts of a make_search_and_fuse_scene dict that api.search_and_fuse reads, as flat named arrays (np.savez)"""
    out = dict(n_kf=np.int64(len(sc["kfs"])))
    for k, v in sc["points"].items():
        out["points_" + k] = np.asarray(v)
    for i, kf in enumerate(sc["kfs"]):
        for k in _SF_KF_KEYS:
            out["kf%d_%s" % (i, k)] = np.asarray(kf[k])
    return out


def search_and_fuse_scene_from_arrays(z):
    """inverse of search_and_fuse_scene_arrays"""
    kfs = []
    for i in range(int(z["n_kf"])):
        kf = {k: z["kf%d_%s" % (i, k)] for k in _SF_KF_KEYS}
        kf["bounds"] = tuple(float(b) for b in kf["bounds"])
        kf["cols"], kf["rows"] = int(kf["cols"]), int(kf["rows"])
        kf["log_scale_factor"] = np.float32(kf["log_scale_factor"])
        kfs.append(kf)
    points = {k[len("points_"):]: z[k] for k in z.files if k.startswith("points_")}
    return dict(kfs=kfs, points=points)
