"""NumPy restatement of the 2D keypoint merge of the keypoint-free SfM coarse matching
(src/KeypointFreeSfM/coarse_match: Match2Pts2D, points2D_worker with agg_groupby_2d(agg="sum"),
update_matches and transform_points2D), with every quirk that decides a bit written out:

  * An image's observations are the rows (x, y, conf) of every pair that names it, pairs in the
    order of the matches dict, rows in match order; a pair naming one image twice gives all its
    side-0 rows, then all its side-1 rows (Match2Pts2D appends (k, 0) before (k, 1)).
  * Coordinates are truncated toward zero (.astype(int) on the float32 columns).
  * A keypoint's score is the fp64 sum of the float32 confs of its observations, in observation
    order (np.bincount with float64 weights adds sequentially).
  * Keypoint ids rank the unique (x, y) by descending sum; ties keep np.unique's ascending
    lexicographic (x, y) order, because sorted(reverse=True) is stable.
  * Keypoints are float32 (x, y) in id order, scores the sums rounded to float32; index matches are
    int64 [id0, id1] in match order, an empty pair gives an empty int64 [0, 2].

Pure NumPy, no reference import: the GPU tests compare the kernels against this module.
"""
import random

import numpy as np

PAIR_SPLIT = " "


def pair_lines(text, seed=None):
    """The pair list LoftrCoarseDataset reads: the file's text without its trailing newlines, split at
    newlines, shuffled by Python's random module (seeded first when `seed` is given)."""
    lines = text.rstrip("\n").split("\n")
    if seed is not None:
        random.seed(seed)
    random.shuffle(lines)
    return lines


def observations(matches, name):
    """Float32 [n, 3] rows (x, y, conf) of `name`, in Match2Pts2D order."""
    rows = []
    for k, v in matches.items():
        n0, n1 = k.split(PAIR_SPLIT)
        if n0 == name:
            rows.append(v[:, [0, 1, 4]])
        if n1 == name:
            rows.append(v[:, [2, 3, 4]])
    return np.concatenate(rows, 0) if rows else np.empty((0, 3), np.float32)


def merge_image(obs):
    """One image: (unique xy int64 [K, 2] in id order, sums fp64 [K] in id order)."""
    xy = obs[:, :2].astype(np.int64)
    w = obs[:, 2].astype(np.float64)
    order = np.lexsort((xy[:, 1], xy[:, 0]))                 # ascending (x, y), stable
    sx = xy[order]
    head = np.ones(len(order), bool)
    head[1:] = np.any(sx[1:] != sx[:-1], axis=1)
    group_sorted = np.cumsum(head) - 1
    group = np.empty(len(order), np.int64)
    group[order] = group_sorted
    uniq = sx[head]
    sums = np.bincount(group, weights=w, minlength=len(uniq))   # sequential, in observation order
    rank = np.argsort(-sums, kind="stable")                  # descending; ties keep (x, y) order
    return uniq[rank], sums[rank]


def merge(matches, names):
    """matches: ordered dict "name0 name1" -> float32 [M, 5]; names: the image list.
    Returns (keypoints {name: float32 [K, 2]}, scores {name: float32 [K]}, idx {pair: int64 [M, 2]})."""
    kpts, scores, lookup = {}, {}, {}
    for name in names:
        uniq, sums = merge_image(observations(matches, name))
        if len(uniq) == 0:
            raise ValueError(f"image {name} has no keypoint")
        kpts[name] = uniq.astype(np.float32)
        scores[name] = sums.astype(np.float32)
        lookup[name] = {(int(x), int(y)): i for i, (x, y) in enumerate(uniq)}
    idx = {}
    for k, v in matches.items():
        n0, n1 = k.split(PAIR_SPLIT)
        p0, p1 = v[:, :2].astype(np.int64), v[:, 2:4].astype(np.int64)
        ids = [[lookup[n0][(int(a), int(b))], lookup[n1][(int(c), int(d))]] for (a, b), (c, d) in zip(p0, p1)]
        idx[k] = np.asarray(ids, np.int64).reshape(-1, 2)
    return kpts, scores, idx


def flat(matches, names):
    """The device merge's inputs from a matches dict: (matches fp32 [M, 5], offsets int64 [P + 1],
    pair_img int32 [P, 2]) in dict order."""
    ids = {n: i for i, n in enumerate(names)}
    keys = list(matches)
    rows = [matches[k].astype(np.float32).reshape(-1, 5) for k in keys]
    offsets = np.zeros(len(keys) + 1, np.int64)
    offsets[1:] = np.cumsum([len(r) for r in rows])
    pair_img = np.asarray([[ids[n] for n in k.split(PAIR_SPLIT)] for k in keys], np.int32).reshape(-1, 2)
    return np.concatenate(rows, 0) if rows else np.empty((0, 5), np.float32), offsets, pair_img


def seeded_matches(seed, n_images=12, n_pairs=30, max_matches=200, scale=(1.0, 1.0), grid=8, size=(480, 640),
                   empty_every=7, hub=None, tie_conf=False, one_sided=True):
    """A seeded matches dict shaped like the coarse matcher's output: coordinates on the 8-px grid
    times `scale` (non-integer for scale != 1), confs in (0.2, 1].  `hub` = (image, n): n pairs all
    hit one keypoint of that image.  `tie_conf` draws the confs from 4 values so sums tie exactly.
    `one_sided` adds two images seen only as name0 resp. only as name1.  Every image appears in a
    non-empty pair."""
    rng = np.random.default_rng(seed)
    names = [f"img/{seed}/{i:04d}.png" for i in range(n_images)]
    h, w = size
    pairs = []
    for i in range(n_images):                    # a chain of non-empty pairs: every image has a match
        pairs.append((i, (i + 1) % n_images, True) if n_images > 1 else (0, 0, True))
    while len(pairs) < n_pairs:
        a, b = rng.integers(0, n_images, 2)
        pairs.append((int(a), int(b), False))
    if one_sided:
        names += [f"img/{seed}/only0.png", f"img/{seed}/only1.png"]
        for j in range(3):
            pairs += [(n_images, j % n_images, True), (j % n_images, n_images + 1, True)]
    rng.shuffle(pairs)
    chain_keys = {PAIR_SPLIT.join((names[a], names[b])) for a, b, c in pairs if c}
    out = {}
    for pi, (a, b, _) in enumerate(pairs):
        k = PAIR_SPLIT.join((names[a], names[b]))
        if k in out:
            continue
        empty = empty_every and k not in chain_keys and pi % empty_every == 3
        m = 0 if empty else int(rng.integers(1, max_matches + 1))
        cx = rng.integers(0, w // grid, (m, 2)) * grid
        cy = rng.integers(0, h // grid, (m, 2)) * grid
        pts = np.stack([cx[:, 0] * scale[1], cy[:, 0] * scale[0], cx[:, 1] * scale[1], cy[:, 1] * scale[0]], 1)
        conf = rng.choice([0.25, 0.5, 0.75, 1.0], m) if tie_conf else rng.uniform(0.2, 1.0, m)
        out[k] = np.concatenate([pts, conf[:, None]], 1).astype(np.float32)
    if hub is not None:
        img, n = hub
        for j in range(n):
            other = names[(img + 1 + j) % n_images]
            k = PAIR_SPLIT.join((names[img], other) if j % 2 else (other, names[img]))
            row = np.array([[64, 96, 64, 96, rng.uniform(0.2, 1.0)]], np.float32)
            extra = out.pop(k, np.empty((0, 5), np.float32))
            out[k] = np.concatenate([extra, row], 0)
    return out, names
