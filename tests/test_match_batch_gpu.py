"""The matcher in the regimes the product runs: submissions of more than a thousand pairs (one train chunk per job,
the persistent tensor-core kernel walking mixed-size jobs, the 1024-pair carry of the result scan), images without
rows inside a batch, L2 distances next to the tensor-core kernel's norm bound, and the guided-matching epipolar
masks read back bit for bit.  Every result is compared with the reference's cv2 path (`oracle/match_oracle.py`)."""
import math

import numpy as np
import pytest

from oracle import match_oracle as mo
from opensfm_b200 import matching, synthetic as syn

pytestmark = pytest.mark.gpu
CFG = {"lowes_ratio": 0.8}
# image sizes around the kernels' tile edges: 32-bit mask words, 64-row SIMT tiles, 128-row train tiles, 256-row
# tensor-core query tiles
EDGE_SIZES = [1, 2, 31, 127, 128, 129, 255, 256, 257, 511, 513]
BIG_SIZES = [2000, 3100, 4000]


def _pairset(x):
    return sorted((int(a), int(b)) for a, b in x)


def _rows(x):
    return [tuple(r) for r in np.asarray(x, dtype=np.int64).reshape(-1, 2).tolist()]


def _num_sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------
# Thousand-pair submissions
# ---------------------------------------------------------------------------------------------------------------
def _sizes(seed, n_images):
    rng = np.random.RandomState(seed)
    small = EDGE_SIZES + rng.randint(40, 420, n_images - len(EDGE_SIZES) - len(BIG_SIZES)).tolist()
    return small + BIG_SIZES


def _l2_images(sizes, seed):
    """HAHOG-like images drawn from one pool of scene points (with integer noise), so pairs share features."""
    rng = np.random.RandomState(seed)
    pool = syn.hahog_like_descriptors(1500, seed + 1)
    return [np.clip(pool[rng.choice(len(pool), n, replace=n > len(pool))] + rng.randint(-4, 5, (n, 128)), 0,
                    255).astype(np.float32) for n in sizes]


def _hamming_images(sizes, seed, nbytes=61):
    rng = np.random.RandomState(seed)
    pool = syn.binary_descriptors(1500, seed + 1, nbytes)
    out = []
    for n in sizes:
        d = pool[rng.choice(len(pool), n, replace=n > len(pool))].copy()
        d[:, rng.randint(0, nbytes, 3)] ^= rng.randint(0, 256, (n, 3)).astype(np.uint8)
        out.append(d)
    return out


def _float_images(sizes, seed, dim=96):
    rng = np.random.RandomState(seed)
    pool = rng.rand(1000, dim).astype(np.float32)
    return [pool[rng.choice(len(pool), n, replace=n > len(pool))] + rng.normal(0, 0.02, (n, dim)).astype(np.float32)
            for n in sizes]


def _pair_list(sizes, seed, n_pairs):
    """n_pairs pairs in shuffled order: (a, b) and (b, a) both present for a tenth of them, self-pairs, every big
    image against a handful of others and against each other."""
    rng = np.random.RandomState(seed)
    n = len(sizes)
    small = [i for i in range(n) if sizes[i] < 1000]
    big = [i for i in range(n) if sizes[i] >= 1000]
    pairs = [(small[0], small[0]), (small[5], small[5])]
    if big:
        pairs += [(big[0], big[1]), (big[1], big[0]), (big[2], big[2])]
    for b in big:
        for o in rng.choice(small, 6, replace=False):
            pairs += [(b, int(o)), (int(o), b)]
    seen = set(pairs)
    while len(pairs) < n_pairs:
        a, b = (int(x) for x in rng.choice(small, 2, replace=False))
        for p in ([(a, b), (b, a)] if rng.rand() < 0.1 else [(a, b)]):
            if p not in seen:
                seen.add(p)
                pairs.append(p)
    order = rng.permutation(len(pairs))
    return [pairs[i] for i in order]


def _reference(images, pairs, cfg=CFG):
    """cv2's one-way lists for both directions of every pair, and the symmetric sets built from them exactly like
    matching.py:759-777."""
    ow = {}
    for a, b in pairs:
        for p in ((a, b), (b, a)):
            if p not in ow:
                fa, fb = images[p[0]], images[p[1]]
                ow[p] = mo.match_brute_force(fa, fb, cfg) if len(fa) and len(fb) else []
    sym = {(a, b): _pairset(set(ow[(a, b)]) & {(q, t) for t, q in ow[(b, a)]}) for a, b in pairs}
    return ow, sym


def _query_tiles(images, pairs, tile):
    return sum((len(images[a]) + tile - 1) // tile + (len(images[b]) + tile - 1) // tile for a, b in pairs)


def _check_batch(pm, images, pairs, ref_ow, ref_sym, kernel, cfg=CFG):
    one = pm.match_pairs(pairs, cfg, symmetric=False)
    assert pm.last_kernel() == kernel
    for p in pairs:
        assert _rows(one[p]) == ref_ow[p], p
    sym = pm.match_pairs(pairs, cfg, symmetric=True)
    assert pm.last_kernel() == kernel
    for p in pairs:
        assert _pairset(sym[p]) == ref_sym[p], p
    return one, sym


@pytest.fixture(scope="module")
def l2_batch():
    sizes = _sizes(1, 80)
    images = _l2_images(sizes, 2)
    pairs = _pair_list(sizes, 3, 1100)
    ref_ow, ref_sym = _reference(images, pairs)
    return images, pairs, ref_ow, ref_sym


@pytest.mark.parametrize("variant", ["tensor_core", "simt", "uint8_stored"])
def test_thousand_pair_l2_submission_matches_cv2(l2_batch, variant):
    """1100 pairs of 1 ... 4000 features in one call: every job is one train chunk (enough query tiles to fill the
    GPU), the persistent tensor-core kernel decodes thousands of jobs, the result scan carries over 1024-pair
    blocks.  Then the same pairs one at a time on the same matcher (train split across CTAs, chunk merge in
    bf_top2_finalize) must give identical lists."""
    images, pairs, ref_ow, ref_sym = l2_batch
    assert len(pairs) > 1024
    assert _query_tiles(images, pairs, 256) >= 2 * _num_sms()    # planner: no train split at this size
    pm = matching.PairMatcher(kernel=1 if variant == "simt" else 0)
    if variant == "uint8_stored":
        pm.add_many([(i, d.astype(np.uint8)) for i, d in enumerate(images)], uint8_is_l2=True)
    else:
        pm.add_many(list(enumerate(images)))
    kernel = 1 if variant == "simt" else 2
    one, sym = _check_batch(pm, images, pairs, ref_ow, ref_sym, kernel)
    assert sum(len(v) for v in sym.values()) > 10000
    assert sum(len(v) > 0 for v in sym.values()) > len(pairs) // 2
    for p in pairs:
        alone = pm.match_pairs([p], CFG, symmetric=True)[p]
        assert pm.last_kernel() == kernel
        assert np.array_equal(alone, sym[p]), p
    for p in pairs[::7]:
        assert np.array_equal(pm.match_pairs([p], CFG, symmetric=False)[p], one[p]), p


def test_thousand_pair_submission_reuses_buffers_and_raw_results_agree(l2_batch):
    """big batch -> small batch -> big batch on one matcher (workspaces grown, then reused at a smaller size, then
    again), and the per-query results of fetch_raw() against the device-compacted lists of fetch_lists()."""
    images, pairs, ref_ow, ref_sym = l2_batch
    pm = matching.PairMatcher()
    pm.add_many(list(enumerate(images)))
    first = pm.match_pairs(pairs, CFG, symmetric=True)
    assert pm.last_kernel() == 2
    few = pairs[:9]
    small = pm.match_pairs(few, CFG, symmetric=True)
    for p in few:
        assert _pairset(small[p]) == ref_sym[p]
    again = pm.match_pairs(pairs, CFG, symmetric=True)
    for p in pairs:
        assert np.array_equal(again[p], first[p]), p
    pm.submit(pairs, CFG["lowes_ratio"], symmetric=False)
    lists = pm.fetch_lists()
    raw = pm.fetch_raw()
    counts = np.array([len(images[a]) for a, _ in pairs])
    assert len(raw) == counts.sum()
    for p, got, want in zip(pairs, lists, matching.split_match_lists(raw, counts)):
        assert np.array_equal(got, want), p
        assert _rows(got) == ref_ow[p], p


@pytest.mark.parametrize("kernel", [0, 1])
def test_thousand_pair_hamming_submission_matches_cv2(kernel):
    """AKAZE-sized binary descriptors, 1100 pairs in one call: the fp8 tensor-core kernel (3) and the popcount
    kernel (1), one chunk per job, then pair by pair."""
    sizes = _sizes(4, 80)
    images = _hamming_images(sizes, 5)
    pairs = _pair_list(sizes, 6, 1100)
    ref_ow, ref_sym = _reference(images, pairs)
    assert _query_tiles(images, pairs, 128) >= 2 * _num_sms()
    pm = matching.PairMatcher(kernel=kernel)
    pm.add_many(list(enumerate(images)))
    want = 3 if kernel == 0 else 1
    one, sym = _check_batch(pm, images, pairs, ref_ow, ref_sym, want)
    assert sum(len(v) for v in sym.values()) > 10000
    for p in pairs[::3]:
        assert np.array_equal(pm.match_pairs([p], CFG, symmetric=True)[p], sym[p]), p


def test_thousand_pair_general_float_submission_matches_cv2():
    """Arbitrary float32 values (cv2-order SIMT kernel), smaller images, 1030 pairs in one call and pair by pair."""
    rng = np.random.RandomState(7)
    sizes = [1, 2, 31, 63, 64, 65, 127, 128, 129] + rng.randint(20, 160, 31).tolist()
    images = _float_images(sizes, 8)
    pairs = [(a, b) for a in range(len(sizes)) for b in range(len(sizes)) if a != b]
    pairs = [pairs[i] for i in rng.permutation(len(pairs))[:1030]]
    ref_ow, ref_sym = _reference(images, pairs)
    pm = matching.PairMatcher()
    pm.add_many(list(enumerate(images)))
    one, sym = _check_batch(pm, images, pairs, ref_ow, ref_sym, 1)
    assert sum(len(v) for v in sym.values()) > 3000
    for p in pairs[::5]:
        assert np.array_equal(pm.match_pairs([p], CFG, symmetric=True)[p], sym[p]), p


# ---------------------------------------------------------------------------------------------------------------
# Images without rows
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["l2", "uint8_stored", "hamming"])
def test_empty_images_inside_a_batch_stay_on_the_tensor_cores(kind):
    """Images with 0 rows at the start, the middle and the end of a 300-pair submission: their pairs come back
    empty, every other pair equals cv2, and the submission stays on the tensor-core kernel -- an image without
    features must not move thousands of pairs to the SIMT kernel.  Jobs without query or train tiles then sit in
    the persistent kernel's job table."""
    rng = np.random.RandomState(9)
    sizes = EDGE_SIZES + rng.randint(40, 400, 24).tolist()
    images = _hamming_images(sizes, 10) if kind == "hamming" else _l2_images(sizes, 10)
    empty_ids = [len(images), len(images) + 1, len(images) + 2]
    for _ in empty_ids:
        images.append(images[0][:0].copy())
    full = list(range(len(sizes)))
    pairs = _pair_list(sizes + [2, 2, 2], 11, 300)
    pairs = [p for p in pairs if p[0] not in empty_ids and p[1] not in empty_ids]
    e0, e1, e2 = empty_ids
    pairs = [(e0, full[3]), (full[4], e1)] + pairs[:150] + [(e1, e2), (e2, full[7]), (full[8], e0), (e0, e0)] + \
        pairs[150:] + [(full[9], e2), (e2, e1)]
    ref_ow, ref_sym = _reference(images, pairs)
    pm = matching.PairMatcher()
    if kind == "uint8_stored":
        pm.add_many([(i, d.astype(np.uint8)) for i, d in enumerate(images)], uint8_is_l2=True)
    else:
        pm.add_many(list(enumerate(images)))
    one, sym = _check_batch(pm, images, pairs, ref_ow, ref_sym, 3 if kind == "hamming" else 2)
    for p in pairs:
        if p[0] in empty_ids or p[1] in empty_ids:
            assert len(one[p]) == 0 and len(sym[p]) == 0
    assert sum(len(v) for v in sym.values()) > 1000


# ---------------------------------------------------------------------------------------------------------------
# The tensor-core kernel's norm bound
# ---------------------------------------------------------------------------------------------------------------
def _four_squares(r):
    """r = x^2 + y^2 + z^2 + w^2 with every term <= 255^2 (Lagrange; searched from the largest term down)."""
    for x in range(min(255, math.isqrt(r)), -1, -1):
        r1 = r - x * x
        if r1 > 3 * 65025:
            break
        for y in range(min(x, math.isqrt(r1)), -1, -1):
            r2 = r1 - y * y
            if r2 > 2 * 65025:
                break
            for z in range(min(y, math.isqrt(r2)), -1, -1):
                r3 = r2 - z * z
                if r3 > 65025:
                    break
                w = math.isqrt(r3)
                if w * w == r3:
                    return [x, y, z, w]
    raise AssertionError(r)


def _with_norm(norm, rng, n=64, scale=None):
    """n integers in [0, 255] whose squares sum to exactly `norm`: n - 4 random values sized to leave about 1.2e5,
    which four more values take up exactly."""
    v = rng.uniform(0.3, 1.0, n - 4) if scale is None else np.asarray(scale, np.float64).copy()
    v *= math.sqrt((norm - 1.2e5) / float(v @ v))
    v = np.clip(np.round(v), 0, 255)
    out = np.concatenate([v, _four_squares(int(norm - v @ v))])
    assert int(out @ out) == norm
    return out


def _near_bound_sets(total, seed):
    """Query images with |a|^2 <= A and train images with |b|^2 <= B, A + B = total, so that the host's admission
    test 2 (max|a|^2 + max|b|^2) < 2^22 sits at 2 total / 2^22.  Queries live in dims 0..63.  A train is
    c + s: c in dims 64..127 carries its norm, s in dims 0..63 is one vector shared by the image (zero for half of
    the images: d^2 = |a|^2 + |b|^2, the largest d^2 the bound allows; a query-like vector for the other half:
    large partial sums of -2 a.b in the accumulator).  Every train image has norms X, X + 1 (the two best of
    every query: their d^2 differ by exactly 1), larger ones up to B, and a tie."""
    rng = np.random.RandomState(seed)
    A = total // 2
    B = total - A
    direction = rng.uniform(0.3, 1.0, 60)
    queries = []
    for k in range(4):
        q = np.zeros((200, 128))
        for i in range(200):
            q[i, :64] = _with_norm(A - (0 if i == 0 else int(rng.randint(0, 3000))), rng,
                                   scale=direction + rng.uniform(0, 0.3, 60))
        queries.append(q.astype(np.float32))
    trains = []
    for k in range(6):
        s = np.zeros(64)
        if k % 2:
            s[:60] = np.round(direction * (60.0, 110.0, 160.0)[k // 2])
        s2 = int(s @ s)
        X = B - int(rng.randint(2000, 4000))
        norms = [X, X + 1, B, B] + (X + 2 + rng.randint(0, B - X - 1, 156)).tolist()
        t = np.zeros((160, 128))
        for j, nb in enumerate(norms):
            t[j, :64] = s
            t[j, 64:] = _with_norm(nb - s2, rng)
        trains.append(t[rng.permutation(160)].astype(np.float32))
    return queries, trains


def _exact_d2(a, b):
    a = a.astype(np.int64)
    b = b.astype(np.int64)
    return (a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2 * a @ b.T


@pytest.mark.parametrize("side", ["below", "above"])
def test_distances_next_to_the_tensor_core_norm_bound(side):
    """The tensor-core kernel ranks in d^2 and needs float32 sqrt to keep distinct integers apart; the host admits
    it when 2 (max|a|^2 + max|b|^2) < 2^22.  Below the bound (ratio in [0.97, 1)) the kernel must be the
    tensor-core one; the two best d^2 of every query are 1 apart (computed exactly in int64), their float32 square
    roots differ by a few ulps, and the lists must equal cv2's at ratios that keep (1.0, 1.001) or drop (0.8,
    0.999) every such query.  Just above the bound the exact SIMT kernel must run and give the same lists.
    Descriptor values are non-negative, so d^2 <= |a|^2 + |b|^2 < 2^21 whenever the bound admits a pair."""
    ratio = 0.985 if side == "below" else 1.004
    total = int(ratio * 2 ** 21)
    queries, trains = _near_bound_sets(total, 12 if side == "below" else 13)
    pm = matching.PairMatcher()
    names = {}
    for i, q in enumerate(queries):
        names["q%d" % i] = q
    for j, t in enumerate(trains):
        names["t%d" % j] = t
    pm.add_many(list(names.items()))
    pairs = [("q%d" % i, "t%d" % j) for i in range(len(queries)) for j in range(len(trains))]
    largest, near_ties = 0, 0
    for a, b in pairs:
        na = int((names[a].astype(np.int64) ** 2).sum(1).max())
        nb = int((names[b].astype(np.int64) ** 2).sum(1).max())
        bound = 2.0 * (na + nb) / 2 ** 22
        assert (0.97 <= bound < 1.0) if side == "below" else (1.0 <= bound < 1.03), (a, b, bound)
        d2 = _exact_d2(names[a], names[b])
        two = np.sort(d2, axis=1)[:, :2]
        assert (two[:, 1] - two[:, 0] == 1).all()
        assert (np.sqrt(two[:, 0].astype(np.float32)) != np.sqrt(two[:, 1].astype(np.float32))).all()
        near_ties += len(two)
        largest = max(largest, int(d2.max()))
    if side == "below":
        assert largest >= 0.97 * 2 ** 21
    print("largest d^2 %d = %.4f * 2^21 over %d queries whose two best d^2 differ by 1" % (
        largest, largest / 2 ** 21, near_ties))
    for r in (0.8, 0.999, 1.0, 1.001):
        cfg = {"lowes_ratio": r}
        one = pm.match_pairs(pairs, cfg, symmetric=False)
        assert pm.last_kernel() == (2 if side == "below" else 1)
        sym = pm.match_pairs(pairs, cfg, symmetric=True)
        n = 0
        for a, b in pairs:
            want = mo.match_brute_force(names[a], names[b], cfg)
            assert _rows(one[(a, b)]) == want, (a, b, r)
            assert _pairset(sym[(a, b)]) == _pairset(mo.match_brute_force_symmetric(names[a], names[b], cfg)), (a, b, r)
            n += len(want)
        assert (n == 0) if r < 1.0 else (n == sum(len(names[a]) for a, _ in pairs))


# ---------------------------------------------------------------------------------------------------------------
# Guided matching: the epipolar masks, bit for bit
# ---------------------------------------------------------------------------------------------------------------
THRESHOLDS = [0.0, 1e-6, 0.006, 0.1, 1.0, math.pi / 2 - 1e-9, 2.0, -0.01]


def _sphere(n, seed):
    b = np.random.RandomState(seed).normal(size=(n, 3))
    return (b / np.linalg.norm(b, axis=1, keepdims=True)).astype(np.float32)


def _rotation(seed):
    q, r = np.linalg.qr(np.random.RandomState(seed).normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def _check_masks(pm, i, b1, b2, R, t, thr):
    """The pair's device masks against the fp64 reference.  Elements whose fp64 angle is within 1e-12 of the
    threshold, or whose symmetric_epi is within 1e-12 of 1 (acos turns NaN there), depend on the summation order
    and are excluded -- except an exact 0, which only zero epipolar vectors produce (t = 0, a bearing along t).
    Returns (elements, guard-band elements, excluded elements)."""
    F, T = pm.last_epipolar_masks(i)
    assert F.shape == (len(b1), len(b2)) and T.shape == (len(b2), len(b1))
    assert np.array_equal(T, F.T)
    sym = mo.epipolar_sym(b1, b2, R, t)
    with np.errstate(invalid="ignore"):
        ang = np.pi / 2 - np.arccos(sym)
        want = ang < thr
    excl = ((np.abs(ang - thr) < 1e-12) & (sym != 0.0)) | (np.abs(sym - 1.0) < 1e-12)
    bad = np.argwhere((F != want) & ~excl)
    assert len(bad) == 0, (thr, len(bad), [(int(x), int(y), float(sym[x, y])) for x, y in bad[:5]])
    band = np.abs(sym - math.sin(min(max(thr, -math.pi / 2), math.pi / 2))) < 2e-6
    return F.size, int(band.sum()), int(excl.sum())


def _guided_case(seed=20):
    """One guided submission: the guided_scene cameras (HAHOG-like scene, real epipolar geometry), bearings uniform
    on the sphere for images of 1 ... 300 features (word boundaries, 256 x 256 CTA tiles), a pair with t = 0 and
    a pair whose bearings include +-t^ exactly."""
    descs, bears, Rs, Os = syn.guided_scene(4, 700, seed=seed)
    images = {("s", i): (descs[i], bears[i]) for i in range(4)}
    pairs = [(("s", a), ("s", b)) for a, b in [(0, 1), (1, 2), (0, 3), (3, 2)]]
    poses = [syn.relative_pose(Rs[a], Os[a], Rs[b], Os[b]) for a, b in [(0, 1), (1, 2), (0, 3), (3, 2)]]
    sizes = [1, 31, 32, 33, 255, 256, 257, 300]
    pool = syn.hahog_like_descriptors(400, seed)
    rng = np.random.RandomState(seed)
    for k, n in enumerate(sizes):
        d = np.clip(pool[rng.choice(400, n)] + rng.randint(-3, 4, (n, 128)), 0, 255).astype(np.float32)
        images[("r", k)] = (d, _sphere(n, seed + 100 + k))
    for k, (a, b) in enumerate([(0, 1), (1, 0), (2, 3), (3, 2), (4, 5), (5, 6), (6, 4), (7, 7), (7, 0), (5, 7)]):
        pairs.append((("r", a), ("r", b)))
        poses.append((_rotation(seed + k), np.random.RandomState(seed + k).normal(size=3) * 2.0))
    # t = 0 and bearings exactly along +-t^ (t^ = e_z, so the cross products are exactly 0)
    pairs.append((("r", 6), ("r", 7)))
    poses.append((_rotation(seed + 50), np.zeros(3)))
    d8, b8 = images[("r", 7)]
    b8 = b8.copy()
    b8[[0, 17, 299]] = [[0, 0, 1], [0, 0, -1], [0, 0, 1]]
    images[("p", 0)] = (d8, b8)
    Rz = np.array([[0.0, 1.0, 0.0], [0.0, 0.0, 1.0], [1.0, 0.0, 0.0]])   # a permutation: R b2 is exact
    b6 = images[("r", 6)][1].copy()
    b6[[5, 100]] = [[1, 0, 0], [-1, 0, 0]]                              # R b2 = +-e_z
    images[("p", 1)] = (images[("r", 6)][0], b6)
    pairs.append((("p", 0), ("p", 1)))
    poses.append((Rz, np.array([0.0, 0.0, 3.5])))
    return images, pairs, poses


def _guided_matcher(images, kernel=0):
    pm = matching.PairMatcher(kernel=kernel)
    for k, (d, b) in images.items():
        pm.add(k, d)
        pm.set_bearings(k, b)
    return pm


@pytest.mark.parametrize("thr", THRESHOLDS)
def test_epipolar_masks_bit_for_bit(thr):
    """Every mask bit the device builds, both layouts, against the reference's fp64 angle test, for thresholds
    from below 0 to past pi/2 (where the reference keeps every element with a finite angle)."""
    images, pairs, poses = _guided_case()
    pm = _guided_matcher(images)
    pm.match_pairs_guided(pairs, poses, thr, CFG)
    band = excl = total = 0
    for i, ((a, b), (R, t)) in enumerate(zip(pairs, poses)):
        n, nb, ne = _check_masks(pm, i, images[a][1], images[b][1], R, t, thr)
        total += n
        band += nb
        excl += ne
    print("threshold %.9g: %d elements, %d in the guard band, %d excluded" % (thr, total, band, excl))
    assert excl <= 2


def test_guided_matching_past_half_pi_keeps_every_finite_angle():
    """threshold 2.0 > pi/2: the reference's pi/2 - acos(sym) < 2.0 holds for every sym <= 1, so guided matching
    of bearings spread over the sphere is (nearly) unguided; a test in sine space against sin(2.0) < 1 drops
    elements and changes the matches."""
    d1, d2 = _l2_images([300, 300], 30)
    b1, b2 = _sphere(300, 31), _sphere(300, 32)
    R, t = _rotation(33), np.array([0.4, -1.0, 0.3])
    pm = _guided_matcher({"a": (d1, b1), "b": (d2, b2)})
    got = pm.match_pairs_guided([("a", "b")], [(R, t)], 2.0, CFG)[("a", "b")]
    mask = mo.epipolar_mask(b1, b2, R, t, 2.0)
    assert mask.mean() > 0.999
    ref = _pairset(mo.match_brute_force_symmetric(d1, d2, CFG, mask))
    assert len(ref) > 20
    assert _pairset(got) == ref
    _check_masks(pm, 0, b1, b2, R, t, 2.0)


def test_guided_matching_with_zero_translation_is_unguided():
    """t = 0 (a pure rotation): Eigen's normalized() leaves the zero vector unchanged, so the reference's angle is
    0 everywhere, the mask all true and guided matching equals unguided symmetric matching -- not zero matches."""
    d1, d2 = _l2_images([400, 500], 34)
    b1, b2 = _sphere(400, 35), _sphere(500, 36)
    R = _rotation(37)
    pm = _guided_matcher({"a": (d1, b1), "b": (d2, b2)})
    got = pm.match_pairs_guided([("a", "b")], [(R, np.zeros(3))], 0.006, CFG)[("a", "b")]
    ref = _pairset(mo.match_brute_force_symmetric(d1, d2, CFG))
    assert len(ref) > 20
    assert _pairset(got) == ref
    F, T = pm.last_epipolar_masks(0)
    assert F.all() and T.all()
    assert _pairset(pm.match_pairs([("a", "b")], CFG)[("a", "b")]) == ref


def _offset_scene(n1, thr, seed):
    """Bearings whose symmetric_epi sits at signed offsets from sin(threshold): b1_i and R b2_j perpendicular to t,
    at in-plane angles whose difference has the prescribed sine (then both terms of symmetric_epi equal it), the
    whole configuration turned by a random rotation.  Returns (b1, b2, R, t)."""
    rng = np.random.RandomState(seed)
    offsets = [1e-3, 1e-5, 3e-6, 2e-6, 1e-6, 1e-7, 1e-9]
    s0 = math.sin(thr)
    th1 = rng.uniform(0, 2 * np.pi, n1)
    th2 = []
    for th in th1:
        for off in offsets:
            for sign in (1, -1):
                s = s0 + sign * off
                if 0.0 <= s <= 1.0:
                    th2.append(th + math.asin(s) * (1 if rng.rand() < 0.5 else -1) + (np.pi if rng.rand() < 0.5 else 0))
    th2 = np.array(th2)
    Q = _rotation(seed + 1)
    b1 = np.stack([np.zeros(n1), np.cos(th1), np.sin(th1)], 1) @ Q.T
    b2w = np.stack([np.zeros(len(th2)), np.cos(th2), np.sin(th2)], 1) @ Q.T
    R = _rotation(seed + 2)
    t = Q @ np.array([2.5, 0.0, 0.0])
    return b1.astype(np.float32), (b2w @ R).astype(np.float32), R, t


@pytest.mark.parametrize("thr", [0.006, 0.1, 1.0])
def test_epipolar_guard_band_elements_match_the_fp64_reference(thr):
    """Elements placed at +-{1e-3, 1e-5, 3e-6, 2e-6, 1e-6, 1e-7, 1e-9} from the threshold in sine space: at least
    1000 of them are inside the float32 test's +-2e-6 guard band, so the kernel's fp64 branch decides them, and
    every bit equals the reference's.  None is within 1e-12 of the threshold."""
    b1, b2, R, t = _offset_scene(200, thr, 40)
    descs = _l2_images([len(b1), len(b2)], 41)
    pm = _guided_matcher({"a": (descs[0], b1), "b": (descs[1], b2)})
    pm.match_pairs_guided([("a", "b")], [(R, t)], thr, CFG)
    n, band, excl = _check_masks(pm, 0, b1, b2, R, t, thr)
    print("threshold %g: %d elements, %d in the guard band, %d excluded" % (thr, n, band, excl))
    assert band >= 1000
    assert excl == 0


def test_guided_matching_at_scale_and_in_budget_rounds():
    """105 pairs of 2000 features in one submission (no train split), against cv2 under the reference's mask; then
    the same pairs in rounds of different sizes (mask_budget_bytes), which must give the same lists, and the masks
    of the last round read back bit for bit."""
    n_img, n_desc, thr = 15, 2000, 0.006
    descs, bears, Rs, Os = syn.guided_scene(n_img, n_desc, seed=50)
    pm = matching.PairMatcher()
    for i in range(n_img):
        pm.add(i, descs[i])
        pm.set_bearings(i, bears[i])
    pairs = [(a, b) for a in range(n_img) for b in range(a + 1, n_img)]
    poses = [syn.relative_pose(Rs[a], Os[a], Rs[b], Os[b]) for a, b in pairs]
    assert len(pairs) >= 100
    got = pm.match_pairs_guided(pairs, poses, thr, CFG)
    assert pm.last_kernel() == 2
    total = 0
    for (a, b), (R, t) in zip(pairs, poses):
        mask = mo.epipolar_mask(bears[a], bears[b], R, t, thr)
        ref = _pairset(mo.match_brute_force_symmetric(descs[a], descs[b], CFG, mask))
        assert _pairset(got[(a, b)]) == ref, (a, b)
        total += len(ref)
    assert total > 5000
    per_pair = 2 * n_desc * ((n_desc + 31) // 32) * 4
    budget = 45 * per_pair                     # rounds of 45, 45 and 15 pairs
    rounds = pm.match_pairs_guided(pairs, poses, thr, CFG, mask_budget_bytes=budget)
    for p in pairs:
        assert np.array_equal(rounds[p], got[p]), p
    last = len(pairs) - 90
    for i, k in enumerate(range(90, len(pairs))):
        a, b = pairs[k]
        _check_masks(pm, i, bears[a], bears[b], poses[k][0], poses[k][1], thr)
    with pytest.raises(ValueError):
        pm.last_epipolar_masks(last)
    pm.match_pairs(pairs[:3], CFG)
    with pytest.raises(ValueError):
        pm.last_epipolar_masks(0)


def test_reference_known_answer_two_cams_many_points_on_the_engine():
    """triangulation_test.cc:327-341 (TwoCamsManyPointsFixture): the epipolar angle of a point with itself is below
    1e-6 and above it for the other point, so at threshold 1e-6 the device's mask is the identity."""
    from test_epipolar_oracle import two_cams_many_points

    b1, b2, R, t = two_cams_many_points()
    d = syn.hahog_like_descriptors(2, 60)
    pm = _guided_matcher({"a": (d, b1), "b": (d, b2)})
    pm.match_pairs_guided([("a", "b")], [(R, t)], 1e-6, CFG)
    F, T = pm.last_epipolar_masks(0)
    assert np.array_equal(F, np.eye(2, dtype=bool)) and np.array_equal(T, np.eye(2, dtype=bool))
