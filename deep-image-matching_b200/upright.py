"""``upright`` on the host: the reference's rotation search (ImageMatcher.run, image_matching.py:496 rotates, :703 rotates back;
find_matches_per_rotation, :69-118) restated with every detail this project fixes itself.  It is the oracle of the device path
(``sharded.ImageSetMatcher(upright=...)``) and serves callers whose images are on disk.

Each image gets the rotation in ``ROTATIONS`` (degrees clockwise, the ``cv2.rotate`` codes of ``CV2_CODES``) that gives the most
SuperPoint + LightGlue matches against an image already oriented; features are extracted from the rotated images and matched, and
the keypoints are rotated back to the original image.  SuperPoint is not rotation invariant, so this is what sets with mixed camera
orientations need.

Stated here, not pinned to the reference (whose exact choices are unverified):
  * the schedule (``upright_schedule``): pairs visited in list order; a pair with both images decided is skipped, with neither
    decided its first image becomes a root at 0 and the second is searched against it, with one decided the other is searched against
    it; images in no pair stay at 0.  Whether an image is decided never depends on match counts, so the schedule is known before any
    matching, as a forest of *waves*: wave d holds the decisions whose reference was decided in wave d - 1 (wave 0: against roots);
  * the search image: gray float32, resized with INTER_AREA to longest side ``resize_max`` (``sharded._lowres_size``, enlarging too),
    then turned by ``cv2.rotate`` (resize first, then rotate);
  * the search of target t against reference a at rotation r_a: c_k = number of LightGlue matches between SuperPoint(rot(low_a, r_a))
    and SuperPoint(rot(low_t, k)), k = 0..3, and r_t = ROTATIONS[argmax c] (the first maximum wins ties); the networks are the
    plugins' defaults (``SP_UPRIGHT_CONF`` with the keypoint cap ``max_keypoints``, ``LG_UPRIGHT_CONF`` on features without
    image_size, so keypoints are normalised by their own extent), features stay float32;
  * the back-rotation (``rotate_back_keypoints``): the exact inverse of cv2.rotate on pixel indices of the original H x W image, so an
    integer keypoint lands on the pixel it was detected on;
  * F (``rotate_back_F``): A1^T F A0 with A the original -> rotated pixel map, and ``image_size`` the original image's.
"""
from __future__ import annotations

import numpy as np

ROTATIONS = (0, 90, 180, 270)
# SuperPointExtractor._default_conf without the cap (max_keypoints -1 has no device buffer; the caller's cap goes in)
SP_UPRIGHT_CONF = {"nms_radius": 4, "keypoint_threshold": 0.005, "remove_borders": 4}
# LightGlueMatcher._default_conf with LightGlue's own defaults for the keys it leaves out
LG_UPRIGHT_CONF = {"n_layers": 9, "depth_confidence": 0.95, "width_confidence": 0.99, "filter_threshold": 0.1, "prune_min_kpts": 1536}


def cv2_code(rotation: int):
    """The cv2.rotate code of `rotation` (None for 0)."""
    import cv2
    return dict(zip(ROTATIONS, (None, cv2.ROTATE_90_CLOCKWISE, cv2.ROTATE_180, cv2.ROTATE_90_COUNTERCLOCKWISE)))[rotation]


def rotate_image(img: np.ndarray, rotation: int) -> np.ndarray:
    """cv2.rotate of `img` by `rotation` degrees clockwise (a copy for 0)."""
    import cv2
    code = cv2_code(rotation)
    return np.ascontiguousarray(img) if code is None else cv2.rotate(np.ascontiguousarray(img), code)


def rotated_size(height: int, width: int, rotation: int):
    """(H, W) of an H x W image turned by `rotation`."""
    return (width, height) if rotation in (90, 270) else (height, width)


def upright_schedule(pairs, n_images: int) -> list:
    """The search forest of `pairs` (module docstring): a list of waves, wave d the (target, reference) decisions whose reference was
    decided in wave d - 1 (roots for wave 0), each wave in decision order.  Pure: no GPU, no match counts."""
    depth = [None] * n_images  # 0 for a root, d + 1 for a target of wave d
    waves = []
    for i, j in pairs:
        i, j = int(i), int(j)
        if depth[i] is not None and depth[j] is not None:
            continue
        if depth[i] is None and depth[j] is None:
            depth[i] = 0
        t, a = (j, i) if depth[j] is None else (i, j)
        depth[t] = depth[a] + 1
        while len(waves) < depth[t]:
            waves.append([])
        waves[depth[t] - 1].append((t, a))
    return waves


def search_image(gray: np.ndarray, resize_max: int) -> np.ndarray:
    """The unrotated search image: gray float32, INTER_AREA to longest side `resize_max` (pairs_generator.read_lowres' rule)."""
    import cv2

    from .sharded import _lowres_size
    H, W = gray.shape[:2]
    _, h, w = _lowres_size(H, W, resize_max)
    return cv2.resize(np.asarray(gray, np.float32), (w, h), interpolation=cv2.INTER_AREA)


def choose(counts) -> int:
    """The rotation of the largest count, the first one on ties."""
    return ROTATIONS[int(np.argmax(np.asarray(counts)))]


def search_plugins(max_keypoints: int = 2048, fix_sampling: bool = False, lightglue_weights=None, superpoint_weights=None, device: int = 0):
    """The search's SuperPointExtractor (``SP_UPRIGHT_CONF``, cap `max_keypoints`) and LightGlueMatcher (``LG_UPRIGHT_CONF``)."""
    from .config import Config
    from .extractors.superpoint import SuperPointExtractor
    from .matchers.lightglue import LightGlueMatcher
    ext = SuperPointExtractor(Config(general={"device": device}, extractor={
        **SP_UPRIGHT_CONF, "max_keypoints": int(max_keypoints), "fix_sampling": bool(fix_sampling), "weights_dict": superpoint_weights}))
    return ext, LightGlueMatcher(Config(general={"device": device}, matcher={**LG_UPRIGHT_CONF, "weights_dict": lightglue_weights}))


def upright_rotations(images, pairs, resize_max: int, max_keypoints: int = 2048, fix_sampling: bool = False, lightglue_weights=None,
                      superpoint_weights=None, device: int = 0, plugins=None):
    """The host flow of the search (find_matches_per_rotation): for every decision of ``upright_schedule``, one plugin ``_extract`` of
    the reference at its rotation and of the target at each of the four, and one ``_match_pairs`` per rotation.  `images`: gray float32
    arrays at full size.  `plugins`: the (extractor, matcher) of ``search_plugins`` to reuse across calls (built here otherwise).
    Returns (rotations, {(target, reference): [c_0, c_90, c_180, c_270]})."""
    ext, lg = plugins or search_plugins(max_keypoints, fix_sampling, lightglue_weights, superpoint_weights, device)
    rotations = [0] * len(images)
    counts = {}
    low = {}
    for wave in upright_schedule(pairs, len(images)):
        for t, a in wave:
            for k in (t, a):
                if k not in low:
                    low[k] = search_image(images[k], resize_max)
            ref = ext._extract(rotate_image(low[a], rotations[a]))
            c = [len(lg._match_pairs(ref, ext._extract(rotate_image(low[t], r)))) for r in ROTATIONS]
            counts[(t, a)] = c
            rotations[t] = choose(c)
    return rotations, counts


def rotate_back_keypoints(kpts, rotation: int, height: int, width: int) -> np.ndarray:
    """Keypoints (N, 2) x, y of the image turned by `rotation` -> pixel indices of the original `height` x `width` image, in float32
    (each difference rounded once): 90 (y', H - 1 - x'), 180 (W - 1 - x', H - 1 - y'), 270 (W - 1 - y', x')."""
    k = np.asarray(kpts, np.float32).reshape(-1, 2)
    x, y = k[:, 0], k[:, 1]
    h1, w1 = np.float32(height - 1), np.float32(width - 1)
    out = {0: (x, y), 90: (y, h1 - x), 180: (w1 - x, h1 - y), 270: (w1 - y, x)}[rotation]
    return np.stack(out, axis=1).astype(np.float32)


def rotation_matrix(rotation: int, height: int, width: int) -> np.ndarray:
    """A (3, 3) float64: homogeneous pixel indices of the original `height` x `width` image -> those of the image turned by `rotation`."""
    h1, w1 = height - 1, width - 1
    return np.array({0: [[1, 0, 0], [0, 1, 0]], 90: [[0, -1, h1], [1, 0, 0]], 180: [[-1, 0, w1], [0, -1, h1]],
                     270: [[0, 1, 0], [-1, 0, w1]]}[rotation] + [[0, 0, 1]], np.float64)


def rotate_back_F(F, r0: int, size0, r1: int, size1):
    """F (3, 3) of a pair matched in the rotated frames (x1'^T F x0' = 0) -> F in original pixels, A1^T F A0 (A: ``rotation_matrix`` of
    each image's original (H, W)), computed in float64 and returned as float32 without rescaling (A holds 0, +-1 and integer
    translations).  None stays None."""
    if F is None:
        return None
    A0, A1 = rotation_matrix(r0, *size0), rotation_matrix(r1, *size1)
    return (A1.T @ np.asarray(F, np.float64) @ A0).astype(np.float32)
