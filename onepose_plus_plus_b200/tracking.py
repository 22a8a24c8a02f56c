"""The demo's tracking step on the device — drop-ins for the reference's bbox crop
(src/local_feature_object_detector/local_feature_2D_detector.py:133-159 ``crop_img_by_bbox``,
:200-226 ``previous_pose_detect``; src/utils/data_utils.py:22-52 ``get_affine_transform``, :239-255
``get_image_crop_resize``, :258-280 ``get_K_crop_resize``; src/utils/vis_utils.py:10-37 ``reproj``)
and a batched crop -> matcher -> pose loop over the frames after the first (demo.py:105-132).

The reference reads every frame from disk a second time, runs two full-frame ``cv2.warpAffine``
calls (the box at native scale, then a resize to 512 x 512), converts the crop to float and uploads
it.  Here the crop is one kernel (``opp_crop_resize_u8``) that reads the uint8 frame on the device
and writes the uint8 crop the matcher takes directly, bit for bit what the two cv2 calls produce:

* the geometry stays on the host in fp64 — the box from the previous pose (``reproj`` and the
  int32 truncation), the two affine maps from ``cv2.getAffineTransform`` with the reference's point
  construction, K_crop composed twice — and the kernel gets the inverse of the second map exactly as
  ``cv2.warpAffine`` forms it, so its fixed-point coordinates are cv2's integers;
* the first warp maps the box to a w x h image at scale 1, an integer shift (checked on the
  fixed-point terms for every box), so the kernel runs the second warp alone over a virtual source:
  the frame shifted by the box origin, zero outside the frame and outside the box.

``PoseTracker`` runs B independent sequences (several cameras, several objects' sequences with one
resident bank) per call; with ``model.enable_cuda_graphs()`` the crop is captured in the same CUDA
graph as the matcher's forward.
"""
import numpy as np
import torch

from . import _lib, pnp

__all__ = ["reproj", "bbox_from_pose", "get_affine_transform", "get_K_crop_resize", "crop_K",
           "crop_params", "crop_resize_batched", "get_image_crop_resize", "crop_img_by_bbox",
           "previous_pose_detect", "PoseTracker"]

# opp_crop_params (include/opp_b200.h): the inverse map, then the virtual source box
CROP_PARAMS = np.dtype([("m", "<f8", (6,)), ("x0", "<i4"), ("y0", "<i4"), ("w", "<i4"), ("h", "<i4")])
assert CROP_PARAMS.itemsize == 64
COORD_LIMIT = 1 << 20    # |box coordinate| bound of the kernel's int32 fixed-point sums
SIDE_LIMIT = 32767       # cv2.warpAffine: every image side < SHRT_MAX
MIN_INLIERS = 20         # demo.py:108: fewer inliers -> the previous pose is not trusted


def _cv2():
    import cv2
    return cv2


# ------------------------------------------------------------------------------------------------
# host geometry (fp64 numpy, the reference's arithmetic)
# ------------------------------------------------------------------------------------------------
def reproj(K, pose, pts_3d):
    """vis_utils.reproj: pixel coordinates [n, 2] of pts_3d [n, 3] under K [3, 3|4] and pose [3|4, 4]."""
    K, pose = np.asarray(K), np.asarray(pose)
    if K.shape not in ((3, 3), (3, 4)) or pose.shape not in ((3, 4), (4, 4)):
        raise ValueError(f"K must be [3, 3] or [3, 4] and pose [3, 4] or [4, 4], got {K.shape}, {pose.shape}")
    P = np.concatenate([K, np.zeros((3, 1))], axis=1) if K.shape == (3, 3) else K
    T = np.concatenate([pose, np.array([[0, 0, 0, 1]])], axis=0) if pose.shape == (3, 4) else pose
    pts = np.asarray(pts_3d).reshape(-1, 3)
    X = np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1).T
    uvw = P @ T @ X
    return (uvw[:] / uvw[2:])[:2, :].T


def bbox_from_pose(K, pose, bbox3d):
    """previous_pose_detect's box: the 2D extent of the projected 3D box corners, truncated to
    int32 [x0, y0, x1, y1]."""
    uv = reproj(K, pose, bbox3d)
    lo, hi = np.min(uv, axis=0), np.max(uv, axis=0)
    return np.array([lo[0], lo[1], hi[0], hi[1]]).astype(np.int32)


def _third_point(a, b):
    d = a - b
    return b + np.array([-d[1], d[0]], dtype=np.float32)


def get_affine_transform(center, scale, rot, output_size, shift=np.array([0, 0], dtype=np.float32), inv=0):
    """data_utils.get_affine_transform: the 2x3 map taking the box (centre, width scale[0]) rotated by
    `rot` degrees to the output_size = (w, h) image, from three float32 point pairs (the centre, the
    top-middle point, and its 90 degree rotation about the centre) through cv2.getAffineTransform."""
    if not isinstance(scale, (np.ndarray, list)):
        scale = np.array([scale, scale], dtype=np.float32)
    off = scale * shift
    half_w = scale[0] * -0.5
    a = np.pi * rot / 180
    sn, cs = np.sin(a), np.cos(a)
    up_src = [0 * cs - half_w * sn, 0 * sn + half_w * cs]
    out_w, out_h = output_size[0], output_size[1]
    src = np.zeros((3, 2), dtype=np.float32)
    dst = np.zeros((3, 2), dtype=np.float32)
    src[0] = center + off
    src[1] = center + up_src + off
    dst[0] = [out_w * 0.5, out_h * 0.5]
    dst[1] = np.array([out_w * 0.5, out_h * 0.5], np.float32) + np.array([0, out_w * -0.5], np.float32)
    src[2] = _third_point(src[0], src[1])
    dst[2] = _third_point(dst[0], dst[1])
    cv2 = _cv2()
    return cv2.getAffineTransform(dst, src) if inv else cv2.getAffineTransform(src, dst)


def _box_map(box, resize_shape):
    """get_affine_transform of data_utils.get_image_crop_resize / get_K_crop_resize."""
    center = np.array([(box[0] + box[2]) / 2.0, (box[1] + box[3]) / 2.0])
    scale = np.array([box[2] - box[0], box[3] - box[1]])
    resize_h, resize_w = resize_shape
    return get_affine_transform(center, scale, 0, [resize_w, resize_h])


def get_K_crop_resize(box, K_orig, resize_shape):
    """data_utils.get_K_crop_resize: (K_crop [3, 3], K_crop_homo [3, 4]) of the crop of `box`
    resized to resize_shape = (h, w)."""
    T = np.concatenate([_box_map(box, resize_shape), np.array([[0, 0, 1]])], axis=0)
    K_orig = np.asarray(K_orig)
    if K_orig.shape == (3, 3):
        Kh = np.concatenate([K_orig, np.zeros((3, 1))], axis=-1)
    elif K_orig.shape == (3, 4):
        Kh = K_orig.copy()
    else:
        raise ValueError(f"K_orig must be [3, 3] or [3, 4], got {K_orig.shape}")
    K_crop_homo = T @ Kh
    return K_crop_homo[:3, :3], K_crop_homo


def crop_K(bbox, K, crop_size=512):
    """crop_img_by_bbox's K_crop: get_K_crop_resize for the box at native scale, then for the
    resize of [0, 0, w, h] to crop_size x crop_size."""
    x0, y0, x1, y1 = bbox[0], bbox[1], bbox[2], bbox[3]
    K_crop, _ = get_K_crop_resize(bbox, K, np.array([y1 - y0, x1 - x0]))
    K_crop, _ = get_K_crop_resize(np.array([0, 0, x1 - x0, y1 - y0]), K_crop, np.array([crop_size, crop_size]))
    return K_crop


def _invert_affine(M):
    """The inverse cv2.warpAffine forms from M (imgwarp.cpp; also cv2.invertAffineTransform)."""
    M = np.asarray(M, dtype=np.float64).reshape(-1).copy()
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[4] * D, M[0] * D
    M[0], M[4] = A11, A22
    M[1] *= -D
    M[3] *= -D
    b1 = -M[0] * M[2] - M[1] * M[5]
    b2 = -M[3] * M[2] - M[4] * M[5]
    M[2], M[5] = b1, b2
    return M


def _fixed_point_terms(m, out_w, out_h):
    """cv2's per-column (adelta, bdelta) and per-row (X0, Y0) fixed-point terms of inverse map m."""
    xs = np.arange(out_w, dtype=np.float64)
    ys = np.arange(out_h, dtype=np.float64)
    return (np.rint(m[0] * xs * 1024).astype(np.int64), np.rint(m[3] * xs * 1024).astype(np.int64),
            np.rint((m[1] * ys + m[2]) * 1024).astype(np.int64) + 16,
            np.rint((m[4] * ys + m[5]) * 1024).astype(np.int64) + 16)


def _is_integer_shift(m, w, h, x0, y0):
    """True when cv2's fixed-point warp with inverse m onto a w x h image reads pixel
    (x + x0, y + y0) with zero fraction for every output pixel (x, y) — checked separably:
    X0[y] + adelta[x] must lie in [1024 (x0 + x), 1024 (x0 + x) + 31] for all x, y."""
    ad, bd, X0, Y0 = _fixed_point_terms(m, w, h)
    ax = ad - 1024 * np.arange(w)
    by = Y0 - 1024 * np.arange(h)
    lo_x, hi_x = X0.min() + ax.min(), X0.max() + ax.max()
    lo_y, hi_y = by.min() + bd.min(), by.max() + bd.max()
    return lo_x >= 1024 * x0 and hi_x <= 1024 * x0 + 31 and lo_y >= 1024 * y0 and hi_y <= 1024 * y0 + 31


def _check_box(box):
    x0, y0, x1, y1 = (int(v) for v in box)
    w, h = x1 - x0, y1 - y0
    if w < 1 or h < 1:
        raise ValueError(f"box {[x0, y0, x1, y1]} has width {w} / height {h} < 1 (cv2.warpAffine fails on it)")
    if w >= SIDE_LIMIT or h >= SIDE_LIMIT:
        raise ValueError(f"box {[x0, y0, x1, y1]}: sides must be < {SIDE_LIMIT} (cv2.warpAffine fails beyond)")
    if max(abs(x0), abs(y0), abs(x1), abs(y1)) >= COORD_LIMIT:
        raise ValueError(f"box {[x0, y0, x1, y1]}: coordinates must satisfy |c| < 2^20")
    return x0, y0, w, h


def crop_params(boxes, crop_size=512):
    """opp_crop_params records (numpy, CROP_PARAMS) for crop_img_by_bbox's two warps of each box
    [x0, y0, x1, y1]: the inverse of the second (resize) map and the box as the virtual source."""
    boxes = np.asarray(boxes)
    if boxes.ndim != 2 or boxes.shape[1] != 4:
        raise ValueError(f"boxes must be [B, 4] = (x0, y0, x1, y1), got {boxes.shape}")
    if boxes.dtype.kind not in "iu":
        raise ValueError(f"boxes must be integers (the reference truncates to int32), got {boxes.dtype}")
    _check_side(crop_size, "crop_size")
    rec = np.zeros(len(boxes), dtype=CROP_PARAMS)
    for i, box in enumerate(boxes):
        x0, y0, w, h = _check_box(box)
        # first warp: box -> w x h at scale 1 must be the shift by (x0, y0) the kernel applies
        if not _is_integer_shift(_invert_affine(_box_map(box, (h, w))), w, h, x0, y0):
            raise RuntimeError(f"box {box.tolist()}: the first warp is not an integer shift")
        rec[i]["m"] = _invert_affine(_box_map(np.array([0, 0, w, h]), (crop_size, crop_size)))
        rec[i]["x0"], rec[i]["y0"], rec[i]["w"], rec[i]["h"] = x0, y0, w, h
    return rec


def _check_side(n, name):
    if not (isinstance(n, (int, np.integer)) and 1 <= n < SIDE_LIMIT):
        raise ValueError(f"{name} must be an integer in [1, {SIDE_LIMIT - 1}], got {n!r}")


# ------------------------------------------------------------------------------------------------
# device crop
# ------------------------------------------------------------------------------------------------
def _device():
    return torch.device("cuda", torch.cuda.current_device())


def _frames(frames, device=None, batched=True):
    """uint8 frames as a contiguous CUDA tensor [B, H, W] ([H, W] -> [1, H, W]).  Accepts a CUDA or
    CPU tensor, a numpy array, a path (read like the reference: cv2.imread(path, IMREAD_GRAYSCALE)) or
    a list of arrays / paths of one size."""
    if isinstance(frames, (list, tuple)):
        frames = np.stack([_read(f) for f in frames])
    elif isinstance(frames, str):
        frames = _read(frames)
    t = frames if torch.is_tensor(frames) else torch.from_numpy(np.ascontiguousarray(frames))
    if t.dtype != torch.uint8:
        raise TypeError(f"frames must be uint8 grayscale, got {t.dtype}")
    if t.dim() == 4 and t.shape[1] == 1:
        t = t[:, 0]
    elif t.dim() == 2:
        t = t[None]
    if t.dim() != 3:
        raise ValueError(f"frames must be [B, H, W], [B, 1, H, W] or [H, W], got {tuple(t.shape)}")
    _check_side(int(t.shape[1]), "frame height")
    _check_side(int(t.shape[2]), "frame width")
    dev = device if device is not None else (t.device if t.is_cuda else _device())
    return t.to(dev).contiguous()


def _read(f):
    if isinstance(f, str):
        img = _cv2().imread(f, _cv2().IMREAD_GRAYSCALE)
        if img is None:
            raise FileNotFoundError(f"cannot read image {f!r}")
        return img
    if torch.is_tensor(f):
        f = f.cpu().numpy()
    return np.asarray(f).reshape(np.asarray(f).shape[-2:])


def _launch_crop(frames, params, out, status=None):
    """opp_crop_resize_u8 on the current stream.  frames uint8 CUDA [B, H, W]; params: CUDA uint8
    [B * 64] (CROP_PARAMS records); out uint8 CUDA [B, 1, h, w] (or [B, h, w]); status int32 [B] or None."""
    B, H, W = frames.shape
    oh, ow = out.shape[-2:]
    if params.numel() != B * CROP_PARAMS.itemsize or out.numel() != B * oh * ow:
        raise ValueError("params / out do not match the frame batch")
    _lib.call("opp_crop_resize_u8", _lib.ptr(frames), B, H, W, _lib.ptr(params), _lib.ptr(out), oh, ow,
              _lib.ptr(status), _lib.stream())


def _params_tensor(rec):
    return torch.from_numpy(np.ascontiguousarray(rec).view(np.uint8))


def crop_resize_batched(frames_u8, boxes, crop_size=512):
    """crop_img_by_bbox's crop of B frames at once: frames uint8 [B, H, W] (CUDA tensor, or host data
    that is uploaded), boxes int [B, 4] = (x0, y0, x1, y1).  Returns the CUDA uint8 crops
    [B, 1, crop_size, crop_size], equal to the reference's two cv2.warpAffine calls."""
    rec = crop_params(boxes, crop_size)
    f = _frames(frames_u8)
    if len(rec) != f.shape[0]:
        raise ValueError(f"{len(rec)} boxes for {f.shape[0]} frames")
    with torch.cuda.device(f.device):
        out = torch.empty((f.shape[0], 1, crop_size, crop_size), dtype=torch.uint8, device=f.device)
        _launch_crop(f, _params_tensor(rec).to(f.device), out)
    return out


def get_image_crop_resize(image, box, resize_shape):
    """data_utils.get_image_crop_resize: (image_crop, trans_crop_homo [3, 3]) — the box of `image`
    resized to resize_shape = (h, w) by one cv2.warpAffine-exact warp on the device.  A numpy image
    gives a numpy crop, a tensor gives a CUDA uint8 tensor [h, w]."""
    as_numpy = not torch.is_tensor(image)
    f = _frames(image)
    if f.shape[0] != 1:
        raise ValueError("get_image_crop_resize takes one image")
    rh, rw = int(resize_shape[0]), int(resize_shape[1])
    _check_side(rh, "resize height")
    _check_side(rw, "resize width")
    M = _box_map(box, (rh, rw))
    rec = np.zeros(1, dtype=CROP_PARAMS)
    rec[0]["m"] = _invert_affine(M)
    rec[0]["w"], rec[0]["h"] = f.shape[2], f.shape[1]
    with torch.cuda.device(f.device):
        out = torch.empty((1, rh, rw), dtype=torch.uint8, device=f.device)
        _launch_crop(f, _params_tensor(rec).to(f.device), out)
    crop = out[0].cpu().numpy() if as_numpy else out[0]
    return crop, np.concatenate([M, np.array([[0, 0, 1]])], axis=0)


def crop_img_by_bbox(query_img, bbox, K=None, crop_size=512):
    """LocalFeatureObjectDetector.crop_img_by_bbox without `self`: (crop, K_crop or None).  query_img
    is a path (read as the reference does), a uint8 array or a uint8 tensor [H, W] / [1, 1, H, W];
    the crop is the CUDA uint8 tensor [1, 1, crop_size, crop_size] the matcher takes as query_image
    (the reference returns the numpy crop and divides by 255 afterwards; the matcher folds the /255
    into its first convolution)."""
    bbox = np.asarray(bbox)
    crop = crop_resize_batched(_frames(query_img), bbox[None], crop_size)
    return crop, (crop_K(bbox, K, crop_size) if K is not None else None)


def previous_pose_detect(query_img, K, pre_pose, bbox3D_corner, crop_size=512):
    """LocalFeatureObjectDetector.previous_pose_detect without `self`: (bbox int32 [4], crop CUDA
    uint8 [1, 1, crop_size, crop_size], K_crop [3, 3]) for the box of the 3D box corners projected
    with the previous frame's pose.  The reference's optional saving of the crop / K_crop is not done."""
    bbox = bbox_from_pose(K, pre_pose, bbox3D_corner)
    crop, K_crop = crop_img_by_bbox(query_img, bbox, K, crop_size)
    return bbox, crop, K_crop


# ------------------------------------------------------------------------------------------------
# tracking loop
# ------------------------------------------------------------------------------------------------
class _CropPrologue:
    """The crop as the first node of the matcher's forward (OnePosePlus_model._forward): `inputs` are
    copied to the device (into the graph's static buffers in CUDA-graph mode), then run() writes the
    crops into the forward's query_image."""

    def __init__(self, frames, rec):
        self.inputs = [frames, _params_tensor(rec)]
        self.key = ("crop_resize_u8", tuple(frames.shape))

    def run(self, inputs, out):
        _launch_crop(inputs[0], inputs[1], out)


class PoseTracker:
    """demo.py's tracking step for B independent sequences per call (demo.py:105-132): crop each frame
    at the box of its previous pose (``previous_pose_detect``) or at a box the caller supplies (the
    first frame, or a re-detection), run the matcher on the B crops in one forward, and solve the B
    poses with ``ransac_pnp_batched(solver="colmap")`` — the demo's
    ``ransac_PnP(K_crop, ..., pnp_reprojection_error=7, use_pycolmap_ransac=True)``.

    model: an eval-mode OnePosePlus_model on the GPU with the object's 3D bank resident
    (``model.set_bank``); K: the original intrinsics [3, 3] (shared) or [B, 3, 3]; bbox3d: the
    8 corners [8, 3] of the object's 3D box.  With a bank set (``model.set_banks``, several objects
    in one forward): bbox3d is [K_obj, 8, 3], one box per object, and object_ids (int [B]) gives each
    sequence's object; its crop uses its object's box and its frame is matched against its object.

    ``step(frames_u8, init_bbox=None)``: frames uint8 [B, H, W] (CUDA, host array, or a list of
    arrays / paths); init_bbox: None, or B entries of None or (x0, y0, x1, y1).  A sequence whose
    previous frame had fewer than 20 inliers (or that has no previous pose) and that gets no box
    comes back with ``needs_detection=True`` and nothing else: the demo would run its detector on it
    (``tracker.needs_detection`` tells beforehand).  Returns one dict per sequence: needs_detection,
    bbox (int32 [4]), K_crop [3, 3], crop (CUDA uint8 [1, 1, crop, crop]), pose [3, 4], pose_homo
    [4, 4], inliers (int64 indices into the frame's matches, as ransac_PnP returns them), state,
    mkpts_3d_db and mkpts_query_f (the frame's matches, CUDA)."""

    def __init__(self, model, K, bbox3d, reprojection_error=7, crop_size=512, object_ids=None):
        bank_set = getattr(model, "_bank_set", None)
        if getattr(model, "_bank", None) is None and bank_set is None:
            raise ValueError("PoseTracker needs the object's 3D bank resident: call model.set_bank(...) first")
        if (bank_set is None) != (object_ids is None):
            raise ValueError("object_ids goes with a bank set (model.set_banks) and only with one")
        _check_side(crop_size, "crop_size")
        if crop_size % 8 or crop_size < 16:
            raise ValueError(f"crop_size must be a multiple of 8 (>= 16) for the matcher, got {crop_size}")
        self.model = model
        self.K = np.asarray(K, dtype=np.float64)
        if self.K.shape[-2:] != (3, 3) or self.K.ndim not in (2, 3):
            raise ValueError(f"K must be [3, 3] or [B, 3, 3], got {self.K.shape}")
        self.object_ids = None
        if bank_set is None:
            self.bbox3d = np.asarray(bbox3d, dtype=np.float64).reshape(-1, 3)
        else:
            n_obj = len(bank_set["raw"])
            self.bbox3d = np.asarray(bbox3d, dtype=np.float64)
            if self.bbox3d.shape != (n_obj, 8, 3):
                raise ValueError(f"bbox3d must be [K_obj, 8, 3] = [{n_obj}, 8, 3] with a bank set, "
                                 f"got {self.bbox3d.shape}")
            self.object_ids = np.asarray(object_ids)
            if self.object_ids.ndim != 1 or self.object_ids.dtype.kind not in "iu" \
                    or self.object_ids.min(initial=0) < 0 or self.object_ids.max(initial=0) >= n_obj:
                raise ValueError(f"object_ids must be ints in [0, {n_obj}), got {object_ids}")
        self.reprojection_error = float(reprojection_error)
        self.crop_size = int(crop_size)
        self._pose = None
        self._n_inliers = None

    def reset(self):
        """Forget every sequence's previous pose."""
        self._pose = self._n_inliers = None

    @property
    def needs_detection(self):
        """bool [B]: sequences whose next frame has no trusted previous pose (None before the first step)."""
        if self._pose is None:
            return None
        return np.array([p is None or n < MIN_INLIERS for p, n in zip(self._pose, self._n_inliers)])

    def _K(self, b):
        return self.K if self.K.ndim == 2 else self.K[b]

    def _box3d(self, b):
        return self.bbox3d if self.object_ids is None else self.bbox3d[self.object_ids[b]]

    def step(self, frames_u8, init_bbox=None):
        if self.object_ids is not None:
            bank_set = getattr(self.model, "_bank_set", None)   # set_banks may have run since __init__
            if bank_set is None or len(bank_set["raw"]) != len(self.bbox3d):
                raise ValueError(f"PoseTracker was built for a set of {len(self.bbox3d)} objects; the model "
                                 f"now holds {'no set' if bank_set is None else len(bank_set['raw'])}")
        frames = _frames(frames_u8, device=torch.device("cuda", torch.cuda.current_device())
                         if not (torch.is_tensor(frames_u8) and frames_u8.is_cuda) else None)
        B = frames.shape[0]
        if self.K.ndim == 3 and self.K.shape[0] != B:
            raise ValueError(f"K holds {self.K.shape[0]} cameras for {B} sequences")
        if self.object_ids is not None and len(self.object_ids) != B:
            raise ValueError(f"object_ids holds {len(self.object_ids)} objects for {B} sequences")
        if self._pose is None:
            self._pose, self._n_inliers = [None] * B, [0] * B
        if len(self._pose) != B:
            raise ValueError(f"the tracker follows {len(self._pose)} sequences, got {B} frames (reset() first)")
        if init_bbox is None:
            init_bbox = [None] * B
        if len(init_bbox) != B:
            raise ValueError(f"init_bbox has {len(init_bbox)} entries for {B} sequences")
        results = [{"needs_detection": True} for _ in range(B)]
        active, boxes = [], []
        for b in range(B):
            if init_bbox[b] is not None:
                box = np.asarray(init_bbox[b])
                if box.shape != (4,):
                    raise ValueError(f"init_bbox[{b}] must be (x0, y0, x1, y1), got shape {box.shape}")
                box = box.astype(np.int32) if box.dtype.kind == "f" else box
            elif self._pose[b] is not None and self._n_inliers[b] >= MIN_INLIERS:
                box = bbox_from_pose(self._K(b), self._pose[b], self._box3d(b))
            else:
                continue
            active.append(b)
            boxes.append(box)
        if not active:
            return results
        rec = crop_params(np.stack(boxes), self.crop_size)
        K_crop = [crop_K(box, self._K(b), self.crop_size) for b, box in zip(active, boxes)]
        dev = frames.device
        sel = frames if len(active) == B else frames[torch.tensor(active, device=dev)]
        n = len(active)
        with torch.cuda.device(dev):
            crops = torch.empty((n, 1, self.crop_size, self.crop_size), dtype=torch.uint8, device=dev)
            data = {"query_image": crops}
            if self.object_ids is not None:
                data["object_ids"] = torch.as_tensor(self.object_ids[active], dtype=torch.int32)
            self.model._forward(data, prologue=_CropPrologue(sel, rec))
            Kc = torch.as_tensor(np.stack(K_crop), dtype=torch.float32).to(dev)
            r = pnp.ransac_pnp_batched(data["m_bids"], data["mkpts_3d_db"], data["mkpts_query_f"], Kc,
                                       reprojection_error=self.reprojection_error, solver="colmap")
            pose = r["pose"].double().cpu().numpy()      # the step's one wait for the device
            homo = r["pose_homo"].double().cpu().numpy()
            state = r["state"].cpu().numpy()
            mask = r["inlier_mask"].cpu().numpy()
            m_bids = data["m_bids"].cpu().numpy()
        for i, b in enumerate(active):
            sel_i = m_bids == i
            ok = bool(state[i])
            inl = np.nonzero(mask[sel_i])[0] if ok else np.array([], dtype=np.int64)
            idx = torch.as_tensor(np.nonzero(sel_i)[0], device=dev)
            results[b] = {"needs_detection": False, "bbox": boxes[i], "K_crop": K_crop[i], "crop": crops[i:i + 1],
                          "pose": pose[i], "pose_homo": homo[i], "inliers": inl, "state": ok,
                          "mkpts_3d_db": data["mkpts_3d_db"][idx], "mkpts_query_f": data["mkpts_query_f"][idx]}
            self._pose[b], self._n_inliers[b] = pose[i], len(inl)
        return results
