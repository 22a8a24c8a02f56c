"""pytest -m gpu: the tracking front end on the device against cv2 and the composed host path.

* opp_crop_resize_u8 through crop_resize_batched is bit-equal to crop_img_by_bbox's two
  cv2.warpAffine calls, at B = 1 and B = 8 with mixed boxes;
* the drop-ins (get_image_crop_resize, crop_img_by_bbox, previous_pose_detect) return the crops of
  cv2 and the host geometry's bbox / K_crop;
* PoseTracker.step gives the same crop bytes, matches, poses and inliers as the host path
  (cv2 crop -> the same model on that uint8 crop -> ransac_pnp_batched(solver="colmap")) over a
  5-frame planted sequence of two cameras, eager and with CUDA graphs;
* a sequence whose previous frame had fewer than 20 inliers comes back needs_detection;
* the kernel's per-frame status on a zero-width box and on a far box."""
import cv2
import numpy as np
import pytest
import torch

from onepose_plus_plus_b200 import OnePosePlus_model, pnp, tracking
from oracle import oracle, workload

pytestmark = pytest.mark.gpu

CROP = 512


def _frame(rng, H, W):
    return cv2.GaussianBlur(rng.integers(0, 256, (H, W), dtype=np.uint8), (0, 0), 1.5)


def _cv2_crop(frame, box, crop=CROP):
    x0, y0, x1, y1 = (int(v) for v in box)
    w, h = x1 - x0, y1 - y0
    s1 = cv2.warpAffine(frame, tracking._box_map(box, (h, w)), (w, h), flags=cv2.INTER_LINEAR)
    return cv2.warpAffine(s1, tracking._box_map(np.array([0, 0, w, h]), (crop, crop)), (crop, crop),
                          flags=cv2.INTER_LINEAR)


def _mixed_boxes(rng, n, H, W):
    kinds = [(W // 4, H // 4, 3 * W // 4, 3 * H // 4), (-W // 5, -H // 6, W // 2, H + 30),
             (W + 10, 5, W + 90, 300), (-W, -H, 2 * W, 2 * H), (37, 11, 38, H - 3), (5, 40, W - 9, 41),
             (100, -20, 104, H + 20), (-30, 200, W + 30, 203)]
    out = [kinds[i % len(kinds)] for i in range(n)]
    if n == 1:
        out = [(int(rng.integers(-50, W // 3)), int(rng.integers(-50, H // 3)), W - 7, H - 5)]
    return np.array(out, dtype=np.int32)


@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("size", [(480, 640), (1441, 1919)])
def test_crop_resize_batched_bit_equal_to_cv2(B, size):
    rng = np.random.default_rng(B * 7 + size[0])
    H, W = size
    frames = np.stack([_frame(rng, H, W) for _ in range(B)])
    boxes = _mixed_boxes(rng, B, H, W)
    for src in (torch.from_numpy(frames).cuda(), frames):    # device frames, host frames
        got = tracking.crop_resize_batched(src, boxes, CROP)
        assert got.shape == (B, 1, CROP, CROP) and got.dtype == torch.uint8 and got.is_cuda
        got = got.cpu().numpy()
        for b in range(B):
            assert np.array_equal(got[b, 0], _cv2_crop(frames[b], boxes[b])), (b, boxes[b].tolist())
    # a crop side that is not a multiple of 4 (byte stores at the row ends)
    got = tracking.crop_resize_batched(frames, boxes, 203).cpu().numpy()
    for b in range(B):
        assert np.array_equal(got[b, 0], _cv2_crop(frames[b], boxes[b], 203))


def test_dropins_return_reference_values(tmp_path):
    rng = np.random.default_rng(11)
    frame = _frame(rng, 480, 640)
    path = str(tmp_path / "frame.png")
    cv2.imwrite(path, frame)
    K = np.array([[572.4, 0, 325.3], [0, 573.6, 242.0], [0, 0, 1]])
    box = np.array([120, 60, 391, 433], dtype=np.int32)
    want = _cv2_crop(frame, box)
    for q in (path, frame, torch.from_numpy(frame).cuda(), torch.from_numpy(frame)[None, None].cuda()):
        crop, K_crop = tracking.crop_img_by_bbox(q, box, K)
        assert crop.shape == (1, 1, CROP, CROP) and crop.dtype == torch.uint8 and crop.is_cuda
        assert np.array_equal(crop[0, 0].cpu().numpy(), want)
        assert np.array_equal(K_crop, tracking.crop_K(box, K, CROP))
    assert tracking.crop_img_by_bbox(frame, box)[1] is None
    # one warp, reference signature: numpy in -> numpy out, tensor in -> CUDA tensor out
    for bx, shape in ((box, (box[3] - box[1], box[2] - box[0])), (np.array([0, 0, 271, 373]), (512, 512)),
                      (np.array([-40, 30, 700, 90]), (100, 333))):
        ref = cv2.warpAffine(frame, tracking._box_map(bx, shape), (int(shape[1]), int(shape[0])), flags=cv2.INTER_LINEAR)
        img, T = tracking.get_image_crop_resize(frame, bx, np.array(shape))
        assert isinstance(img, np.ndarray) and np.array_equal(img, ref)
        assert np.array_equal(T[:2], tracking._box_map(bx, shape)) and np.array_equal(T[2], [0, 0, 1])
        img_t, _ = tracking.get_image_crop_resize(torch.from_numpy(frame).cuda(), bx, shape)
        assert img_t.is_cuda and np.array_equal(img_t.cpu().numpy(), ref)
    # previous_pose_detect: the box of the projected corners, truncated to int32
    pose = np.concatenate([np.eye(3), [[0.01], [-0.02], [0.7]]], 1)
    corners = np.array([[x, y, z] for x in (-0.1, 0.1) for y in (-0.08, 0.12) for z in (-0.05, 0.05)])
    bbox, crop, K_crop = tracking.previous_pose_detect(path, K, pose, corners)
    assert bbox.dtype == np.int32 and np.array_equal(bbox, tracking.bbox_from_pose(K, pose, corners))
    assert np.array_equal(crop[0, 0].cpu().numpy(), _cv2_crop(frame, bbox))
    assert np.array_equal(K_crop, tracking.crop_K(bbox, K, CROP))


def test_kernel_status_on_invalid_boxes():
    frames = torch.from_numpy(np.full((3, 64, 64), 200, np.uint8)).cuda()
    rec = tracking.crop_params(np.array([[4, 4, 60, 60]] * 3), 32)
    rec[1]["w"] = 0                        # zero-width box: cv2 raises on it
    rec[2]["x0"] = 1 << 20                 # outside the fixed-point range
    params = tracking._params_tensor(rec).cuda()
    out = torch.full((3, 32, 32), 7, dtype=torch.uint8, device="cuda")
    status = torch.full((3,), -1, dtype=torch.int32, device="cuda")
    tracking._launch_crop(frames, params, out, status)
    assert status.cpu().tolist() == [0, 1, 2]
    assert (out[0] == 200).all().item() and (out[1:] == 0).all().item()
    with pytest.raises(ValueError, match="width 0"):
        tracking.crop_resize_batched(frames, np.array([[4, 4, 4, 60]] * 3), 32)


# ------------------------------------------------------------------------------------------------
# PoseTracker against the composed host path
# ------------------------------------------------------------------------------------------------
F, Z, HALF = 600.0, 0.6, 0.25
FRAME_HW = (600, 720)
OFFSETS = [(96, 40), (150, 70)]     # (ox, oy) of the object image in each camera's frames


@torch.no_grad()
def _tracking_scene(sd, n_points=2000, n_planted=1200, seed=1, alpha=20.0, beta=8.0):
    """A 512 x 512 object image and a bank planted from its own features (as
    oracle/workload.planted_workload) whose 3D points sit where a camera with focal F at distance Z
    sees the planted fine features, so the PnP finds a pose with 20 to 40 inliers on the object's
    true box (fewer on boxes a few pixels off, which then need re-detection).  Returns the uint8 image,
    the bank and the object's 3D box corners."""
    g = torch.Generator().manual_seed(seed)
    # smooth texture: its features survive the pixel or two the tracked box moves between frames
    noise = torch.rand(CROP, CROP, generator=g).numpy()
    smooth = cv2.GaussianBlur(noise, (0, 0), 2.0)
    smooth = (smooth - smooth.min()) / (smooth.max() - smooth.min())
    base = torch.from_numpy(np.round(smooth * 255) / 255).float()[None, None]   # what the uint8 frames hold
    fc, ff = oracle.backbone(sd, base)
    hc, wc = fc.shape[2:]
    pe = oracle.position_encoding_sine(256, hc, wc)
    qc = (fc + pe[None]).flatten(2).transpose(1, 2)[0]
    mu = qc.mean(0)
    r = qc - mu
    mu_dir = mu / mu.norm()
    r = r - (r @ mu_dir)[:, None] * mu_dir[None]
    ys, xs = torch.meshgrid(torch.arange(2, hc), torch.arange(2, wc), indexing="ij")
    interior = (ys * wc + xs).flatten()
    cells = interior[torch.randperm(interior.numel(), generator=g)[:n_planted]]
    hf, wf = ff.shape[2:]
    stride = hf // hc
    off = torch.randint(-2, 3, (n_planted, 2), generator=g)
    fy = ((cells // wc) * stride + off[:, 0]).clamp(0, hf - 1)
    fx = ((cells % wc) * stride + off[:, 1]).clamp(0, wf - 1)
    # planted points: back-projection of their fine pixel (2 fx, 2 fy) of the crop, depth Z +- 1 cm
    z = Z + 0.01 * (torch.rand(n_planted, generator=g) * 2 - 1)
    u, v = 2.0 * fx.double(), 2.0 * fy.double()
    planted = torch.stack([(u - 256) / F * z, (v - 256) / F * z, z - Z], 1)
    rest = torch.rand(n_points - n_planted, 3, generator=g, dtype=torch.float64) * 0.4 - 0.2
    kpts = torch.cat([planted, rest], 0).float()[None]
    kenc = oracle.keypoint_encoding(sd, oracle.normalize_3d_keypoints(kpts), torch.zeros(1, 256, n_points))
    dc = torch.randn(1, 256, n_points, generator=g) * r.std() * alpha / 4
    dc[0, :, :n_planted] = alpha * r[cells].t() - kenc[0, :, :n_planted]
    ffc = ff[0] - ff[0].mean((1, 2), keepdim=True)
    df = torch.randn(1, 128, n_points, generator=g) * ff.std()
    df[0, :, :n_planted] = beta * ffc[:, fy, fx]
    img = (base[0, 0] * 255).round().to(torch.uint8).numpy()
    corners = np.array([[x, y, dz] for x in (-HALF, HALF) for y in (-HALF, HALF) for dz in (-0.01, 0.01)])
    return img, (kpts, df, dc), corners


def _sequence(img, n_frames=5, seed=2):
    """n_frames x cameras uint8 frames: the object image at each camera's offset over a textured
    background, fresh +-3 noise per frame; frame 3 of camera 1 shows only background."""
    rng = np.random.default_rng(seed)
    H, W = FRAME_HW
    frames = []
    for t in range(n_frames):
        fr = []
        for c, (ox, oy) in enumerate(OFFSETS):
            f = _frame(rng, H, W).astype(np.int16)
            if not (t == 3 and c == 1):
                f[oy:oy + CROP, ox:ox + CROP] = img
            f += rng.integers(-3, 4, f.shape).astype(np.int16)
            fr.append(np.clip(f, 0, 255).astype(np.uint8))
        frames.append(np.stack(fr))
    return frames


def _cameras():
    return np.stack([np.array([[F, 0, ox + 256.0], [0, F, oy + 256.0], [0, 0, 1]]) for ox, oy in OFFSETS])


def _init_boxes():
    return [np.array([ox, oy, ox + CROP, oy + CROP], dtype=np.int32) for ox, oy in OFFSETS]


@pytest.fixture(scope="module")
def scene():
    sd = workload.synthetic_state_dict(0)
    model = OnePosePlus_model(oracle.DEFAULT_CONFIG)
    model.load_state_dict(sd, strict=True)
    model = model.eval().cuda()
    img, (kpts, df, dc), corners = _tracking_scene(sd)
    model.set_bank(kpts.cuda(), df.cuda(), dc.cuda())
    return model, img, corners


def _host_path(model, frames, corners, K):
    """demo.py's loop composed from the host pieces: box from the previous pose, the two cv2 warps,
    the matcher on the uint8 crops, ransac_pnp_batched(solver="colmap") on K_crop."""
    B = len(OFFSETS)
    prev = [None] * B
    out = []
    for t, fr in enumerate(frames):
        active, boxes = [], []
        for b in range(B):
            if prev[b] is not None and len(prev[b][1]) >= 20:
                box = tracking.bbox_from_pose(K[b], prev[b][0], corners)
            else:   # demo.py:108-112: the detector supplies the box (here: the object's true box)
                box = _init_boxes()[b]
            active.append(b)
            boxes.append(box)
        step = [None] * B
        if active:
            crops = np.stack([_cv2_crop(fr[b], box) for b, box in zip(active, boxes)])
            data = {"query_image": torch.from_numpy(crops[:, None]).cuda()}
            model(data)
            Kc = np.stack([tracking.crop_K(box, K[b], CROP) for b, box in zip(active, boxes)])
            r = pnp.ransac_pnp_batched(data["m_bids"], data["mkpts_3d_db"], data["mkpts_query_f"],
                                       torch.as_tensor(Kc, dtype=torch.float32).cuda(), reprojection_error=7,
                                       solver="colmap")
            mb = data["m_bids"].cpu().numpy()
            for i, b in enumerate(active):
                sel = mb == i
                ok = bool(r["state"][i].item())
                inl = np.nonzero(r["inlier_mask"].cpu().numpy()[sel])[0] if ok else np.array([], np.int64)
                pose = r["pose"][i].double().cpu().numpy()
                step[b] = {"detected": prev[b] is None or len(prev[b][1]) < 20, "bbox": boxes[i], "crop": crops[i], "K_crop": Kc[i], "pose": pose, "inliers": inl,
                           "mkpts_3d_db": data["mkpts_3d_db"].cpu().numpy()[sel],
                           "mkpts_query_f": data["mkpts_query_f"].cpu().numpy()[sel]}
                prev[b] = (pose, inl)
        out.append(step)
    return out


@pytest.mark.parametrize("graphs", [False, True])
def test_pose_tracker_equals_host_path(scene, graphs):
    model, img, corners = scene
    frames = _sequence(img)
    K = _cameras()
    model.enable_cuda_graphs(False)
    host = _host_path(model, frames, corners, K)
    model.enable_cuda_graphs(graphs)
    try:
        tr = tracking.PoseTracker(model, K, corners, reprojection_error=7)
        tracked = redetected = 0
        for t, fr in enumerate(frames):
            src = torch.from_numpy(fr).cuda() if t % 2 else fr      # device and host frames
            # the tracker's own verdict on which sequences need the detector is the host path's
            need = [True] * len(OFFSETS) if t == 0 else tr.needs_detection.tolist()
            assert need == [host[t][b]["detected"] for b in range(len(OFFSETS))], t
            res = tr.step(src, init_bbox=[_init_boxes()[b] if need[b] else None for b in range(len(OFFSETS))])
            for b in range(len(OFFSETS)):
                h, g = host[t][b], res[b]
                assert not g["needs_detection"]
                assert np.array_equal(g["bbox"], h["bbox"]) and np.array_equal(g["K_crop"], h["K_crop"])
                assert np.array_equal(g["crop"][0, 0].cpu().numpy(), h["crop"]), (t, b)
                for k in ("mkpts_3d_db", "mkpts_query_f"):
                    assert np.array_equal(g[k].cpu().numpy(), h[k]), (t, b, k)
                assert np.array_equal(g["pose"], h["pose"]) and np.array_equal(g["inliers"], h["inliers"]), (t, b)
                assert np.array_equal(g["pose_homo"][:3], g["pose"]) and g["pose_homo"][3].tolist() == [0, 0, 0, 1]
                if t > 0:
                    redetected += h["detected"]
                    tracked += not h["detected"]
    finally:
        model.enable_cuda_graphs(False)
    # the sequence exercises both branches: frames cropped at the previous pose's box, and frames
    # re-detected after fewer than 20 inliers (camera 1 loses the object at frame 3)
    counts = [[len(s["inliers"]) for s in step] for step in host]
    print("inliers per frame and camera:", counts, "tracked", tracked, "re-detected", redetected)
    assert min(counts[0]) >= 20 and tracked >= 2 and redetected >= 1
    assert counts[3][1] < 20 and host[4][1]["detected"]


def test_needs_detection(scene):
    model, img, corners = scene
    K = _cameras()
    frames = _sequence(img)
    tr = tracking.PoseTracker(model, K, corners)
    assert tr.needs_detection is None
    res = tr.step(frames[0], init_bbox=[_init_boxes()[0], None])     # camera 1: no box, no pose
    assert not res[0]["needs_detection"] and res[1] == {"needs_detection": True}
    assert tr.needs_detection.tolist() == [False, True]
    # camera 0 on a frame without the object: few inliers -> its next frame needs detection
    blank = np.stack([_frame(np.random.default_rng(9), *FRAME_HW)] * 2)
    res = tr.step(blank)
    assert len(res[0]["inliers"]) < 20 and res[1]["needs_detection"]
    assert tr.needs_detection.tolist() == [True, True]
    res = tr.step(frames[1])
    assert all(r == {"needs_detection": True} for r in res)
    # a re-detection box restarts the sequence
    res = tr.step(frames[1], init_bbox=_init_boxes())
    assert all(len(r["inliers"]) >= 20 for r in res) and not tr.needs_detection.any()
    with pytest.raises(ValueError, match="sequences"):
        tr.step(frames[1][:1])
