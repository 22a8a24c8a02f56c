"""Writes tests/golden/reference/train_batch.npz: two collated batches of four items built by the
live reference OnePosePlusDataset (src/datasets/OnePosePlus_dataset.py) over seeded stand-ins
(oracle/train_batch.make_case), for the GPU tests, which cannot read the reference.

  warp   items 0..3 = indices 0..3 of an image_warp_adapt dataset: 1 and 3 warped; a 160x120 source
         resized to 128x96 (query_image_scale 1.25), collisions, a repeated 2D keypoint, points
         behind the camera and outside the image
  exact  four unwarped items with exact geometry (every reference matmul exact): the reference's
         fine locations equal the restatement's bit for bit

Per batch: the ProjectedGTDataset items' inputs (the unwarped image as the uint8 pixels it was read
from — the dataset's image is uint8 / 255 — keypoints3d, query_image_scale, assign / offsets /
n_2d, K_crop, pose_gt, homographies, 0 where none), the reference's warped images of the warped
items (its other images are the inputs), its query_intrinsic, and its list (SparseGT.from_dense of
the reference's collated dense tensors).  The images are 128x96 so that the file stays small; the
training shape (512², shape3d 7000) is covered by the synthetic batches of the GPU tests.
Run: python -m oracle.make_train_batch_golden
"""
import os
import tempfile

import numpy as np
import torch
from torch.utils.data import default_collate

from onepose_plus_plus_b200 import train_batch, train_gt
from . import ref_shims
from . import train_batch as otb

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference",
                      "train_batch.npz")

CASES = {
    "warp": dict(seed=7, n_items=2, warp=True, src_hw=(120, 160), img_resize=(128, 96), shape3d=300, n_3d=420,
                 n_corr=160, collide=6, repeat_2d=4, behind=4, outside=8),
    "exact": dict(seed=8, n_items=4, warp=False, src_hw=(120, 160), img_resize=(128, 96), shape3d=300, n_3d=260,
                  n_corr=150, collide=6, repeat_2d=4, exact=True),
}


def build(name, root):
    case = otb.make_case(root, **CASES[name])
    ds = otb.reference_dataset(case)
    mine = train_batch.ProjectedGTDataset(ds)
    refs, items = [], []
    for idx in range(4):
        seed = case["item_seeds"][idx // 2 if case["warp"] else idx]
        np.random.seed(seed)
        torch.manual_seed(seed)
        refs.append(ds[idx])
        np.random.seed(seed)
        torch.manual_seed(seed)
        items.append(mine[idx])
    return refs, items


def image_of(u8):
    """the dataset's fp32 image of uint8 pixels (read_grayscale: grayscale2tensor, image / 255.)"""
    return torch.from_numpy(u8.numpy().astype(np.float32) / 255.).float()


def load(path, name):
    """one batch of the golden file as torch tensors, with "image" and the reference's "ref_image"
    rebuilt at full size"""
    z = np.load(path)
    d = {k.split("/", 1)[1]: torch.from_numpy(z[k]) for k in z.files if k.startswith(name + "/")}
    d["image"] = image_of(d.pop("image_u8"))
    ref = d["image"].clone()
    ref[d["warped"]] = d.pop("ref_warped")
    d["ref_image"] = ref
    return d


def arrays(name, refs, items):
    rb = default_collate(refs)
    gt = train_gt.SparseGT.from_dense(rb["conf_matrix_gt"], rb["fine_location_matrix_gt"])
    src = train_batch.collate(items)["gt_source"]
    H = np.stack([np.zeros((3, 3)) if h is None else np.asarray(h) for h in src.homography])
    mb = default_collate([{k: v for k, v in it.items() if k != "gt_source"} for it in items])
    warped = torch.tensor([h is not None for h in src.homography])
    u8 = torch.round(mb["query_image"] * 255).to(torch.uint8)
    assert torch.equal(image_of(u8), mb["query_image"]), "the image is not uint8 / 255"
    assert torch.equal(rb["query_image"][~warped], mb["query_image"][~warped])
    out = {"image_u8": u8, "keypoints3d": mb["keypoints3d"], "scale": mb["query_image_scale"],
           "assign": src.assign, "offsets": src.offsets, "kp_offsets": src.kp_offsets, "K_crop": src.K_crop,
           "pose_gt": src.pose_gt, "homography": torch.from_numpy(H),
           "warped": warped, "ref_warped": rb["query_image"][warped], "ref_intrinsic": rb["query_intrinsic"].double(),
           "ref_b": gt.b_ids, "ref_i": gt.i_ids, "ref_j": gt.j_ids, "ref_xy": gt.fine_xy,
           "shape": torch.tensor(gt.shape)}
    return {f"{name}/{k}": v.numpy() for k, v in out.items()}


def main():
    assert ref_shims.available(), "needs the reference tree"
    out = {}
    for name in CASES:
        with tempfile.TemporaryDirectory() as root:
            out.update(arrays(name, *build(name, root)))
    np.savez_compressed(GOLDEN, **out)
    print(f"{GOLDEN}: {os.path.getsize(GOLDEN) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
