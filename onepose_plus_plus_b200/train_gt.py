"""Sparse ground truth of a training batch: the correspondences as a list instead of the two
[B, L, S]-sized tensors the reference dataset builds (``conf_matrix_gt`` int16 [B, L, S] and
``fine_location_matrix_gt`` fp32 [B, L, S, 2], OnePosePlus_dataset.py:174-236).

``data["gt_sparse"]`` (a SparseGT) is read by the training forward (the ground-truth padding of the
coarse matches), by ``fine_supervision`` below (drop-in for
src/models/OnePosePlus/utils/fine_supervision.py) and by ``losses.Loss``.  On CUDA the coarse loss and
the fine supervision run on the opp_coarse_focal_*_sparse / opp_fine_supervision kernels; on the CPU
they are the reference formulas.  A batch carries either ``gt_sparse`` or the dense tensors, never both.
"""
import torch

FINE_FILL = -50.0      # fine_location_matrix_gt where there is no correspondence (OnePosePlus_dataset.py:190)


def _validate(b_ids, i_ids, j_ids, shape):
    """Ranges, and strictly ascending (b, i, j) — which is also uniqueness."""
    B, L, S = shape
    if len(b_ids) == 0:
        return
    for name, t, n in (("b_ids", b_ids, B), ("i_ids", i_ids, L), ("j_ids", j_ids, S)):
        if bool(((t < 0) | (t >= n)).any()):
            raise ValueError(f"SparseGT: {name} outside [0, {n})")
    key = (b_ids * L + i_ids) * S + j_ids
    if bool((key[1:] <= key[:-1]).any()):
        raise ValueError("SparseGT: the list must be ascending in (b, i, j) without duplicates "
                         "(the order of torch.where(conf_matrix_gt))")


class SparseGT:
    """The positives of conf_matrix_gt [B, L, S] with their fine locations.
      b_ids, i_ids, j_ids  int64 [G], ascending in (b, i, j), no duplicates — the order of
                           torch.where(conf_matrix_gt), which the ground-truth padding draws from
      fine_xy              fp32 [G, 2], (x, y) in query-image pixels = fine_location_matrix_gt[b, i, j]
      shape                (B, L, S)
    CPU tensors are validated on construction; for CUDA tensors call .check() (one synchronisation)."""

    def __init__(self, b_ids, i_ids, j_ids, fine_xy, shape):
        self.shape = torch.Size(tuple(int(n) for n in shape))
        if len(self.shape) != 3 or min(self.shape) <= 0:
            raise ValueError(f"SparseGT: shape must be (B, L, S), got {tuple(shape)}")
        ids = []
        for name, t in (("b_ids", b_ids), ("i_ids", i_ids), ("j_ids", j_ids)):
            if t.dtype != torch.int64 or t.dim() != 1 or t.shape != b_ids.shape or t.device != b_ids.device:
                raise ValueError(f"SparseGT: {name} must be an int64 [G] tensor on the device of b_ids")
            ids.append(t.contiguous())
        self.b_ids, self.i_ids, self.j_ids = ids
        if fine_xy.dtype != torch.float32 or tuple(fine_xy.shape) != (len(b_ids), 2) or \
                fine_xy.device != b_ids.device:
            raise ValueError("SparseGT: fine_xy must be a float32 [G, 2] tensor on the device of b_ids")
        self.fine_xy = fine_xy.contiguous()
        if not b_ids.is_cuda:
            self.check()

    def check(self):
        """Raises ValueError unless the list is in range, ascending in (b, i, j) and free of duplicates."""
        _validate(self.b_ids, self.i_ids, self.j_ids, self.shape)
        return self

    def __len__(self):
        return self.b_ids.shape[0]

    @property
    def device(self):
        return self.b_ids.device

    @property
    def counts(self):
        """int64 [B]: positives per sample"""
        return torch.bincount(self.b_ids, minlength=self.shape[0])

    @classmethod
    def from_dense(cls, conf_matrix_gt, fine_location_matrix_gt):
        if fine_location_matrix_gt.shape != conf_matrix_gt.shape + (2,):
            raise ValueError(f"fine_location_matrix_gt has shape {tuple(fine_location_matrix_gt.shape)}, "
                             f"conf_matrix_gt {tuple(conf_matrix_gt.shape)}")
        if bool(((conf_matrix_gt != 0) & (conf_matrix_gt != 1)).any()):
            raise ValueError("SparseGT holds positives only: conf_matrix_gt must be 0 or 1 everywhere")
        b, i, j = torch.where(conf_matrix_gt)
        return cls(b, i, j, fine_location_matrix_gt[b, i, j].float(), conf_matrix_gt.shape)

    def to_dense(self):
        """(conf_matrix_gt int16 [B, L, S], fine_location_matrix_gt fp32 [B, L, S, 2] filled with -50)"""
        conf = torch.zeros(self.shape, dtype=torch.int16, device=self.device)
        fine = torch.full(tuple(self.shape) + (2,), FINE_FILL, dtype=torch.float32, device=self.device)
        conf[self.b_ids, self.i_ids, self.j_ids] = 1
        fine[self.b_ids, self.i_ids, self.j_ids] = self.fine_xy
        return conf, fine

    def _map(self, fn):
        out = object.__new__(SparseGT)
        out.shape = self.shape
        out.b_ids, out.i_ids, out.j_ids, out.fine_xy = (fn(t) for t in (self.b_ids, self.i_ids, self.j_ids,
                                                                        self.fine_xy))
        return out

    def to(self, device, non_blocking=False):
        return self._map(lambda t: t.to(device, non_blocking=non_blocking))

    def pin_memory(self):
        return self._map(lambda t: t.pin_memory())

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in (self.b_ids, self.i_ids, self.j_ids, self.fine_xy))


def sparse_gt_sample(i_ids, j_ids, fine_xy, L, S):
    """What a dataset returns per item in place of build_assignmatrix's two matrices
    (OnePosePlus_dataset.py:174-236): i_ids = 3D point of each correspondence (assign_matrix[1]),
    j_ids = its coarse cell, fine_xy [n, 2] = its fine 2D location.  The reference's filters apply
    (i < L = shape3d kept, j > S dropped), a cell written twice keeps the last location as the
    matrix assignment does, and the result is sorted by (i, j)."""
    i_ids, j_ids = torch.as_tensor(i_ids).long().reshape(-1), torch.as_tensor(j_ids).long().reshape(-1)
    fine_xy = torch.as_tensor(fine_xy).float().reshape(-1, 2)
    if not len(i_ids) == len(j_ids) == len(fine_xy):
        raise ValueError("sparse_gt_sample: i_ids, j_ids and fine_xy differ in length")
    keep = (i_ids < L) & ~(j_ids > S)
    i_ids, j_ids, fine_xy = i_ids[keep], j_ids[keep], fine_xy[keep]
    if bool(((i_ids < 0) | (j_ids < 0) | (j_ids >= S)).any()):
        raise ValueError(f"sparse_gt_sample: correspondence outside the {L} x {S} assignment matrix")
    key = i_ids * S + j_ids
    order = torch.argsort(key, stable=True)
    key = key[order]
    last = torch.ones(len(key), dtype=torch.bool)
    last[:-1] = key[1:] != key[:-1]
    order = order[last]
    return {"i_ids": i_ids[order], "j_ids": j_ids[order], "fine_xy": fine_xy[order], "shape": (int(L), int(S))}


def collate_sparse_gt(samples):
    """The SparseGT of a batch from its sparse_gt_sample items (they may differ in length or be empty)."""
    shapes = {tuple(s["shape"]) for s in samples}
    if len(shapes) != 1:
        raise ValueError(f"collate_sparse_gt: samples of different shapes {sorted(shapes)}")
    (L, S), = shapes
    b_ids = torch.cat([torch.full((len(s["i_ids"]),), b, dtype=torch.int64) for b, s in enumerate(samples)])
    return SparseGT(b_ids, *(torch.cat([s[k] for s in samples]) for k in ("i_ids", "j_ids", "fine_xy")),
                    (len(samples), L, S))


class SparseGTDataset(torch.utils.data.Dataset):
    """Wraps a dataset with the reference's items: in the worker, an item's conf_matrix_gt [L, S] and
    fine_location_matrix_gt [L, S, 2] become item["gt_sparse"] (a sparse_gt_sample) and the two dense
    keys are dropped, so they are never collated, pinned or copied.  Use with collate_fn=collate."""

    def __init__(self, dataset):
        self.dataset = dataset

    def __len__(self):
        return len(self.dataset)

    def __getitem__(self, index):
        item = self.dataset[index]
        if "conf_matrix_gt" in item:
            conf, fine = item.pop("conf_matrix_gt"), item.pop("fine_location_matrix_gt")
            i, j = torch.where(conf)
            item["gt_sparse"] = sparse_gt_sample(i, j, fine[i, j], *conf.shape)
        return item


def collate(items):
    """collate_fn of a DataLoader over SparseGTDataset: torch's default collation, with the
    gt_sparse items joined by collate_sparse_gt."""
    from torch.utils.data import default_collate
    sparse = [it["gt_sparse"] for it in items if "gt_sparse" in it]
    if sparse and len(sparse) != len(items):
        raise ValueError("collate: some items of the batch have gt_sparse and some do not")
    batch = default_collate([{k: v for k, v in it.items() if k != "gt_sparse"} for it in items])
    if sparse:
        batch["gt_sparse"] = collate_sparse_gt(sparse)
    return batch


def gt_of(data):
    """data["gt_sparse"] or None; a batch that also carries conf_matrix_gt is ambiguous."""
    gt = data.get("gt_sparse")
    if gt is None:
        return None
    if not isinstance(gt, SparseGT):
        raise TypeError(f'data["gt_sparse"] must be a SparseGT, got {type(gt).__name__}')
    if "conf_matrix_gt" in data:
        raise ValueError('data has both "gt_sparse" and "conf_matrix_gt": pass one ground truth')
    return gt


@torch.no_grad()
def fine_supervision(data, config):
    """Drop-in for the reference fine_supervision (utils/fine_supervision.py): writes
    data["expec_f_gt"] [M, 2], the ground-truth offset of each coarse match inside its fine window.
    With data["gt_sparse"] on CUDA it is one opp_fine_supervision launch (fp32, the bits of the
    PyTorch formula); with gt_sparse on the CPU, or a dense fine_location_matrix_gt, the formula."""
    coarse_res, fine_res = list(config["OnePosePlus"]["loftr_backbone"]["resolution"])
    radius = config["OnePosePlus"]["loftr_fine"]["window_size"] // 2
    b_ids, i_ids, j_ids = data["b_ids"], data["i_ids"], data["j_ids"]
    w_c = data["q_hw_c"][1]
    gt = gt_of(data)
    if gt is not None and b_ids.is_cuda:
        from . import ops
        if gt.device != b_ids.device:
            raise ValueError(f"gt_sparse is on {gt.device}, the matches on {b_ids.device}")
        scale = data["query_image_scale"].float().contiguous() if "query_image_scale" in data else None
        data.update({"expec_f_gt": ops.fine_supervision(gt.b_ids, gt.i_ids, gt.j_ids, gt.fine_xy, gt.shape,
                                                        b_ids.contiguous(), i_ids.contiguous(), j_ids.contiguous(),
                                                        w_c, (coarse_res, fine_res), radius, scale)})
        return
    if gt is not None:
        B, L, S = gt.shape
        key = (gt.b_ids * L + gt.i_ids) * S + gt.j_ids
        want = (b_ids * L + i_ids) * S + j_ids
        pos = torch.searchsorted(key, want).clamp(max=max(len(key) - 1, 0))
        loc = torch.full((len(want), 2), FINE_FILL, device=want.device)
        if len(key):
            hit = key[pos] == want
            loc[hit] = gt.fine_xy[pos[hit]]
    else:
        loc = data["fine_location_matrix_gt"][b_ids, i_ids, j_ids]
    # fine_supervision.py:18-28, including its coarse scale = fine scale without query_image_scale
    if "query_image_scale" in data:
        coarse_scale = coarse_res * data["query_image_scale"][b_ids][:, [1, 0]]
        fine_scale = fine_res * data["query_image_scale"][b_ids][:, [1, 0]]
    else:
        coarse_scale = fine_scale = fine_res
    mkpts_query = torch.stack([j_ids % w_c, j_ids // w_c], dim=1) * coarse_scale
    data.update({"expec_f_gt": (loc - mkpts_query) / fine_scale / radius})
