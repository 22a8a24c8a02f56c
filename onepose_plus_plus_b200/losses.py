"""Training loss of OnePose++ (drop-in for ``src/lightning_model/losses.py:Loss``) with the coarse
focal loss on the device when the model leaves a TrainConfHandle in ``data["conf_matrix"]``
(``conf_matrix_mode = "lazy"`` in train mode): forward and backward run on the opp_coarse_focal
kernels and the [B, L, S] confidence matrix is never built.  With a tensor in
``data["conf_matrix"]`` the loss is the reference formula on that tensor.  The fine loss (M x 3) is
PyTorch either way.  The ground truth is data["conf_matrix_gt"] or the list data["gt_sparse"]
(train_gt.SparseGT), which the handle's kernels read without its dense form.
"""
import torch
import torch.nn as nn

from .train_gt import SparseGT, gt_of
from .train_path import TrainConfHandle

try:
    from loguru import logger
except ImportError:          # the reference logs through loguru; the standard logger otherwise
    import logging
    logger = logging.getLogger(__name__)


class _CoarseFocal(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat3d, feat2d, handle, gt, alpha, gamma, pos_w, neg_w):
        from . import ops
        gt = gt.contiguous()
        loss, counts, wts, r, c = ops.coarse_focal_fwd(handle.a32, handle.b32, handle.st_rows, handle.st_cols, gt,
                                                       handle.col_mask, handle.scale, alpha, gamma, pos_w, neg_w)
        ctx.save_for_backward(r, c, wts, gt)
        ctx.handle, ctx.focal = handle, (alpha, gamma)
        ctx.mark_non_differentiable(counts)
        return loss, counts

    @staticmethod
    def backward(ctx, grad_loss, _grad_counts):
        from . import ops
        r, c, wts, gt = ctx.saved_tensors
        h = ctx.handle
        grad = grad_loss.detach().float().contiguous()
        da, db = ops.coarse_focal_bwd(h.a32, h.b32, h.st_rows, h.st_cols, r, c, wts, grad, gt, h.col_mask, h.scale,
                                      *ctx.focal)
        return da, db, None, None, None, None, None, None


class _CoarseFocalSparse(torch.autograd.Function):
    """_CoarseFocal with the ground truth as a SparseGT: its index is built once, here, and kept for
    the backward."""

    @staticmethod
    def forward(ctx, feat3d, feat2d, handle, gt, alpha, gamma, pos_w, neg_w):
        from . import ops
        row_ptr, col_ptr, col_rows = ops.gt_index(gt.b_ids, gt.i_ids, gt.j_ids, gt.shape)
        loss, counts, wts, r, c = ops.coarse_focal_fwd_sparse(handle.a32, handle.b32, handle.st_rows, handle.st_cols,
                                                              row_ptr, gt.j_ids, handle.col_mask, handle.scale,
                                                              alpha, gamma, pos_w, neg_w)
        ctx.save_for_backward(r, c, wts, row_ptr, gt.j_ids, col_ptr, col_rows)
        ctx.handle, ctx.focal = handle, (alpha, gamma)
        ctx.mark_non_differentiable(counts)
        return loss, counts

    @staticmethod
    def backward(ctx, grad_loss, _grad_counts):
        from . import ops
        r, c, wts, row_ptr, j_ids, col_ptr, col_rows = ctx.saved_tensors
        h = ctx.handle
        grad = grad_loss.detach().float().contiguous()
        da, db = ops.coarse_focal_bwd_sparse(h.a32, h.b32, h.st_rows, h.st_cols, r, c, wts, grad, row_ptr, j_ids,
                                             col_ptr, col_rows, h.col_mask, h.scale, *ctx.focal)
        return da, db, None, None, None, None, None, None


def _check_query_mask(handle):
    if handle.col_mask is not None and not bool(handle.col_mask.any(1).all()):
        raise ValueError("query_image_mask keeps no column of at least one sample: the coarse loss is not "
                         "defined for a fully padded query image")


def coarse_focal_loss(handle, conf_gt, alpha, gamma, pos_w, neg_w):
    """Focal loss of the dual-softmax confidence of `handle` against conf_gt (bool, uint8 or int16
    [B, L, S] on the device, or a SparseGT on the device: every listed element is a positive, every
    other one a negative), differentiable with respect to handle.feat3d / handle.feat2d.
    Returns (loss, counts): counts = int64 [2] (positives, negatives) on the device.
    A query mask that keeps no column of some sample raises ValueError (one synchronisation): the
    softmax over S of that sample has no terms, and the reference's -1e9 masking gives it a value
    (the unmasked softmax in fp64, a uniform one in fp32) that the kernels do not reproduce."""
    if isinstance(conf_gt, SparseGT):
        if tuple(conf_gt.shape) != tuple(handle.shape):
            raise ValueError(f"gt_sparse has shape {tuple(conf_gt.shape)}, the confidence {tuple(handle.shape)}")
        _check_query_mask(handle)
        return _CoarseFocalSparse.apply(handle.feat3d, handle.feat2d, handle, conf_gt, float(alpha), float(gamma),
                                        float(pos_w), float(neg_w))
    if conf_gt.dtype not in (torch.bool, torch.uint8, torch.int16):
        raise TypeError(f"conf_matrix_gt: expected bool, uint8 or int16, got {conf_gt.dtype}")
    if tuple(conf_gt.shape) != tuple(handle.shape):
        raise ValueError(f"conf_matrix_gt has shape {tuple(conf_gt.shape)}, the confidence {tuple(handle.shape)}")
    _check_query_mask(handle)
    return _CoarseFocal.apply(handle.feat3d, handle.feat2d, handle, conf_gt, float(alpha), float(gamma),
                              float(pos_w), float(neg_w))


class Loss(nn.Module):
    """Same constructor, forward(data) and outputs ("loss", "loss_scalars") as the reference Loss."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.correct_thr = config["fine_correct_thr"]
        self.c_pos_w = config["pos_weight"]
        self.c_neg_w = config["neg_weight"]
        self.fine_type = config["fine_type"]

    def compute_coarse_loss(self, conf, conf_gt, weight=None):
        """Focal loss over the positives (gt == 1) and negatives (gt == 0) of conf, each class
        averaged; an empty class drops out with a warning.  conf: tensor or TrainConfHandle; conf_gt:
        tensor or SparseGT.  A tensor conf with a SparseGT is the formula below on the list's dense
        form: correct, and as large as the dense ground truth while it runs."""
        if self.config["coarse_type"] != "focal":
            raise NotImplementedError
        alpha, gamma = self.config["focal_alpha"], self.config["focal_gamma"]
        if isinstance(conf, TrainConfHandle):
            if weight is not None:
                raise NotImplementedError("mask0 / mask1 loss weights are not built for the lazy confidence")
            loss, counts = coarse_focal_loss(conf, conf_gt, alpha, gamma, self.c_pos_w, self.c_neg_w)
            npos, nneg = counts.tolist()
            if npos == 0:
                logger.warning('len of loss pos is zero!')
            elif nneg == 0:
                logger.warning('len of loss neg is zero!')
            return loss
        if isinstance(conf_gt, SparseGT):
            conf_gt = conf_gt.to_dense()[0]
        c = torch.clamp(conf, 1e-6, 1 - 1e-6)
        pos, neg = conf_gt == 1, conf_gt == 0
        loss_pos = -alpha * torch.pow(1 - c[pos], gamma) * c[pos].log()
        loss_neg = -(1 - alpha) * torch.pow(c[neg], gamma) * (1 - c[neg]).log()
        if weight is not None:
            loss_pos = loss_pos * weight[pos]
            loss_neg = loss_neg * weight[neg]
        if loss_pos.shape[0] == 0:
            logger.warning('len of loss pos is zero!')
            return self.c_neg_w * loss_neg.mean()
        if loss_neg.shape[0] == 0:
            logger.warning('len of loss neg is zero!')
            return self.c_pos_w * loss_pos.mean()
        return self.c_pos_w * loss_pos.mean() + self.c_neg_w * loss_neg.mean()

    def compute_fine_loss(self, expec_f, expec_f_gt):
        if self.fine_type != "l2_with_std":
            raise NotImplementedError()
        return self._compute_fine_loss_l2_std(expec_f, expec_f_gt)

    def _compute_fine_loss_l2_std(self, expec_f, expec_f_gt):
        """expec_f [M, 3] (x, y, std), expec_f_gt [M, 2]: inverse-std weighted l2 over the matches
        whose gt offset lies inside the window."""
        correct = torch.linalg.norm(expec_f_gt, ord=float("inf"), dim=1) < self.correct_thr
        inv_std = 1.0 / torch.clamp(expec_f[:, 2], min=1e-10)
        weight = (inv_std / torch.mean(inv_std)).detach()
        if correct.sum() == 0:
            if not self.training:
                return None
            # rare in training (predictions are padded with gt): one near-zero term keeps DDP in step
            logger.warning("assign a false supervision to avoid ddp deadlock")
            correct[0] = True
            weight[0] = 1e-6
        off = ((expec_f_gt[correct] - expec_f[correct, :2]) ** 2).sum(-1)
        return (off * weight[correct]).mean()

    @torch.no_grad()
    def compute_c_weight(self, data):
        if "mask0" not in data:
            return None
        return data["mask0"].flatten(-2)[..., None] * data["mask1"].flatten(-2)[:, None]

    def forward(self, data):
        """Writes data["loss"] (the reduced loss of the batch) and data["loss_scalars"]."""
        scalars = {}
        if "mask0" in data and isinstance(data["conf_matrix"], TrainConfHandle):
            raise NotImplementedError("mask0 / mask1 loss weights are not built for the lazy confidence")
        gt = gt_of(data)
        loss_c = self.compute_coarse_loss(data["conf_matrix"], gt if gt is not None else data["conf_matrix_gt"],
                                          weight=self.compute_c_weight(data))
        loss = loss_c * self.config["coarse_weight"]
        scalars["loss_c"] = loss_c.clone().detach().cpu()
        if "expec_f" in data:
            loss_f = self.compute_fine_loss(data["expec_f"], data["expec_f_gt"])
            if loss_f is not None:
                loss += loss_f * self.config["fine_weight"]
                scalars["loss_f"] = loss_f.clone().detach().cpu()
            else:
                assert self.training is False
                scalars["loss_f"] = torch.tensor(1.0)   # 1 is the upper bound
        scalars["loss"] = loss.clone().detach().cpu()
        data.update({"loss": loss, "loss_scalars": scalars})
