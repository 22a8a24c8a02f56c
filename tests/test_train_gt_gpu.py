"""Sparse ground truth of training on the device: opp_gt_index against a torch construction, the
sparse focal loss and backward bit for bit against the dense entry points and against the fp64
oracle, opp_fine_supervision against the PyTorch formula and the stored reference values, and a
training step end to end with the list in place of the two dense tensors."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import coarse_loss as cl
from oracle import make_reference_golden as mrg
from oracle import make_train_gt_golden as mtg
from oracle import train_gt as otg
from oracle import workload
from onepose_plus_plus_b200 import OnePosePlus_model, SparseGT, losses, ops, train_gt, train_path
from tests import golden_io

pytestmark = pytest.mark.gpu
RTOL = 2e-4
FOCAL = (0.5, 2.0)
CM = types.SimpleNamespace(temperature=cl.TEMPERATURE)


def list_of(conf_gt):
    """SparseGT of a dense 0 / 1 matrix (fine locations: zeros) on the device"""
    b, i, j = torch.where(conf_gt.cuda())
    return SparseGT(b, i, j, torch.zeros(len(b), 2, device="cuda"), conf_gt.shape).check()


def planted_gt(conf_gt, wc=16, seed=4):
    """Fine locations for the planted train batch: cell origin * 8 + a seeded offset in [-6, 10) px."""
    b, i, j = torch.where(conf_gt)
    g = torch.Generator().manual_seed(seed)
    xy = torch.stack([j % wc, j // wc], 1).float() * 8 + torch.rand(len(b), 2, generator=g) * 16 - 6
    return SparseGT(b, i, j, xy, conf_gt.shape)


def many_to_many(B, L, S, density, seed):
    g = torch.Generator().manual_seed(seed)
    conf = torch.rand(B, L, S, generator=g) < density
    conf[0, 3, :] = True          # a 3D point listed on every cell, a cell listed on every 3D point
    conf[B - 1, :, S - 2] = True
    conf[B - 1, L - 1] = False    # an empty last row
    return conf


def index_by_torch(gt):
    B, L, S = gt.shape
    i32 = torch.int32
    row_ptr = torch.searchsorted(gt.b_ids * L + gt.i_ids, torch.arange(B * L + 1, device=gt.device)).to(i32)
    col_key = (gt.b_ids * S + gt.j_ids) * L + gt.i_ids
    order = torch.argsort(col_key)
    col_ptr = torch.searchsorted(col_key[order] // L, torch.arange(B * S + 1, device=gt.device)).to(i32)
    return row_ptr, col_ptr, gt.i_ids[order].to(i32)


# B S + 1 column pointers: 1025, 2049 and 16385 (B = 4, S = 4096, the training shape) take the
# one-CTA scan through 2, 3 and 17 rounds of 1024; "crowded_column" puts 899 entries in one column
SCANS = {"scan_1025": (4, 50, 256, 0.05), "scan_2049": (8, 40, 256, 0.05), "scan_16385": (4, 30, 4096, 0.01),
         "crowded_column": (2, 900, 70, 0.02)}


@pytest.mark.parametrize("case", ["planted", "one_sample_empty", "many_to_many", "empty"] + list(SCANS))
def test_gt_index(case):
    if case == "many_to_many":
        gt = list_of(many_to_many(3, 130, 150, 0.05, 0))
    elif case in SCANS:
        gt = list_of(many_to_many(*SCANS[case], 5))
    else:
        conf = mrg.train_batch(workload.synthetic_state_dict(0), False)["conf_matrix_gt"].clone()
        if case == "one_sample_empty":
            conf[0] = False
        elif case == "empty":
            conf[:] = False
        gt = list_of(conf)
        assert (case == "empty") == (len(gt) == 0)
    got = ops.gt_index(gt.b_ids, gt.i_ids, gt.j_ids, gt.shape)
    again = ops.gt_index(gt.b_ids, gt.i_ids, gt.j_ids, gt.shape)
    for name, g, a, w in zip(("row_ptr", "col_ptr", "col_rows"), got, again, index_by_torch(gt)):
        assert g.dtype == torch.int32 and torch.equal(g, w), name
        assert torch.equal(g, a), name
    if case == "crowded_column":
        assert int(got[1].diff().max()) > 800
    elif case in SCANS:
        assert got[1].numel() == int(case[5:])


def _dense_and_sparse(a, b, conf_gt, mask, grad=0.7):
    """Every output of the forward and the backward, dense and sparse, on one handle."""
    h = train_path.TrainConfHandle(CM, a.cuda(), b.cuda(), mask.cuda() if mask is not None else None)
    gt = list_of(conf_gt)
    dense = gt.to_dense()[0]
    assert torch.equal(dense.bool(), conf_gt.cuda().bool())
    go = torch.tensor(grad, device="cuda")
    fwd_d = ops.coarse_focal_fwd(h.a32, h.b32, h.st_rows, h.st_cols, dense, h.col_mask, h.scale, *FOCAL, 1.0, 1.0)
    bwd_d = ops.coarse_focal_bwd(h.a32, h.b32, h.st_rows, h.st_cols, *fwd_d[3:], fwd_d[2], go, dense, h.col_mask,
                                 h.scale, *FOCAL)
    del dense
    row_ptr, col_ptr, col_rows = ops.gt_index(gt.b_ids, gt.i_ids, gt.j_ids, gt.shape)
    fwd_s = ops.coarse_focal_fwd_sparse(h.a32, h.b32, h.st_rows, h.st_cols, row_ptr, gt.j_ids, h.col_mask, h.scale,
                                        *FOCAL, 1.0, 1.0)
    bwd_s = ops.coarse_focal_bwd_sparse(h.a32, h.b32, h.st_rows, h.st_cols, *fwd_s[3:], fwd_s[2], go, row_ptr,
                                        gt.j_ids, col_ptr, col_rows, h.col_mask, h.scale, *FOCAL)
    names = ("loss", "counts", "wts", "r", "c", "dA", "dB")
    return names, fwd_d + bwd_d, fwd_s + bwd_s, gt


def _assert_bits(names, dense, sparse):
    for name, d, s in zip(names, dense, sparse):
        assert torch.equal(d, s), f"{name}: sparse differs from dense"
    assert torch.isfinite(dense[0]) and int(dense[1][0]) > 0


@pytest.mark.parametrize("key", list(cl.GOLDEN_CASES))
def test_sparse_is_bit_identical_to_dense(key):
    name, batch, rows, cols = cl.GOLDEN_CASES[key]
    a, b, gt, mask = cl.make_case(name, batch, rows, cols)
    names, dense, sparse, _ = _dense_and_sparse(a, b, gt, mask)
    _assert_bits(names, dense, sparse)
    _, _, sparse2, _ = _dense_and_sparse(a, b, gt, mask)
    _assert_bits(names, sparse, sparse2)          # two calls: the same bits


@pytest.mark.parametrize("masked", [False, True])
def test_sparse_is_bit_identical_to_dense_many_to_many(masked):
    B, L, S = 3, 130, 150
    a, b, _, _ = cl.make_case("planted", B, L, S, seed=2)
    mask = None
    if masked:
        mask = torch.ones(B, S, dtype=torch.bool)
        mask[:, S - 40:] = False                  # positives on masked columns stay positives with c = 0
    names, dense, sparse, gt = _dense_and_sparse(a, b, many_to_many(B, L, S, 0.05, 1), mask)
    _assert_bits(names, dense, sparse)
    assert int(gt.counts.min()) > 0 and len(gt) > B * min(L, S)


def test_sparse_at_the_training_shape_holds_no_matrix():
    """B = 4, L = 7000, S = 4096: the bits of the dense path, and statistics -> loss -> backward ->
    fine supervision from the list peak below the size of even a one-byte [B, L, S] matrix."""
    B, L, S = 4, 7000, 4096
    a, b, gt, _ = cl.make_case("planted", B, L, S, seed=1)
    gt[torch.rand(gt.shape, generator=torch.Generator().manual_seed(2)) < 2e-4] = 1
    names, dense, sparse, sp = _dense_and_sparse(a, b, gt, None)
    _assert_bits(names, dense, sparse)
    del dense, sparse
    crit = losses.Loss(cl.LOSS_CONFIG)
    fa, fb = a.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    data = {"b_ids": sp.b_ids[::3].clone(), "i_ids": sp.i_ids[::3].clone(), "j_ids": sp.j_ids[::3].clone(),
            "q_hw_c": (64, 64), "gt_sparse": sp}
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    loss = crit.compute_coarse_loss(train_path.TrainConfHandle(CM, fa, fb, None), sp)
    loss.backward()
    train_gt.fine_supervision(data, otg.config())
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"training shape, sparse ground truth: G = {len(sp)}, peak above inputs {peak / 2**20:.1f} MiB "
          f"(int16 conf_matrix_gt {B * L * S * 2 / 2**20:.0f} MiB, fine_location_matrix_gt "
          f"{B * L * S * 8 / 2**20:.0f} MiB)")
    assert peak < B * L * S and data["expec_f_gt"].shape == (len(data["b_ids"]), 2)


@pytest.mark.parametrize("key", ["planted_300x192", "masked_300x192", "planted_130x150"])
def test_sparse_loss_matches_the_fp64_oracle(key):
    name, batch, rows, cols = cl.GOLDEN_CASES[key]
    a, b, gt, mask = cl.make_case(name, batch, rows, cols)
    fa, fb = a.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    h = train_path.TrainConfHandle(CM, fa, fb, mask.cuda() if mask is not None else None)
    loss, counts = losses.coarse_focal_loss(h, list_of(gt), *FOCAL, 1.0, 1.0)
    loss.backward()
    r_loss, r_da, r_db = cl.focal_loss_and_grads(a.cuda(), b.cuda(), gt.cuda(), cl.scale_of(),
                                                 mask.cuda() if mask is not None else None)
    assert counts.tolist() == [int((gt == 1).sum()), int((gt == 0).sum())]
    assert abs(loss.item() - r_loss.item()) <= RTOL * abs(r_loss.item())
    for got, ref in ((fa.grad, r_da), (fb.grad, r_db)):
        err = (got.double() - ref).abs()
        tol = RTOL * ref.abs() + 1e-6 + RTOL * float(ref.abs().max())
        assert bool((err <= tol).all()), f"max err / tol {float((err / tol).max()):.3f}"
    with pytest.raises(ValueError, match="shape"):
        losses.coarse_focal_loss(h, list_of(gt[:, :-1]), *FOCAL, 1.0, 1.0)


def _gpu_case(case, sparse):
    t = {k: torch.from_numpy(v).cuda() for k, v in case.items()}
    shape = tuple(int(n) for n in case["shape"])
    gt = SparseGT(t["b_ids"], t["i_ids"], t["j_ids"], t["fine_xy"], shape).check()
    data = {"b_ids": t["m_b"], "i_ids": t["m_i"], "j_ids": t["m_j"], "q_hw_c": tuple(int(n) for n in case["hw_c"])}
    if sparse:
        data["gt_sparse"] = gt
    else:
        data["fine_location_matrix_gt"] = gt.to_dense()[1]
    if "scale" in case:
        data["query_image_scale"] = t["scale"]
    return data


@pytest.mark.parametrize("window", [5, 7])
@pytest.mark.parametrize("name", list(mtg.CASES))
def test_fine_supervision_kernel(name, window):
    z = np.load(os.path.join(golden_io.GOLDEN_DIR, "reference", "train_gt.npz"))
    case = {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "_")}
    ref = case.pop("expec_f_gt")
    by_kernel, by_torch = _gpu_case(case, True), _gpu_case(case, False)
    train_gt.fine_supervision(by_kernel, otg.config(window))
    train_gt.fine_supervision(by_torch, otg.config(window))       # the reference formula, by PyTorch on the device
    got = by_kernel["expec_f_gt"]
    assert got.dtype == torch.float32 and got.shape == (len(case["m_b"]), 2)
    assert torch.equal(got, by_torch["expec_f_gt"])
    if window == 5:
        assert float(np.abs(got.cpu().numpy() - ref).max()) <= 1e-6
        absent = torch.from_numpy(otg.lookup((case["b_ids"], case["i_ids"], case["j_ids"], case["fine_xy"]),
                                             (case["m_b"], case["m_i"], case["m_j"]), case["shape"])[:, 0] == -50)
        assert 0 < int(absent.sum()) and bool((got.cpu()[absent].abs().max(1).values > 1).all())
    for k in ("b_ids", "i_ids", "j_ids"):
        by_kernel[k] = by_kernel[k][:0]
    train_gt.fine_supervision(by_kernel, otg.config(window))
    assert by_kernel["expec_f_gt"].shape == (0, 2)


def test_training_step_with_the_list_equals_the_dense_step():
    """model.train() + fine_supervision + Loss, lazy mode, the list against the two dense tensors under
    one seed: the same matches, the same expec_f_gt and loss bits; and on ONE forward the coarse loss and
    its gradients by both routes (two forwards differ in the last bits of their cuDNN convolutions)."""
    sd = workload.synthetic_state_dict(0)
    cfg = otg.config()
    conf = mrg.train_batch(sd, True)["conf_matrix_gt"]
    gt = planted_gt(conf)
    dense_bytes = conf.numel() * conf.element_size() + conf.numel() * 2 * 4
    runs, peaks = {}, {}
    for mode in ("dense", "sparse"):
        m = OnePosePlus_model(mrg.train_config())
        m.load_state_dict(sd, strict=True)
        m = m.cuda().train()
        m.conf_matrix_mode = "lazy"
        data = mrg.train_batch(sd, True)
        if mode == "sparse":
            del data["conf_matrix_gt"]
            data["gt_sparse"] = gt
        else:
            data["fine_location_matrix_gt"] = gt.to_dense()[1]
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()      # the model; the first run's tensors in the second
        data = {k: (v.to("cuda") if torch.is_tensor(v) or isinstance(v, SparseGT) else v) for k, v in data.items()}
        torch.manual_seed(11)
        m(data)
        train_gt.fine_supervision(data, cfg)
        losses.Loss(cl.LOSS_CONFIG).train()(data)
        m.zero_grad()
        data["loss"].backward(retain_graph=True)
        torch.cuda.synchronize()
        peaks[mode] = torch.cuda.max_memory_allocated() - base
        runs[mode] = (m, data)
    (_, dd), (ms, ds) = runs["dense"], runs["sparse"]
    assert isinstance(ds["conf_matrix"], train_path.TrainConfHandle) and "conf_matrix_gt" not in ds
    for k in ("b_ids", "i_ids", "j_ids", "gt_mask", "m_bids", "expec_f_gt"):
        assert torch.equal(dd[k], ds[k]), k
    correct = ds["expec_f_gt"].abs().max(1).values < 1
    assert 0 < int(correct.sum()) < len(correct)
    assert abs(ds["loss"].item() - dd["loss"].item()) <= 1e-5 * abs(dd["loss"].item())
    print(f"peak of the step: dense {peaks['dense'] / 2**20:.2f} MiB, sparse {peaks['sparse'] / 2**20:.2f} MiB, "
          f"the two dense tensors {dense_bytes / 2**20:.2f} MiB")
    # the list and its index (a few KiB) replace the two tensors
    assert peaks["dense"] - peaks["sparse"] >= dense_bytes - 64 * 1024
    # one forward (the sparse run's handle), the coarse loss by both routes
    h = ds["conf_matrix"]
    crit = losses.Loss(cl.LOSS_CONFIG).train()
    params = [p for p in ms.parameters() if p.requires_grad]
    out = []
    for g in (gt.to("cuda"), gt.to("cuda").to_dense()[0]):
        loss = crit.compute_coarse_loss(h, g)
        grads = torch.autograd.grad(loss, [h.feat3d, h.feat2d] + params, retain_graph=True, allow_unused=True)
        out.append((loss.detach(), grads))
    (l_s, g_s), (l_d, g_d) = out
    assert torch.equal(l_s, l_d) and torch.equal(g_s[0], g_d[0]) and torch.equal(g_s[1], g_d[1])
    used = 0
    for a, b in zip(g_s[2:], g_d[2:]):
        assert (a is None) == (b is None)
        if a is not None:
            used += 1
            # identical dA / dB enter the same PyTorch backward, whose cuDNN weight gradients and
            # atomics-based kernels are not bit-reproducible from one call to the next (2e-4 of absmax seen)
            assert torch.allclose(a, b, rtol=0, atol=1e-3 * float(b.abs().max()) + 1e-12)
    assert used > 50
    with pytest.raises(ValueError, match="both"):
        losses.Loss(cl.LOSS_CONFIG)({**ds, "conf_matrix_gt": conf.cuda()})
