"""Sparse ground truth of training on the host: the SparseGT type and its dataset side, the
ground-truth padding drawn from the list, fine_supervision against the reference's own function (live
and stored), and the eager loss on the CPU with the list."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import coarse_loss as cl
from oracle import make_reference_golden as mrg
from oracle import make_train_gt_golden as mtg
from oracle import ref_shims, workload
from oracle import train_gt as otg
from onepose_plus_plus_b200 import OnePosePlus_model, SparseGT, losses, train_gt, train_path
from tests import golden_io

needs_ref = pytest.mark.skipif(not ref_shims.available(), reason="needs the reference tree")


def planted_gt(conf_gt, wc=16, seed=4):
    """The fine locations the planted train batch lacks: cell origin * 8 + a seeded offset in
    [-6, 10) px, so that some fall outside the fine window.  -> (SparseGT, dense fine matrix)"""
    b, i, j = torch.where(conf_gt)
    g = torch.Generator().manual_seed(seed)
    xy = torch.stack([j % wc, j // wc], 1).float() * 8 + torch.rand(len(b), 2, generator=g) * 16 - 6
    fine = torch.full(tuple(conf_gt.shape) + (2,), -50.0)
    fine[b, i, j] = xy
    return SparseGT(b, i, j, xy, conf_gt.shape), fine


@pytest.fixture(scope="module")
def planted():
    sd = workload.synthetic_state_dict(0)
    data = mrg.train_batch(sd, False)
    gt, fine = planted_gt(data["conf_matrix_gt"])
    return sd, data, gt, fine


def test_round_trip_and_order(planted):
    _, data, gt, fine = planted
    conf = data["conf_matrix_gt"]
    again = SparseGT.from_dense(conf, fine)
    for a, b in zip((gt.b_ids, gt.i_ids, gt.j_ids, gt.fine_xy), (again.b_ids, again.i_ids, again.j_ids, again.fine_xy)):
        assert torch.equal(a, b)
    assert all(torch.equal(a, b) for a, b in zip((gt.b_ids, gt.i_ids, gt.j_ids), torch.where(conf)))
    d_conf, d_fine = gt.to_dense()
    assert d_conf.dtype == torch.int16 and torch.equal(d_conf.bool(), conf)
    assert d_fine.dtype == torch.float32 and torch.equal(d_fine, fine)
    assert float(d_fine[~conf].max()) == -50.0 == float(d_fine[~conf].min())
    assert len(gt) == int(conf.sum()) and gt.counts.tolist() == conf.sum((1, 2)).tolist()
    assert gt.nbytes() == len(gt) * 32 and gt.to("cpu").shape == gt.shape
    with pytest.raises(ValueError, match="0 or 1"):
        SparseGT.from_dense(conf.to(torch.int16) * 2, fine)


def test_constructor_validates_cpu_lists():
    i64 = torch.int64
    b, i, j = torch.tensor([0, 0, 1]), torch.tensor([3, 5, 0]), torch.tensor([7, 2, 9])
    xy = torch.zeros(3, 2)
    SparseGT(b, i, j, xy, (2, 6, 10))
    SparseGT(*(torch.empty(0, dtype=i64) for _ in range(3)), torch.empty(0, 2), (2, 6, 10))
    with pytest.raises(ValueError, match="ascending"):
        SparseGT(b, torch.tensor([5, 3, 0]), j, xy, (2, 6, 10))                     # unsorted
    with pytest.raises(ValueError, match="ascending"):
        SparseGT(b, torch.tensor([3, 3, 0]), torch.tensor([7, 7, 9]), xy, (2, 6, 10))   # duplicate
    for shape in ((1, 6, 10), (2, 5, 10), (2, 6, 9)):
        with pytest.raises(ValueError, match="outside"):
            SparseGT(b, i, j, xy, shape)
    with pytest.raises(ValueError, match="outside"):
        SparseGT(b, torch.tensor([-1, 5, 0]), j, xy, (2, 6, 10))
    with pytest.raises(ValueError):
        SparseGT(b.int(), i, j, xy, (2, 6, 10))
    with pytest.raises(ValueError):
        SparseGT(b, i, j, xy.double(), (2, 6, 10))
    with pytest.raises(ValueError):
        SparseGT(b, i, j, torch.zeros(2, 2), (2, 6, 10))


def test_sample_filters_sorts_and_collates():
    L, S = 50, 40
    # a 3D point >= shape3d, a cell index > S, one (i, j) written twice (the later location stays), unsorted input
    i = torch.tensor([9, 60, 3, 9, 3, 20])
    j = torch.tensor([5, 1, 30, 5, 2, 41])
    xy = torch.arange(12.0).view(6, 2)
    s = train_gt.sparse_gt_sample(i, j, xy, L, S)
    assert s["i_ids"].tolist() == [3, 3, 9] and s["j_ids"].tolist() == [2, 30, 5] and s["shape"] == (L, S)
    assert s["fine_xy"].tolist() == [[8.0, 9.0], [4.0, 5.0], [6.0, 7.0]]
    with pytest.raises(ValueError, match="outside"):     # j == S passes the reference's `j > S` filter and
        train_gt.sparse_gt_sample(i, torch.tensor([5, 1, 30, 5, 2, 40]), xy, L, S)   # then indexes past its matrix
    empty = train_gt.sparse_gt_sample(torch.empty(0), torch.empty(0), torch.empty(0, 2), L, S)
    other = train_gt.sparse_gt_sample([1], [0], [[1.5, 2.5]], L, S)
    gt = train_gt.collate_sparse_gt([s, empty, other])
    assert gt.shape == (3, L, S) and gt.b_ids.tolist() == [0, 0, 0, 2] and gt.counts.tolist() == [3, 0, 1]
    assert gt.i_ids.tolist() == [3, 3, 9, 1] and gt.fine_xy[-1].tolist() == [1.5, 2.5]
    with pytest.raises(ValueError, match="shapes"):
        train_gt.collate_sparse_gt([s, train_gt.sparse_gt_sample([1], [0], [[0.0, 0.0]], L, S + 1)])


def test_dataset_wrapper_drops_the_dense_keys(planted):
    _, data, gt, fine = planted
    conf = data["conf_matrix_gt"]

    class Items(torch.utils.data.Dataset):
        def __len__(self):
            return 2

        def __getitem__(self, k):
            return {"conf_matrix_gt": conf[k].to(torch.int16), "fine_location_matrix_gt": fine[k],
                    "query_image": torch.full((1, 8, 8), float(k))}

    ds = train_gt.SparseGTDataset(Items())
    assert len(ds) == 2 and set(ds[0]) == {"query_image", "gt_sparse"}
    loader = torch.utils.data.DataLoader(ds, batch_size=2, collate_fn=train_gt.collate)
    batch = next(iter(loader))
    assert set(batch) == {"query_image", "gt_sparse"} and batch["query_image"].shape == (2, 1, 8, 8)
    got = batch["gt_sparse"]
    assert got.shape == gt.shape
    for a, b in zip((got.b_ids, got.i_ids, got.j_ids, got.fine_xy), (gt.b_ids, gt.i_ids, gt.j_ids, gt.fine_xy)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("n_pred", [10, 3000])     # n_pred <= n_max - pad_min, and above
def test_padding_draws_the_same_matches(planted, n_pred):
    sd, data, gt, _ = planted
    cm = types.SimpleNamespace(config=mrg.train_config()["coarse_matching"])
    B, L, S = gt.shape
    g = torch.Generator().manual_seed(n_pred)
    pred = (torch.randint(0, B, (n_pred,), generator=g), torch.randint(0, L, (n_pred,), generator=g),
            torch.randint(0, S, (n_pred,), generator=g), torch.rand(n_pred, generator=g) + 0.1)
    base = {"q_hw_c": (12, 16), "q_hw_i": (96, 128), "keypoints3d": data["keypoints3d"]}
    outs, states = [], []
    for extra in ({"conf_matrix_gt": data["conf_matrix_gt"]}, {"gt_sparse": gt}):
        torch.manual_seed(5)
        outs.append(train_path._pad_matches(cm, *pred, (B, L, S), {**base, **extra}, True))
        states.append(torch.get_rng_state())
    assert torch.equal(states[0], states[1])
    for k in ("b_ids", "i_ids", "j_ids", "gt_mask", "m_bids", "mconf", "mkpts_query_c"):
        assert torch.equal(outs[0][k], outs[1][k]), k
    assert int(outs[0]["gt_mask"].sum()) >= 20
    with pytest.raises(ValueError, match="both"):
        train_path._pad_matches(cm, *pred, (B, L, S), {**base, "gt_sparse": gt,
                                                      "conf_matrix_gt": data["conf_matrix_gt"]}, True)
    with pytest.raises(ValueError, match="shape"):
        train_path._pad_matches(cm, *pred, (B, L + 1, S), {**base, "gt_sparse": gt}, True)
    none = SparseGT(*(torch.empty(0, dtype=torch.int64) for _ in range(3)), torch.empty(0, 2), gt.shape)
    with pytest.raises(AssertionError):
        train_path._pad_matches(cm, *pred, (B, L, S), {**base, "gt_sparse": none}, True)


def _case_data(case, sparse):
    t = {k: torch.from_numpy(v) for k, v in case.items()}
    shape = tuple(int(n) for n in case["shape"])
    gt = SparseGT(t["b_ids"], t["i_ids"], t["j_ids"], t["fine_xy"], shape)
    data = {"b_ids": t["m_b"], "i_ids": t["m_i"], "j_ids": t["m_j"], "q_hw_c": tuple(int(n) for n in case["hw_c"])}
    if sparse:
        data["gt_sparse"] = gt
    else:
        data["fine_location_matrix_gt"] = gt.to_dense()[1]
    if "scale" in case:
        data["query_image_scale"] = t["scale"]
    return data, gt


@needs_ref
@pytest.mark.parametrize("with_scale", [False, True])
@pytest.mark.parametrize("window", [5, 7])
def test_fine_supervision_matches_the_live_reference(with_scale, window):
    """with and without query_image_scale (non-square), matches that are not ground truth"""
    case = otg.make_case(seed=3, with_scale=with_scale)
    ref = mtg.reference_expec(case, window)
    hit = otg.lookup((case["b_ids"], case["i_ids"], case["j_ids"], case["fine_xy"]),
                     (case["m_b"], case["m_i"], case["m_j"]), case["shape"])[:, 0] != -50
    assert 0 < int(hit.sum()) < len(hit)                     # some predictions are absent from the list
    assert float(np.abs(ref[~hit]).min()) > 1.0              # and land outside the window
    if with_scale:      # (without it the reference takes the fine scale for the coarse one: nothing is inside)
        assert 0 < int((np.abs(ref[hit]).max(1) < 1).sum()) < int(hit.sum())
    ora = otg.fine_supervision((case["b_ids"], case["i_ids"], case["j_ids"], case["fine_xy"]),
                               (case["m_b"], case["m_i"], case["m_j"]), case["shape"], int(case["hw_c"][1]), window,
                               case.get("scale"))
    assert np.array_equal(ora, ref)
    for sparse in (True, False):
        data, _ = _case_data(case, sparse)
        train_gt.fine_supervision(data, otg.config(window))
        assert data["expec_f_gt"].dtype == torch.float32 and np.array_equal(data["expec_f_gt"].numpy(), ref)


@pytest.mark.parametrize("name", list(mtg.CASES))
def test_fine_supervision_matches_the_stored_reference(name):
    z = np.load(os.path.join(golden_io.GOLDEN_DIR, "reference", "train_gt.npz"))
    case = {k[len(name) + 1:]: z[k] for k in z.files if k.startswith(name + "_")}
    ref = case.pop("expec_f_gt")
    made = otg.make_case(**mtg.CASES[name])
    assert all(np.array_equal(made[k], case[k]) for k in made)     # the stored inputs are the seeded ones
    data, _ = _case_data(case, True)
    train_gt.fine_supervision(data, otg.config())
    assert np.array_equal(data["expec_f_gt"].numpy(), ref)
    data["b_ids"] = data["b_ids"][:0]
    data["i_ids"], data["j_ids"] = data["i_ids"][:0], data["j_ids"][:0]
    train_gt.fine_supervision(data, otg.config())
    assert data["expec_f_gt"].shape == (0, 2)


@needs_ref
def test_assign_list_matches_the_reference_dataset():
    """build_assignmatrix live: a 3D point >= shape3d, two keypoints in one cell for one 3D point
    (duplicate), several cells per 3D point, a cell index beyond the grid, non-square image scale."""
    shape3d, hc, wc = 40, 6, 8
    scale = torch.tensor([1.5, 0.75])                  # (h, w)
    g = torch.Generator().manual_seed(0)
    n2d = 30
    cells = torch.stack([torch.randint(0, wc, (n2d,), generator=g), torch.randint(0, hc, (n2d,), generator=g)], 1)
    kc = cells.float() * 8 * scale[[1, 0]]
    kf = kc + torch.rand(n2d, 2, generator=g) * 8 - 4
    am = torch.stack([torch.arange(n2d), torch.randint(0, 55, (n2d,), generator=g)])
    am[1, 4], am[1, 5] = 7, 7                          # one 3D point, two cells
    kc[6], am[1, 6] = kc[4], 7                         # ... and the first cell again: a duplicate (i, j)
    kc[9] = torch.tensor([0.0, (hc + 1) * 8 * 1.5])    # j = (hc + 1) * wc > S: dropped
    assert bool((am[1] >= shape3d).any())
    conf, fine = otg.reference_build_assignmatrix(kc, kf, am, shape3d, hc * wc, wc, scale, 1 / 8)
    i, j, xy = otg.assign_list(kc.numpy(), kf.numpy(), am.numpy(), shape3d, hc * wc, wc, scale.numpy(), 1 / 8)
    ri, rj = torch.where(conf)
    assert np.array_equal(i, ri.numpy()) and np.array_equal(j, rj.numpy())
    assert np.array_equal(xy, fine[ri, rj].numpy()) and len(i) < n2d - 2
    # the dataset-side constructor from the raw correspondences (before the filters)
    keep = am[1] < shape3d
    cell = (kc[am[0][keep]] / scale[[1, 0]] * (1 / 8)).round()
    s = train_gt.sparse_gt_sample(am[1][keep], (cell[:, 1] * wc + cell[:, 0]).long(), kf[am[0][keep]], shape3d, hc * wc)
    assert np.array_equal(s["i_ids"].numpy(), i) and np.array_equal(s["j_ids"].numpy(), j)
    assert np.array_equal(s["fine_xy"].numpy(), xy)
    gt = train_gt.collate_sparse_gt([s])
    d_conf, d_fine = gt.to_dense()
    assert torch.equal(d_conf[0], conf) and torch.equal(d_fine[0], fine)


def test_eager_cpu_step_with_the_list_equals_the_dense_step(planted):
    sd, _, gt, fine = planted
    cfg = otg.config()
    runs = []
    torch.set_num_threads(mrg.TRAIN_THREADS)
    for sparse in (False, True):
        m = OnePosePlus_model(mrg.train_config())
        m.load_state_dict(sd, strict=True)
        m.train()
        data = mrg.train_batch(sd, False)
        if sparse:
            del data["conf_matrix_gt"]
            data["gt_sparse"] = gt
        else:
            data["fine_location_matrix_gt"] = fine
        torch.manual_seed(11)
        m(data)
        train_gt.fine_supervision(data, cfg)
        losses.Loss(cl.LOSS_CONFIG).train()(data)
        runs.append(data)
    dense, sp = runs
    for k in ("b_ids", "i_ids", "j_ids", "gt_mask", "m_bids", "expec_f_gt", "loss"):
        assert torch.equal(dense[k], sp[k]), k
    assert all(torch.equal(dense["loss_scalars"][k], sp["loss_scalars"][k]) for k in ("loss_c", "loss_f", "loss"))
    correct = dense["expec_f_gt"].abs().max(1).values < 1
    assert 0 < int(correct.sum()) < len(correct)
    with pytest.raises(ValueError, match="both"):
        losses.Loss(cl.LOSS_CONFIG)({**sp, "conf_matrix_gt": dense["conf_matrix_gt"]})
    with pytest.raises(TypeError, match="SparseGT"):
        train_gt.fine_supervision({**sp, "gt_sparse": (gt.b_ids, gt.i_ids, gt.j_ids)}, cfg)
