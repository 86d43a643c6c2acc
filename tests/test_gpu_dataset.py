"""The data set feed on the GPU: cnb_extract_patches_indexed against convnet_b200_extract_patches on a physically permuted
chunk, the labels and targets it gathers, DataHandler with and without pipeline_loads, and a net trained from it."""
import numpy as np
import pytest
import torch

from convnet_b200 import lib, net
from convnet_b200.matrix import CUDAMatrix

pytestmark = pytest.mark.gpu


def _crop_reference(chunk, index, wo, ho, fl, C, W, H, pw, ph):
    """convnet_b200_extract_patches on chunk[:, index] (a copy permuted by torch): N x (C*pw*ph), column-major"""
    L = lib.load()
    N = index.numel()
    permuted = chunk[index.long()].contiguous()
    dev = lambda t, r, c: CUDAMatrix(r, c, storage=t.reshape(-1).contiguous())
    out = CUDAMatrix(N, C * pw * ph)
    out.storage.fill_(float("nan"))
    rc = L.convnet_b200_extract_patches(dev(permuted, C * W * H, N).p_mat, out.p_mat, dev(wo, 1, N).p_mat,
                                        dev(ho, 1, N).p_mat, dev(fl, 1, N).p_mat, W, H, pw, ph)
    assert rc == 0
    return out.storage


def _noise(N, W, H, pw, ph, view, mirror, g):
    if view is None:                                             # random jitter and mirror bits
        wo = torch.randint(0, W - pw + 1, (N,), generator=g).float()
        ho = torch.randint(0, H - ph + 1, (N,), generator=g).float()
        fl = torch.rand(N, generator=g)
    else:                                                        # one of the five fixed views, all mirrored or none
        w, h = net.view_offset(view, W - pw, H - ph)
        wo, ho, fl = torch.full((N,), float(w)), torch.full((N,), float(h)), torch.full((N,), float(mirror))
    return wo.cuda(), ho.cuda(), fl.cuda()


CASES = [(45, 3, 37, 29, 27, 21), (70, 1, 28, 28, 28, 28), (33, 3, 40, 40, 33, 35), (128, 3, 64, 64, 56, 56)]


@pytest.mark.parametrize("N,C,W,H,pw,ph", CASES)
@pytest.mark.parametrize("view,mirror", [(None, None)] + [(v, m) for v in range(5) for m in (0, 1)])
def test_indexed_crop_is_extract_patches_on_the_permuted_chunk(N, C, W, H, pw, ph, view, mirror):
    L = lib.load()
    g = torch.Generator().manual_seed(N * 31 + C + (view or 0) * 7 + (mirror or 0))
    chunk_n, F = N + 19, 5
    chunk = torch.randn(chunk_n, C, H, W, generator=g).cuda()
    index = torch.randperm(chunk_n, generator=g)[:N].to(torch.int32).cuda()
    labels = torch.randint(0, 1000, (chunk_n,), generator=g, dtype=torch.int32).cuda()
    targets = torch.randn(chunk_n, F, generator=g).cuda()
    wo, ho, fl = _noise(N, W, H, pw, ph, view, mirror, g)
    want = _crop_reference(chunk, index, wo, ho, fl, C, W, H, pw, ph)
    got = torch.full((N * C * pw * ph,), float("nan"), device="cuda")
    lab = torch.full((N,), -1, dtype=torch.int32, device="cuda")
    tgt = torch.full((N * F,), float("nan"), device="cuda")
    for with_labels in (True, False):
        rc = L.cnb_extract_patches_indexed(chunk.data_ptr(), got.data_ptr(), index.data_ptr(), wo.data_ptr(), ho.data_ptr(),
                                           fl.data_ptr(), N, C, W, H, pw, ph,
                                           labels.data_ptr() if with_labels else None, lab.data_ptr() if with_labels else None,
                                           None if with_labels else targets.data_ptr(), None if with_labels else tgt.data_ptr(),
                                           0 if with_labels else F)
        assert rc == 0
    torch.cuda.synchronize()
    assert torch.equal(got, want)                                # bit for bit, NaN canaries included
    assert torch.equal(lab, labels[index.long()])
    assert torch.equal(tgt.view(F, N), targets[index.long()].t())   # element n + N*j is feature j of image n


def test_indexed_crop_refuses_bad_arguments():
    L = lib.load()
    t = torch.zeros(64, device="cuda")
    p = t.data_ptr()
    assert L.cnb_extract_patches_indexed(p, p, p, p, p, p, 1, 1, 4, 4, 5, 4, None, None, None, None, 0) == -1  # crop > image
    assert L.cnb_extract_patches_indexed(p, p, p, p, p, p, 1, 1, 4, 4, 4, 4, p, None, None, None, 0) == -1    # half a pair
    assert L.cnb_extract_patches_indexed(p, p, p, p, p, p, 1, 1, 4, 4, 4, 4, None, None, p, p, 0) == -1       # no width


def _dataset(n, C, S, classes, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, C, S, S, generator=g).pin_memory(),
            torch.randint(0, classes, (n,), generator=g, dtype=torch.int32))


def _hand_crop(images, info, C, G):
    """the batch a DataHandler reported (data set rows, offsets, mirror bits) cropped by torch indexing, laid out like
    the input layer"""
    rows = torch.tensor(info["rows"])
    out = []
    for k, r in enumerate(rows.tolist()):
        y, x = int(info["height_offset"][k]), int(info["width_offset"][k])
        band = images[r, :, y:y + G, :]
        band = band.flip(-1) if info["flip"][k] > 0.5 else band      # the whole image mirrors, then the crop is cut
        out.append(band[..., x:x + G])
    return torch.stack(out).permute(1, 2, 3, 0).reshape(-1)          # (c, y, x, n): image fastest


def test_pipelined_and_unpipelined_batches_are_identical():
    C, S, G, batch, chunk = 8, 16, 12, 32, 96                    # "tiny" takes 8 x 12 x 12 inputs
    images, labels = _dataset(4 * chunk + 40, C, S, 10, 3)
    n = net.Net("tiny", batch, seed=1)
    common = dict(batch_size=batch, chunk_size=chunk, gpu_image_size=G, translate=True, flip=True, randomize_gpu=True,
                  randomize_cpu=True, random_access_chunk_size=8, max_reuse_count=1, multiplicity=2, seed=5)
    plain = net.DataHandler(images, labels, **common)
    piped = net.DataHandler(images, labels, pipeline_loads=True, **common)
    seen_loads = set()
    for step in range(60):                                       # several passes over several chunks
        if step == 37:
            plain.seek(50); piped.seek(50)
        batches = []
        for h in (plain, piped):
            h.get_batch(n)
            torch.cuda.synchronize()
            batches.append((n.input_tensor().clone(), n.labels_tensor().clone(), h.last_indices()))
        (x0, y0, i0), (x1, y1, i1) = batches
        if step < 37:                                            # a seek discards a preload: the orders part there
            assert i0 == i1
            assert torch.equal(x0, x1) and torch.equal(y0, y1)
        for x, y, info in batches:                               # and each is the crop of the rows it reports
            assert torch.equal(x.cpu(), _hand_crop(images, info, C, G))
            assert torch.equal(y.cpu(), labels[torch.tensor(info["rows"])])
        seen_loads.add(tuple(sorted(i0["rows"])))
    assert len(seen_loads) > 10
    plain.close(); piped.close(); n.close()


def test_targets_follow_the_images():
    C, S, G, batch = 8, 14, 12, 16
    images, _ = _dataset(80, C, S, 10, 4)
    n = net.Net("tiny+squared-error", batch, seed=1)
    F = n.targets_tensor().numel() // batch
    targets = torch.randn(80, F, generator=torch.Generator().manual_seed(9))
    h = net.DataHandler(images, targets=targets, batch_size=batch, chunk_size=48, gpu_image_size=G, translate=True,
                        randomize_gpu=True, pipeline_loads=True, seed=2)
    for _ in range(9):
        h.get_batch(n)
        torch.cuda.synchronize()
        rows = torch.tensor(h.last_indices()["rows"])
        assert torch.equal(n.targets_tensor().cpu().view(F, batch), targets[rows].t())
    with pytest.raises(ValueError, match="labels"):
        h.get_batch(net.Net("tiny", batch, seed=1))              # a net trained on labels, a data set without
    h.close(); n.close()


def test_lenet_trained_from_the_handler_matches_hand_feeding():
    batch, steps, S, G = 64, 20, 32, 28
    images, labels = _dataset(448, 1, S, 10, 6)
    fed, hand = net.Net("lenet", batch, seed=3), net.Net("lenet", batch, seed=3)
    h = net.DataHandler(images, labels, batch_size=batch, chunk_size=192, gpu_image_size=G, translate=True, flip=True,
                        randomize_gpu=True, randomize_cpu=True, random_access_chunk_size=16, pipeline_loads=True, seed=8)
    starts = []
    for _ in range(steps):
        h.get_batch(fed)
        info = h.last_indices()
        starts.append(info["start"])
        fed.train_step(want_loss=False)
        torch.cuda.synchronize()
        hand.input_tensor().copy_(_hand_crop(images, info, 1, G).cuda())
        hand.labels_tensor().copy_(labels[torch.tensor(info["rows"])].cuda())
        torch.cuda.synchronize()
        hand.train_step(want_loss=False)
    torch.cuda.synchronize()
    assert starts[:4] == [0, 64, 128, 0]                        # three batches per chunk of 192
    assert torch.equal(fed.params_tensor(), hand.params_tensor())
    assert torch.isfinite(fed.params_tensor()).all()
    h.close(); fed.close(); hand.close()


def test_from_model_takes_the_dataset_config(tmp_path):
    p = tmp_path / "ds.pbtxt"
    p.write_text(net.model_text("tiny").rstrip() + """
train_dataset {
  batch_size: 16 chunk_size: 32 randomize_gpu: true multiplicity: 2
  data_config { file_pattern: "x" layer_name: "input" can_translate: true gpu_image_size_y: 12 gpu_image_size_x: 12 }
}
""")
    images, labels = _dataset(64, 8, 14, 10, 1)
    n = net.Net(str(p), 16, seed=1)
    h = net.DataHandler.from_model(str(p), images, labels, net=n)
    h.get_batch(n)
    h.get_batch(n)
    info = h.last_indices()
    assert info["multiplicity_id"] == 1 and max(info["width_offset"]) <= 2
    with pytest.raises(ValueError, match="batch_size"):
        net.DataHandler.from_model(str(p), images, labels, net=net.Net(str(p), 8, seed=1))
    h.close(); n.close()
