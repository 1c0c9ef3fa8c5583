"""GPU: the device frame store (csrc/frames.cu, dataset.FrameStore / FrameLoader) against SceneDataset.__getitem__
and torch's DataLoader: bit-identical batches, the same ids and global RNG state, the same training step."""
import ctypes
import os
import random
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, dropin

pytestmark = pytest.mark.gpu

# (frames, H, W, image file type): H*W odd (the per-pixel path of the kernel), H*W a multiple of 4 with W odd (16 B
# stores, groups that run across rows), and a full 1080x1920 frame
SEQS = {"37x53-png": (7, 37, 53, ".png"), "37x53-jpg": (7, 37, 53, ".jpg"), "36x53-png": (7, 36, 53, ".png"),
        "1080x1920": (4, 1080, 1920, ".png")}


@pytest.fixture(scope="module")
def seqs(tmp_path_factory):
    dropin()
    from selfreconcode_b200 import synth
    base = tmp_path_factory.mktemp("frames")
    return {k: synth.write_frame_sequence(str(base / k), F, H, W, seed=i, image_ext=ext)
            for i, (k, (F, H, W, ext)) in enumerate(SEQS.items())}


def _store(root, dev):
    from dataset import SceneDataset, frame_store
    ds = SceneDataset(root)
    ds.store_device = dev
    store = frame_store(ds)
    assert store is not None
    return ds, store


def _host(ds, i):
    _, o = ds[i]
    return {'img': o['img'], 'mask': o['mask'], 'normal': torch.from_numpy(o['normal'])}


@pytest.mark.parametrize("name", list(SEQS))
def test_decode_bit_identical_to_getitem(name, seqs, cuda_dev):
    ds, store = _store(seqs[name], cuda_dev)
    F, H, W = ds.frame_num, ds.H, ds.W
    assert store.nbytes() == F * H * (6 * W + 4 * ((W + 31) // 32))
    ref = [_host(ds, i) for i in range(F)]
    batches = [list(range(F)), [3, 0, 3, F - 1, 1, 1], [F - 1], []]
    for ids in batches:
        outs = store.decode(ids)
        assert set(outs) == {'img', 'mask', 'normal'}
        for k, v in outs.items():
            assert v.is_cuda and v.dtype == torch.float32 and v.shape[0] == len(ids)
            want = torch.stack([ref[i][k] for i in ids]) if ids else v.new_empty(v.shape).cpu()
            assert torch.equal(v.cpu(), want), (name, ids, k)
    a = store.decode([2, 0, 2])
    b = store.decode([2, 0, 2])
    assert all(torch.equal(a[k], b[k]) for k in a)          # reruns are bit-identical


def test_loader_ids_and_rng_match_workers(seqs, cuda_dev):
    from dataset import FrameLoader, RandomSampler, SceneDataset
    root = seqs["37x53-png"]
    runs = {}
    for kind in ("store", "workers"):
        torch.manual_seed(5)
        random.seed(6)
        if kind == "store":
            ds, _ = _store(root, cuda_dev)
            loader = FrameLoader(ds, 3, sampler=RandomSampler(ds, 1, True), num_workers=2)
        else:
            ds = SceneDataset(root)
            loader = torch.utils.data.DataLoader(ds, 3, sampler=RandomSampler(ds, 1, True), num_workers=2)
        got = []
        for _ in range(2):
            for ids, outs in loader:
                got.append((ids.tolist(), {k: v.cpu() for k, v in outs.items()}))
                assert (kind == "store") == outs['img'].is_cuda
                torch.rand(4)
        runs[kind] = (got, torch.get_rng_state(), random.getstate())
    (ga, ra, pa), (gb, rb, pb) = runs["store"], runs["workers"]
    assert [g[0] for g in ga] == [g[0] for g in gb] and len(ga) == 6
    assert torch.equal(ra, rb) and pa == pb
    for (_, oa), (_, ob) in zip(ga, gb):
        assert all(torch.equal(oa[k], ob[k]) for k in oa)


def test_errors(seqs, cuda_dev, tmp_path):
    from selfreconcode_b200 import _lib
    ds, store = _store(seqs["37x53-png"], cuda_dev)
    for bad in ([7], [-1], [0, 9]):
        with pytest.raises(ValueError, match="out of range"):
            store.decode(bad)
    lib = _lib.load()
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
    ids = torch.zeros(2, dtype=torch.int64, device=cuda_dev)
    out = torch.empty(2, 37, 53, 3, device=cuda_dev)
    msk = torch.empty(2, 37, 53, device=cuda_dev)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    F, H, W = 7, 37, 53

    def call(img_s, mask_s, nrm_s, F, H, W, N, img, mask, nrm):
        return lib.sr_frames_decode(p(img_s), p(mask_s), p(nrm_s), F, H, W, p(ids), N, p(img), p(mask), p(nrm), s)
    assert call(store.img, store.mask, store.normal, F, H, W, 2, out, msk, out) == _lib.SR_OK
    for args in ((0, H, W, 2), (F, 0, W, 2), (F, H, -3, 2), (F, H, W, -1)):
        assert call(store.img, store.mask, store.normal, *args, out, msk, None) == _lib.SR_EINVAL, args
    assert call(None, store.mask, store.normal, F, H, W, 2, out, None, None) == _lib.SR_EINVAL
    assert call(store.img, None, store.normal, F, H, W, 2, None, msk, None) == _lib.SR_EINVAL
    assert call(store.img, store.mask, None, F, H, W, 2, None, None, out) == _lib.SR_EINVAL
    assert call(None, None, None, F, H, W, 2, None, None, None) == _lib.SR_OK        # nothing asked for
    torch.cuda.synchronize()
    # a frame of another size than the sequence's
    import cv2
    from selfreconcode_b200 import synth
    root = synth.write_frame_sequence(str(tmp_path / "bad"), 3, 37, 53)
    bad = os.path.join(root, "imgs", "000001.png")
    cv2.imwrite(bad, np.zeros((53, 37, 3), np.uint8))
    from dataset import SceneDataset
    from dataset.dataset import build_frame_store
    with pytest.raises(ValueError, match="000001.png: 53x37"):
        build_frame_store(SceneDataset(root), cuda_dev)


def test_low_memory_selects_host_path(seqs, cuda_dev, monkeypatch, capsys):
    from dataset import FrameLoader, RandomSampler, SceneDataset
    root = seqs["36x53-png"]
    _, store = _store(root, cuda_dev)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (store.nbytes() * 2 - 1, 80 << 30))
    ds = SceneDataset(root)
    ds.store_device = cuda_dev
    loader = FrameLoader(ds, 4, sampler=RandomSampler(ds, 1, False), num_workers=0)
    got = list(loader)
    assert "frames stay on the host: the store needs" in capsys.readouterr().out
    assert getattr(ds, "_frame_store", None) is None and len(got) == 2
    for ids, outs in got:
        assert not outs['img'].is_cuda
        dec = store.decode(ids.tolist())
        assert all(torch.equal(dec[k].cpu(), outs[k]) for k in dec)


def _step_losses_and_grads(tr, datas):
    import bench
    torch.manual_seed(0)                    # the eikonal sample points of forward_rays are drawn from the global RNG
    net = tr["net"]
    for q in tr["params"]:
        q.grad = None
    loss = net.forward_rays(datas, tr["bi"], tr["ri"], tr["ci"], tr["init"].clone(), bench.RATIO, tr["fids"],
                            extra_points=tr["extra"])
    loss.backward()
    torch.cuda.synchronize()
    info = {k: float(v) for k, v in net.info.items() if k.endswith("_loss")}
    grads = torch.cat([(q.grad if q.grad is not None else torch.zeros_like(q)).reshape(-1).double()
                       for q in tr["params"]])
    return info, grads


def test_training_step_same_from_store_and_host(cuda_dev, tmp_path):
    """forward_rays + backward of the bench's synthetic training step with `datas` from the store and from the host
    path (the frames' ids 0..3 at 512x512): the same losses and gradients, within the spread of three host runs."""
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    dropin()
    import bench
    from dataset import SceneDataset
    from selfreconcode_b200 import synth
    sc = bench.build_scene(cuda_dev, 0)
    tr = bench.build_train(sc, cuda_dev, 0, 1)
    root = synth.write_frame_sequence(str(tmp_path / "train"), bench.TRAIN_FRAMES, 512, 512, seed=9)
    ds, store = _store(root, cuda_dev)
    fids = tr["fids"].tolist()
    host = {k: torch.stack([_host(ds, i)[k] for i in fids]) for k in ('img', 'mask', 'normal')}
    dev = store.decode(fids)
    assert all(torch.equal(dev[k].cpu(), host[k]) for k in host)
    hs = [_step_losses_and_grads(tr, host) for _ in range(3)]
    d1 = _step_losses_and_grads(tr, dev)
    spread_g = max(float((a[1] - b[1]).abs().max()) for a in hs for b in hs)
    spread_l = max(abs(a[0][k] - b[0][k]) for a in hs for b in hs for k in a[0])
    assert set(d1[0]) == set(hs[0][0]) and {'color_loss', 'normal_loss'} <= set(d1[0])
    assert min(float((d1[1] - h[1]).abs().max()) for h in hs) <= spread_g
    assert min(max(abs(d1[0][k] - h[0][k]) for k in h[0]) for h in hs) <= spread_l
    print("training step from the store vs the host path: max |d grad| %.3g (host-run spread %.3g), max |d loss| %.3g "
          "(spread %.3g)" % (min(float((d1[1] - h[1]).abs().max()) for h in hs), spread_g,
                             min(max(abs(d1[0][k] - h[0][k]) for k in h[0]) for h in hs), spread_l))
