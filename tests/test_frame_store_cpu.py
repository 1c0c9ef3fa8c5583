"""CPU: the host side of the device frame store (dataset.FrameLoader / FrameStore): mask packing, when the store is
not built, the host path's equality with torch's DataLoader, and the device path's batching and global-RNG use with
the decode replaced by a fake."""
import os
import pickle
import random
import types

import numpy as np
import pytest
import torch

from helpers import dropin


def _write(root, frames=5, H=7, W=37, normals=True, seed=0):
    dropin()
    from dataset import write_sequence
    g = torch.Generator().manual_seed(seed)
    imgs = torch.rand(frames, H, W, 3, generator=g) * 2 - 1
    masks = (torch.rand(frames, H, W, generator=g) > 0.5).float()
    nrm = torch.nn.functional.normalize(torch.randn(frames, H, W, 3, generator=g), dim=-1) if normals else None
    cam = dict(fx=float(W), fy=float(W), cx=W / 2.0, cy=H / 2.0, quat=[0., 0., 0., 1.], T=[0., 0., 2.5])
    write_sequence(root, imgs.numpy(), masks.numpy(), np.zeros((frames, 24, 3), np.float32),
                   np.zeros((frames, 3), np.float32), np.zeros(10, np.float32), cam,
                   normals=None if nrm is None else nrm.numpy())
    return root


def _unpack(words, W):
    bits = np.unpackbits(words.view(np.uint8).reshape(words.shape[0], -1), axis=-1, bitorder='little')
    return bits, bits[:, :W]


def test_pack_mask_bit_order_and_padding():
    dropin()
    from dataset import pack_mask
    W = 70                                         # three words per row, the last one holding 6 columns
    m = np.zeros((3, W), np.uint8)
    m[0, 0] = m[0, 31] = m[0, 32] = m[1, 69] = m[2, 33] = 255
    w = pack_mask(m)
    assert w.dtype == np.int32 and w.shape == (3, 3)
    u = w.view(np.uint32)
    assert u[0, 0] == (1 | (1 << 31)) and u[0, 1] == 1 and u[0, 2] == 0
    assert u[1, 2] == 1 << (69 - 64) and u[2, 1] == 1 << 1
    rng = np.random.default_rng(0)
    for W in (1, 31, 32, 33, 53, 64, 1080):
        fg = rng.random((4, W)) > 0.5
        bits, cols = _unpack(pack_mask(fg.astype(np.uint8) * 255), W)
        assert bits.shape[1] == (W + 31) // 32 * 32
        assert np.array_equal(cols.astype(bool), fg) and not bits[:, W:].any()   # row padding stays 0


def test_pack_mask_any_channel(tmp_path):
    """A mask file where only some channels are nonzero: foreground exactly where SceneDataset.__getitem__ sees it."""
    import cv2
    root = _write(str(tmp_path / "seq"), frames=2)
    rng = np.random.default_rng(1)
    m = np.zeros((7, 37, 3), np.uint8)
    for c in range(3):
        m[..., c] = (rng.random((7, 37)) > 0.8) * rng.integers(1, 256, (7, 37))
    m[0, :4] = 0
    assert ((m > 0).sum(-1) == 1).any()
    cv2.imwrite(os.path.join(root, "masks", "000001.png"), m)
    from dataset import SceneDataset, pack_mask
    ds = SceneDataset(root)
    ref = ds[1][1]['mask'].numpy().astype(bool)
    _, cols = _unpack(pack_mask(cv2.imread(ds.mask_ns[1])), 37)
    assert np.array_equal(cols.astype(bool), ref) and ref.any() and not ref.all()


def test_partial_normals_select_host_path(tmp_path, capsys):
    root = _write(str(tmp_path / "seq"), frames=4)
    os.remove(os.path.join(root, "normals", "000002.png"))
    from dataset import SceneDataset, frame_store
    from dataset.dataset import _host_path_reason
    ds = SceneDataset(root)
    assert _host_path_reason(ds, torch.device("cuda:0")) == "normals exist for 3 of 4 frames"
    ds.store_device = torch.device("cuda:0")
    assert frame_store(ds) is None and frame_store(ds) is None
    out = capsys.readouterr().out
    assert out.count("frames stay on the host: normals exist for 3 of 4 frames") == 1
    ds.store_device = torch.device("cpu")
    assert _host_path_reason(ds, ds.store_device) == "device cpu is not CUDA"
    ds2 = SceneDataset(root)
    assert frame_store(ds2) is None and "frame store" not in capsys.readouterr().out   # no device recorded: silent


def _run_epoch(loader, draws=True):
    """Ids and outs of one epoch, with a ray-subsampling draw after each batch as OptimNetwork.forward makes."""
    out = []
    for ids, outs in loader:
        out.append((ids, outs))
        if draws:
            torch.rand(3)
    return out


def test_host_path_equals_dataloader(tmp_path):
    root = _write(str(tmp_path / "seq"), frames=5)
    from dataset import FrameLoader, RandomSampler, SceneDataset
    ds = SceneDataset(root)
    res = []
    for make in (lambda s: FrameLoader(ds, 2, sampler=s, num_workers=0),
                 lambda s: torch.utils.data.DataLoader(ds, 2, sampler=s, num_workers=0)):
        torch.manual_seed(3)
        random.seed(4)
        loader = make(RandomSampler(ds, 1, True))
        assert len(loader) == 3
        res.append(_run_epoch(loader) + _run_epoch(loader))
    a, b = res
    assert len(a) == len(b) == 6
    for (ia, oa), (ib, ob) in zip(a, b):
        assert ia.dtype == torch.int64 and torch.equal(ia, ib) and set(oa) == set(ob) == {'img', 'mask', 'normal'}
        for k in oa:
            assert torch.equal(oa[k], ob[k]), k


class _Ids(torch.utils.data.Dataset):
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        return i, {'x': torch.zeros(1)}


class _FakeStore:
    def __init__(self):
        self.calls = []

    def decode(self, ids):
        self.calls.append(list(ids))
        return {'ids': torch.tensor(ids)}


def _samplers():
    dropin()
    from dataset import ClipSampler, RandomSampler, ShardedSampler
    return [("random-shuffle", lambda d: RandomSampler(d, 1, True)),
            ("random-ordered", lambda d: RandomSampler(d, 1, False)),
            ("random-every-3rd", lambda d: RandomSampler(d, 3, True)),
            ("clip", lambda d: ClipSampler(d, 4, True)),
            ("sharded-r1of3", lambda d: ShardedSampler(d, 1, 3, True)),
            ("sharded-r0of2-ordered", lambda d: ShardedSampler(d, 0, 2, False))]


@pytest.mark.parametrize("name", [n for n, _ in _samplers()])
@pytest.mark.parametrize("bs", [1, 3, 4])
def test_device_path_batches_and_rng_match_dataloader(name, bs, monkeypatch):
    import dataset.dataset as D
    make = dict(_samplers())[name]
    data = _Ids(13)
    fake = _FakeStore()
    monkeypatch.setattr(D, "frame_store", lambda ds: fake)
    res = {}
    for kind in ("store", "dataloader"):
        torch.manual_seed(11)
        random.seed(12)
        sampler = make(data)
        loader = (D.FrameLoader(data, bs, sampler=sampler, num_workers=0) if kind == "store" else
                  torch.utils.data.DataLoader(data, bs, sampler=sampler, num_workers=0))
        epochs = []
        for ep in range(2):
            if hasattr(sampler, "set_epoch"):
                sampler.set_epoch(ep)
            epochs.append([ids.tolist() for ids, _ in _run_epoch(loader)])
        res[kind] = (epochs, torch.get_rng_state(), random.getstate(), len(loader))
    (ea, ra, pa, la), (eb, rb, pb, lb) = res["store"], res["dataloader"]
    assert ea == eb and la == lb and torch.equal(ra, rb) and pa == pb
    assert fake.calls == [b for e in ea for b in e]          # one decode per batch, with the batch's ids
    assert all(len(b) == bs for e in ea for b in e[:-1])


def test_sharded_ids_per_rank_unchanged(monkeypatch):
    """Every rank's loader yields its ShardedSampler stream: positions r, r+W, ... of one seeded permutation."""
    import dataset.dataset as D
    from dataset import ShardedSampler
    monkeypatch.setattr(D, "frame_store", lambda ds: _FakeStore())
    data, world = _Ids(10), 4
    perm = torch.randperm(10, generator=torch.Generator().manual_seed(0 + 1)).tolist()
    perm = perm + perm[:2]
    seen = []
    for rank in range(world):
        s = ShardedSampler(data, rank, world, True)
        s.set_epoch(1)
        ids = [i for b, _ in D.FrameLoader(data, 2, sampler=s) for i in b.tolist()]
        assert ids == perm[rank::world] == list(s)
        seen += ids
    assert sorted(set(seen)) == list(range(10))


def test_set_hierarchical_config_keeps_frame_loader(tmp_path):
    root = _write(str(tmp_path / "seq"), frames=3)
    import utils
    from dataset import FrameLoader, getDatasetAndLoader
    from selfreconcode_b200 import synth
    conf = synth.reference_config()
    ds, loader = getDatasetAndLoader(root, {}, 1, True, 0, False, False, False)
    assert isinstance(loader, FrameLoader) and loader.dataset is ds and loader.num_workers == 0
    net = types.SimpleNamespace(engine=types.SimpleNamespace(b_min=torch.tensor([-1., -1., -1.]),
                                                             b_max=torch.tensor([1., 1., 1.])))
    for level in ('coarse', 'medium', 'fine'):
        net, new = utils.set_hierarchical_config(conf, level, net, loader, [(9, 13, 5), (17, 25, 9)])
        assert isinstance(new, FrameLoader) and new.sampler is loader.sampler and new.dataset is ds
        assert new.batch_size == conf.get_int('train.%s.point_render.batch_size' % level)
        assert len(new) == -(-len(loader.sampler) // new.batch_size)


def test_store_is_not_pickled(tmp_path):
    root = _write(str(tmp_path / "seq"), frames=2)
    from dataset import SceneDataset
    ds = SceneDataset(root)
    ds._frame_store = lambda: None        # unpicklable stand-in: pickling must not reach it
    back = pickle.loads(pickle.dumps(ds))
    assert not hasattr(back, '_frame_store') and back.frame_num == 2 and hasattr(ds, '_frame_store')
