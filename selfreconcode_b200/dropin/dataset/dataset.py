"""Sequence dataset of the reference (dataset/dataset.py:9-237): same on-disk layout, attribute names and
accessors, so `train.py` / `infer.py` and `utils.save_model` / `load_model` see what they expect.

    <root>/imgs/%06d.(png|jpg)   BGR uint8, mapped to [-1,1]           (dataset.py:86-88)
    <root>/masks/%06d.png        foreground = any channel > 0          (dataset.py:97-98)
    <root>/normals/%06d.png      optional; RGB -> [-1,1]               (dataset.py:99-103)
    <root>/smpl_rec.npz          poses [F,24,3], trans [F,3], shape [10], gender, vid_seg_indices (optional)
    <root>/camera.npz            fx, fy, cx, cy, quat [4], T [3]

Per-frame learnables (poses, trans, latent code tables) live here as leaf tensors, exactly like the
reference: the DataLoader only carries images, `get_grad_parameters(ids)` slices the leaves so gradients reach
them.  Additions for multi-GPU runs: `ShardedSampler` (one disjoint, equally long index stream per rank,
SURVEY.md section 8e) and pinned host staging of the frame tensors.

Once `getOptNet` has recorded the training device on the dataset, the loader of `getDatasetAndLoader` keeps the
whole sequence on that device in file form (`FrameStore`: 6.125 B per pixel) and decodes each batch there
(csrc/frames.cu), so a step reads no image file and copies no frame from the host.
"""
import os
import os.path as osp
import random
import time
from concurrent.futures import ThreadPoolExecutor
from glob import glob

import numpy as np
import torch

import utils


def _frame_id(path):
    return int(osp.basename(path).split('.')[0])


class SceneDataset(torch.utils.data.Dataset):
    def __init__(self, data_root, conds_lens={}, pin_memory=False):
        self.root = data_root
        self.pin_memory = bool(pin_memory) and torch.cuda.is_available()
        self.read_data()
        self.require_albedo = False
        self.conds, self.cond_ns = [], []
        for name, length in conds_lens.items():
            # latent codes start as smooth trajectories: random coefficients on the frame_num/5 lowest DCT modes
            k = max(self.frame_num // 5, 1)
            cond = (0.1 * torch.randn(length, k)).matmul(utils.DCTSpace(k, self.frame_num)).transpose(0, 1).contiguous()
            self.conds.append(cond.requires_grad_())
            self.cond_ns.append(name)

    def read_data(self):
        imgs = []
        for ext in ('.jpg', '.png'):
            imgs.extend(glob(osp.join(self.root, 'imgs/*' + ext)))
        imgs.sort(key=_frame_id)
        self.frame_num = len(imgs)
        self.img_ns = imgs
        self.mask_ns = []
        for i, name in enumerate(imgs):
            assert i == _frame_id(name), "frames must be numbered 0..F-1"
            m = osp.join(self.root, 'masks/%s.png' % osp.basename(name).split('.')[0])
            assert osp.isfile(m), m
            self.mask_ns.append(m)
        import cv2
        self.H, self.W, _ = cv2.imread(self.mask_ns[0]).shape
        d = np.load(osp.join(self.root, 'smpl_rec.npz'))
        self.poses = torch.from_numpy(d['poses'].astype(np.float32)).view(-1, 24, 3)
        self.trans = torch.from_numpy(d['trans'].astype(np.float32)).view(-1, 3)
        self.shape = torch.from_numpy(d['shape'].astype(np.float32)).view(-1)
        self.gender = str(d['gender']) if 'gender' in d else 'neutral'
        seg = d['vid_seg_indices'] if 'vid_seg_indices' in d else []
        self.video_segmented_index = list(np.asarray(seg).reshape(-1)[:-1].tolist()) if len(seg) else []
        c = np.load(osp.join(self.root, 'camera.npz'))
        f32 = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32).reshape(-1))
        self.camera_params = {'focal_length': f32([c['fx'], c['fy']]), 'princeple_points': f32([c['cx'], c['cy']]),
                              'cam2world_coord_quat': f32(c['quat']), 'world2cam_coord_trans': f32(c['T'])}

    def opt_camera_params(self, conf):
        keys = {'focal_length': 'focal_length', 'princeple_points': 'princeple_points',
                'cam2world_coord_quat': 'quat', 'world2cam_coord_trans': 'T'}
        for k, ck in keys.items():
            self.camera_params[k].requires_grad_(conf if isinstance(conf, bool) else conf.get_bool(ck))

    def learnable_weights(self):
        ws = [c for c in self.conds if c.requires_grad]
        ws += [v for v in self.camera_params.values() if v.requires_grad]
        ws += [v for v in (self.shape, self.poses, self.trans) if v.requires_grad]
        return ws

    def __len__(self):
        return self.frame_num

    def _stage(self, t):
        return t.pin_memory() if self.pin_memory else t

    def __getstate__(self):
        # DataLoader workers receive the dataset pickled: the device frame store stays in the main process
        state = self.__dict__.copy()
        state.pop('_frame_store', None)
        return state

    def __getitem__(self, idx):
        import cv2
        out = {}
        img = cv2.imread(self.img_ns[idx]).astype(np.float32)
        out['img'] = self._stage(torch.from_numpy((img / 255. - 0.5) * 2).view(self.H, self.W, 3))
        mask = torch.from_numpy(cv2.imread(self.mask_ns[idx])) > 0
        out['mask'] = self._stage(mask.view(self.H, self.W, -1).any(-1).float())
        nf = self.img_ns[idx].replace('/imgs/', '/normals/')[:-3] + 'png'
        if osp.isfile(nf):
            out['normal'] = 2. * cv2.imread(nf)[:, :, ::-1].astype(np.float32) / 255. - 1.
        if self.require_albedo:
            alb = cv2.imread(osp.join(self.root, 'albedos/%d.png' % idx)).astype(np.float32)
            out['albedo'] = torch.from_numpy((alb / 255. - 0.5) * 2.).view(self.H, self.W, 3)
        return idx, out

    # the DataLoader cannot carry tensors that require grad: sliced here instead (dataset.py:116-122)
    def get_grad_parameters(self, idxs, device):
        conds = [c[idxs].to(device) for c in self.conds]
        if len(conds) < 2:
            conds = conds + [None] * (2 - len(conds))
        return (self.poses[idxs].to(device), self.trans[idxs].to(device), *conds)

    def get_camera_parameters(self, N, device):
        cp = self.camera_params
        return (cp['focal_length'].to(device).view(1, 2).expand(N, 2), cp['princeple_points'].to(device).view(1, 2).expand(N, 2),
                utils.quat2mat(cp['cam2world_coord_quat'].to(device).view(1, 4)).expand(N, 3, 3),
                cp['world2cam_coord_trans'].to(device).view(1, 3).expand(N, 3), self.H, self.W)

    def get_batchframe_data(self, name, fids, batchsize):
        """[len(fids), batchsize, ...] windows of consecutive frames centred on each id, shifted to stay inside
        the video (or inside the id's segment when the sequence is two videos) -> (windows, position of the id in
        its window)  (dataset.py:128-191)."""
        data = getattr(self, name)
        assert data.shape[0] >= self.frame_num
        data = data[:self.frame_num].to(fids.device)
        cuts = [0] + [int(c) for c in self.video_segmented_index] + [self.frame_num]
        if len(cuts) > 3:
            raise NotImplementedError("more than two video segments")
        starts = torch.full_like(fids, -1)
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            assert batchsize < hi - lo
            sel = (fids >= lo) & (fids < hi)
            starts[sel] = (fids[sel] - batchsize // 2).clamp(min=lo, max=hi - batchsize)
        assert (starts >= 0).all().item()
        win = starts.view(-1, 1) + torch.arange(0, batchsize, device=fids.device).view(1, batchsize)
        return data[win], fids - starts


class ClipSampler(torch.utils.data.Sampler):
    """Whole clips of `clip_size` consecutive frames, clip order shuffled (dataset.py:195-215)."""

    def __init__(self, data_source, clip_size, shuffle):
        self.length, self.clip_size, self.shuffle = len(data_source), clip_size, shuffle
        self.n = self.length // clip_size
        if self.length == self.n * clip_size:
            self.n -= 1
        self.start = self.length - self.n * clip_size

    def __iter__(self):
        start = random.randrange(0, self.start + 1) if self.shuffle else 0
        out = torch.arange(start, start + self.n * self.clip_size).view(self.n, self.clip_size)
        if self.shuffle:
            out = out[torch.randperm(self.n)]
        return iter(out.view(-1).tolist())

    def __len__(self):
        return self.n * self.clip_size


class RandomSampler(torch.utils.data.Sampler):
    """Every `intersect`-th frame from a random phase, shuffled (dataset.py:217-237)."""

    def __init__(self, data_source, intersect, shuffle):
        self.length, self.intersect, self.shuffle = len(data_source), intersect, shuffle
        self.n = (self.length - 1) // intersect + 1
        self.start = self.length - intersect * (self.n - 1)

    def __iter__(self):
        if self.shuffle:
            index = torch.arange(random.randrange(0, self.start), self.length, self.intersect)
            index = index[torch.randperm(self.n)]
        else:
            index = torch.arange(0, self.length, self.intersect)
        assert index.numel() == self.n
        return iter(index.tolist())

    def __len__(self):
        return self.n


class ShardedSampler(torch.utils.data.Sampler):
    """Data-parallel split of an epoch (SURVEY.md section 8e): one shuffled permutation of the frames per epoch
    (same seed on every rank), padded to a multiple of the world size, rank r takes positions r, r+W, ...  All
    ranks get equally many frames, so per-frame means averaged across ranks equal the global mean."""

    def __init__(self, data_source, rank, world, shuffle=True, seed=0):
        self.length, self.rank, self.world, self.shuffle, self.seed = len(data_source), rank, world, shuffle, seed
        self.epoch = 0
        self.n = (self.length + world - 1) // world

    def set_epoch(self, epoch):
        self.epoch = epoch

    def __iter__(self):
        if self.shuffle:
            g = torch.Generator().manual_seed(self.seed + self.epoch)
            perm = torch.randperm(self.length, generator=g)
        else:
            perm = torch.arange(self.length)
        pad = self.n * self.world - self.length
        if pad:
            perm = torch.cat([perm, perm[:pad]])
        return iter(perm[self.rank::self.world].tolist())

    def __len__(self):
        return self.n


def _normal_path(img_name):
    return img_name.replace('/imgs/', '/normals/')[:-3] + 'png'     # as SceneDataset.__getitem__ names it


def pack_mask(mask):
    """Foreground of a mask as cv2 reads it ([H,W,C] or [H,W] uint8; a pixel is foreground when any channel is > 0, as
    in SceneDataset.__getitem__) -> int32 [H, ceil(W/32)]: bit c & 31 of word c >> 5 holds column c, rows padded to
    whole words (the mask plane of FrameStore)."""
    fg = np.asarray(mask) > 0
    if fg.ndim == 3:
        fg = fg.any(-1)
    H, W = fg.shape
    bits = np.zeros((H, (W + 31) // 32 * 32), np.bool_)
    bits[:, :W] = fg
    return np.packbits(bits, axis=-1, bitorder='little').view('<u4').view(np.int32)


class FrameStore:
    """A sequence's frames on one device, as the files hold them: img and normal uint8 [F,H,W,3] in file (BGR) order,
    mask bit-packed int32 [F,H,ceil(W/32)] (pack_mask).  `decode(ids)` -> the batch SceneDataset.__getitem__ and the
    DataLoader's collate would give for the host ids, as fp32 CUDA tensors on the current stream."""

    def __init__(self, img, mask, normal, W):
        self.img, self.mask, self.normal, self.W = img, mask, normal, W
        self.outputs = ('img', 'mask') + (('normal',) if normal is not None else ())

    @staticmethod
    def nbytes_for(F, H, W, with_normal):
        return F * H * (3 * W * (2 if with_normal else 1) + 4 * ((W + 31) // 32))

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in (self.img, self.mask, self.normal) if t is not None)

    def decode(self, ids):
        from selfreconcode_b200 import ops
        return ops.frames_decode(self.img, self.mask, self.normal, ids, self.W, self.outputs)


_STAGE_BYTES = 128 << 20    # pinned staging per chunk (two chunks in flight)


def _read_frame(paths, H, W):
    import cv2
    planes = []
    for p in paths:
        a = cv2.imread(p)
        if a is None or a.shape != (H, W, 3):
            raise ValueError("%s: %s, the sequence's frames are %dx%d" % (
                p, "unreadable" if a is None else "%dx%d" % a.shape[:2], H, W))
        planes.append(a)
    planes[1] = pack_mask(planes[1])
    return planes


def _host_path_reason(dataset, device):
    if device.type != 'cuda':
        return "device %s is not CUDA" % device
    if dataset.require_albedo:
        return "albedo planes are requested"
    n_normal = sum(osp.isfile(_normal_path(n)) for n in dataset.img_ns)
    if 0 < n_normal < dataset.frame_num:
        return "normals exist for %d of %d frames" % (n_normal, dataset.frame_num)
    need = FrameStore.nbytes_for(dataset.frame_num, dataset.H, dataset.W, n_normal > 0)
    free = torch.cuda.mem_get_info(device)[0]
    if 2 * need > free:
        return "the store needs %.2f GB, more than half of the %.2f GB free on %s" % (need / 1e9, free / 1e9, device)
    return None


def build_frame_store(dataset, device):
    """Decodes every frame's files once on the host (a thread pool: cv2 releases the GIL), packs the masks and copies
    the frames to `device` in chunks through pinned staging, so the host never holds the whole sequence."""
    t0 = time.perf_counter()
    F, H, W = dataset.frame_num, dataset.H, dataset.W
    with_normal = osp.isfile(_normal_path(dataset.img_ns[0]))
    shapes = [((H, W, 3), torch.uint8), ((H, (W + 31) // 32), torch.int32)] + \
        ([((H, W, 3), torch.uint8)] if with_normal else [])
    planes = [torch.empty((F,) + sh, dtype=dt, device=device) for sh, dt in shapes]
    chunk = max(1, min(F, _STAGE_BYTES // (FrameStore.nbytes_for(1, H, W, with_normal))))
    stages = [[torch.empty((chunk,) + sh, dtype=dt, pin_memory=True) for sh, dt in shapes] for _ in range(2)]
    copied = [None, None]

    def paths(i):
        return [dataset.img_ns[i], dataset.mask_ns[i]] + ([_normal_path(dataset.img_ns[i])] if with_normal else [])

    with torch.cuda.device(device), ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as pool:
        stream = torch.cuda.current_stream()
        for c, lo in enumerate(range(0, F, chunk)):
            hi = min(F, lo + chunk)
            frames = list(pool.map(lambda i: _read_frame(paths(i), H, W), range(lo, hi)))
            st = stages[c % 2]
            if copied[c % 2] is not None:
                copied[c % 2].synchronize()        # this staging buffer's previous copy has left it
            for j, fr in enumerate(frames):
                for k, a in enumerate(fr):
                    st[k][j].copy_(torch.from_numpy(a))
            for k in range(len(planes)):
                planes[k][lo:hi].copy_(st[k][:hi - lo], non_blocking=True)
            copied[c % 2] = torch.cuda.Event()
            copied[c % 2].record(stream)
        stream.synchronize()
    store = FrameStore(planes[0], planes[1], planes[2] if with_normal else None, W)
    print("[frame store] %d frames of %dx%d%s on %s: %.2f GB, built in %.1f s" % (
        F, H, W, " with normals" if with_normal else "", device, store.nbytes() / 1e9, time.perf_counter() - t0),
        flush=True)
    return store


def frame_store(dataset):
    """The dataset's device frame store, built at the first call after getOptNet recorded the training device
    (`dataset.store_device`); None while the frames stay on the host, with the reason printed once."""
    store = getattr(dataset, '_frame_store', None)
    device = getattr(dataset, 'store_device', None)
    if device is None or getattr(dataset, 'require_albedo', False):
        return None
    if store is None and getattr(dataset, '_frame_store_reason', None) is None:
        device = torch.device(device)
        why = _host_path_reason(dataset, device)
        if why is not None:
            print("[frame store] frames stay on the host: %s" % why, flush=True)
            dataset._frame_store_reason = why
        else:
            store = dataset._frame_store = build_frame_store(dataset, device)
    return store


class FrameLoader:
    """The loader of getDatasetAndLoader, with the DataLoader surface the drivers use: `dataset`, `batch_size`,
    `sampler`, `num_workers`, len() (drop_last=False) and iteration -> (frame_ids int64 CPU [B], outs).

    With a device frame store (frame_store), iteration runs in the main process without workers and `outs` holds
    CUDA tensors decoded by one launch per batch; otherwise it is a torch DataLoader built with the same arguments.
    Both paths draw the same numbers from the global RNGs in the same order, so a seeded run trains the same."""

    def __init__(self, dataset, batch_size=1, sampler=None, num_workers=0):
        self._host = torch.utils.data.DataLoader(dataset, batch_size, sampler=sampler, num_workers=num_workers)
        self.dataset, self.batch_size, self.num_workers = dataset, batch_size, num_workers
        self.sampler = self._host.sampler

    def __len__(self):
        return len(self._host)

    def __iter__(self):
        store = frame_store(self.dataset)
        if store is None:
            return iter(self._host)
        # a DataLoader iterator draws its base seed from the global generator when it is created
        # (_BaseDataLoaderIter), before the batch sampler first runs the sampler
        torch.empty((), dtype=torch.int64).random_()
        return self._batches(iter(self.sampler), store)

    def _batches(self, ids, store):
        batch = []
        for i in ids:
            batch.append(int(i))
            if len(batch) == self.batch_size:
                yield torch.tensor(batch, dtype=torch.int64), store.decode(batch)
                batch = []
        if batch:
            yield torch.tensor(batch, dtype=torch.int64), store.decode(batch)


def getDatasetAndLoader(root, conds_lens, batch_size, shuffle, num_workers, opt_pose, opt_trans, opt_camera,
                        rank=0, world=1):
    dataset = SceneDataset(root, conds_lens)
    dataset.poses.requires_grad_(bool(opt_pose))
    dataset.trans.requires_grad_(bool(opt_trans))
    dataset.opt_camera_params(opt_camera)
    sampler = RandomSampler(dataset, 1, shuffle) if world == 1 else ShardedSampler(dataset, rank, world, shuffle)
    loader = FrameLoader(dataset, batch_size, sampler=sampler, num_workers=num_workers)
    return dataset, loader


def write_sequence(root, imgs, masks, poses, trans, shape, camera, normals=None, gender='neutral'):
    """Writes a sequence in the layout above (used to build synthetic PeopleSnapshot-shaped sequences;
    the reference's own writer is people_snapshot_process.py:32-87).  imgs [F,H,W,3] in [-1,1] BGR,
    masks [F,H,W] {0,1}, normals [F,H,W,3] in [-1,1] RGB or None, camera = dict(fx,fy,cx,cy,quat,T)."""
    import cv2
    for sub in ('imgs', 'masks') + (('normals',) if normals is not None else ()):
        os.makedirs(osp.join(root, sub), exist_ok=True)
    to8 = lambda a: np.clip(np.round((np.asarray(a, dtype=np.float32) / 2. + 0.5) * 255.), 0, 255).astype(np.uint8)
    for i in range(len(imgs)):
        cv2.imwrite(osp.join(root, 'imgs/%06d.png' % i), to8(imgs[i]))
        cv2.imwrite(osp.join(root, 'masks/%06d.png' % i), (np.asarray(masks[i]) > 0).astype(np.uint8) * 255)
        if normals is not None:
            cv2.imwrite(osp.join(root, 'normals/%06d.png' % i), to8(normals[i])[:, :, ::-1])
    np.savez(osp.join(root, 'smpl_rec.npz'), poses=np.asarray(poses, np.float32), trans=np.asarray(trans, np.float32),
             shape=np.asarray(shape, np.float32), gender=gender)
    np.savez(osp.join(root, 'camera.npz'), **{k: np.asarray(v, np.float32) for k, v in camera.items()})
