"""Data time of a training batch on the two input paths of dataset.FrameLoader, on seeded synthetic sequences of 64
frames at 1080x1080 and 1080x1920 (smooth images, masks and normals, written with dataset.write_sequence):

  host  : torch DataLoader with 4 workers (config.conf's num_workers) decoding the PNGs with cv2, then the three
          `.to(device)` copies of OptimNetwork.forward / forward_rays (pageable memory: the main thread blocks);
  store : the device frame store built once per sequence, one sr_frames_decode launch per batch.

For N = 3, 2, 1 frames per batch the two paths alternate, each timing covering >= 50 batches after warm-up and ending
in a device synchronise; the main thread's time blocked in the copies and waiting for the workers is shown apart.
Then the bench's training step (bench.build_train / train_step, frames 512x512 of rays) runs with `datas` taken per
step from each path, alternated.  Host-to-device bytes per batch are computed from the shapes.  Prints the card and
its power limit first.

    python tools/frame_store_bench.py [--out DIR] [--batches 60] [--rounds 2] [--steps 30]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(1080, 1080), (1080, 1920)]
FRAMES = 64
WORKERS = 4


def _card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                             str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        pl = pl.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return "%s, power limit %s" % (name, pl)


class _Batches:
    """Endless batches of one path: a new loader iterator per epoch, as a training loop makes."""

    def __init__(self, loader):
        self.loader, self.it = loader, iter(loader)

    def next(self):
        try:
            return next(self.it)
        except StopIteration:
            self.it = iter(self.loader)
            return next(self.it)


def _host_batch(src, dev, acc):
    t0 = time.perf_counter()
    ids, outs = src.next()
    t1 = time.perf_counter()
    datas = {k: outs[k].to(dev) for k in ('img', 'mask', 'normal')}
    t2 = time.perf_counter()
    acc[0] += t1 - t0
    acc[1] += t2 - t1
    return ids, datas


def _time_batches(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def data_time(ds, store, dev, N, batches, rounds):
    from dataset import FrameLoader, RandomSampler
    host = _Batches(torch.utils.data.DataLoader(ds, N, sampler=RandomSampler(ds, 1, True), num_workers=WORKERS))
    dev_loader = FrameLoader(ds, N, sampler=RandomSampler(ds, 1, True), num_workers=WORKERS)
    assert dev_loader.dataset._frame_store is store
    dsrc = _Batches(dev_loader)
    res = {"host_ms": [], "host_wait_ms": [], "host_copy_ms": [], "store_ms": []}
    for _ in range(10):                      # warm-up: worker start, allocator, module load
        _host_batch(host, dev, [0.0, 0.0])
        dsrc.next()
    for _ in range(rounds):
        acc = [0.0, 0.0]
        res["host_ms"].append(_time_batches(lambda: _host_batch(host, dev, acc), batches))
        res["host_wait_ms"].append(acc[0] / batches * 1e3)
        res["host_copy_ms"].append(acc[1] / batches * 1e3)
        res["store_ms"].append(_time_batches(dsrc.next, batches))
    H, W = ds.H, ds.W
    out = {k: float(np.median(v)) for k, v in res.items()}
    out.update(N=N, h2d_bytes_host=N * H * W * 28, h2d_bytes_store=N * 8,
               store_decode_hbm_bytes=int(N * H * (6 * W + 4 * ((W + 31) // 32)) + N * H * W * 28))
    return out


def step_time(root, dev, steps, rounds):
    import bench
    from dataset import FrameLoader, RandomSampler, SceneDataset, frame_store
    sc = bench.build_scene(dev, 0)
    tr = bench.build_train(sc, dev, 0, 1)
    ds = SceneDataset(root)
    ds.store_device = dev
    frame_store(ds)
    nb = bench.TRAIN_FRAMES
    host = _Batches(torch.utils.data.DataLoader(ds, nb, sampler=RandomSampler(ds, 1, True), num_workers=WORKERS))
    store = _Batches(FrameLoader(ds, nb, sampler=RandomSampler(ds, 1, True), num_workers=WORKERS))

    def run(src):
        # forward_rays copies what it reads (img, normal) with .to(device), a no-op on the store's tensors
        tr["datas"] = src.next()[1]
        bench.train_step(tr)

    ms = {"host": [], "store": [], "resident": []}
    resident = {k: v.clone() for k, v in store.next()[1].items()}

    def run_resident():
        tr["datas"] = resident
        bench.train_step(tr)
    for _ in range(5):
        run(host)
        run(store)
        run_resident()
    for _ in range(rounds):
        ms["host"].append(_time_batches(lambda: run(host), steps))
        ms["store"].append(_time_batches(lambda: run(store), steps))
        ms["resident"].append(_time_batches(run_resident, steps))
    return {k + "_step_ms": float(np.median(v)) for k, v in ms.items()} | {
        "frames": "%d of %dx%d per step, %d rays" % (nb, ds.H, ds.W, tr["n_rays"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_store_bench"),
                    help="where the sequences and frame_store_bench.json are written")
    ap.add_argument("--batches", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("frame_store_bench: needs a CUDA device")
    from selfreconcode_b200 import enable_dropin, synth
    enable_dropin()
    from dataset import SceneDataset, frame_store
    dev = torch.device("cuda:0")
    print("card: %s" % _card(), flush=True)
    report = {"card": _card(), "frames": FRAMES, "workers": WORKERS, "sequences": []}
    roots = {}
    for i, (H, W) in enumerate(SIZES):
        root = os.path.join(args.out, "seq_%dx%d" % (H, W))
        t0 = time.perf_counter()
        if not os.path.isfile(os.path.join(root, "camera.npz")):
            synth.write_frame_sequence(root, FRAMES, H, W, seed=100 + i)
        print("wrote %s in %.1f s" % (root, time.perf_counter() - t0), flush=True)
        roots[(H, W)] = root
        ds = SceneDataset(root)
        ds.store_device = dev
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        store = frame_store(ds)
        build_s = time.perf_counter() - t0
        seq = {"H": H, "W": W, "store_build_s": build_s, "store_bytes": store.nbytes(), "batches": []}
        for N in (3, 2, 1):
            try:
                r = data_time(ds, store, dev, N, args.batches, args.rounds)
            except RuntimeError as e:          # e.g. the workers' shared memory runs out at large frames
                r = {"N": N, "error": str(e)[:300]}
            print("%dx%d N=%d %s" % (H, W, N, json.dumps(r)), flush=True)
            seq["batches"].append(r)
        report["sequences"].append(seq)
        del store, ds
        torch.cuda.empty_cache()
    try:
        report["train_step"] = step_time(roots[SIZES[0]], dev, args.steps, args.rounds)
    except RuntimeError as e:
        report["train_step"] = {"error": str(e)[:300]}
    print("train step %s" % json.dumps(report["train_step"]), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "frame_store_bench.json"), "w") as f:
        json.dump(report, f, indent=1)
    print(json.dumps(report))


if __name__ == "__main__":
    main()
