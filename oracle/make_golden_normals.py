"""TEST INFRASTRUCTURE -- writes tests/golden/normals_io.npz by running the UNMODIFIED reference script
generate_normals.py on the CPU (needs the reference tree, no GPU, no PIFuHD checkout):

    python oracle/make_golden_normals.py [OUT.npz]

The script runs as it is (runpy) with three things patched:
  * `lib.networks.define_G` -> a cheap fixed stand-in: a 1x1 channel mix of its input with power-of-two weights,
    rounded to multiples of 2^-10, one float32 operation at a time (STANDIN below), so the tests recompute its output
    exactly from the input instead of storing it; it records every [1,3,512,512] input it receives and its output;
  * `torch.load` -> a checkpoint with only a 'netG.netB.' entry (the stand-in records the keys the script passes on);
  * `torch.device` -> the CPU.
It runs on small synthetic sequences written here: a multi-row _rect.txt with a tie, a box with negative x / y, a box
past the right and bottom edges, a frame without a mask, an RGBA frame, a frame without _rect.txt (the reference
skips it), and a digit-subfolder layout with a .jpg frame.

Keys:  files/<path>           bytes of every input file (images, masks, rect files), relative to the temp root
       frames                 '<layout>|<fold>|<stem>' of each frame the script processed, in order
       x_sha256/<frame>       SHA-256 of the stand-in's input, float32 [3,512,512] C order (bit-for-bit identity)
       y_sha256/<frame>       the same of its output
       png/<frame>            the normal map the script wrote, uint8 BGR [H,W,3]
       written/<layout>       the png paths the script wrote, relative to the layout root
       loaded_keys            the keys the script passed to load_state_dict
"""
import hashlib
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = "/root/reference"

# output channel o = round((0.5 x[o] + 0.25 x[o+1] - 0.125 x[o+2] + STANDIN_B[o]) * 1024) / 1024 (channels mod 3),
# added left to right: products by powers of two are exact, so every step is one correctly rounded float32 operation
# (restated in tests/normal_net_ref.py standin)
STANDIN_B = (0.0625, -0.125, 0.03125)


def _image(H, W, seed, ch=3):
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    planes = [127.5 + 120 * np.sin(xx / (5 + 3 * c + seed) + yy / (7 + 2 * c)) * np.cos(yy / (9 + c + seed))
              for c in range(3)]
    img = np.stack(planes, -1)
    img = np.clip(np.round(img), 0, 255).astype(np.uint8)
    if ch == 4:
        a = np.clip(np.round(255 * (0.3 + 0.7 * (xx / W))), 0, 255).astype(np.uint8)
        img = np.concatenate([img, a[..., None]], -1)
    return img


def _mask(H, W, cx, cy, rx, ry):
    yy, xx = np.mgrid[0:H, 0:W]
    return ((((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2) <= 1).astype(np.uint8) * 255


def write_inputs(base):
    """Synthetic layouts under base -> {layout: imgpath}."""
    import cv2
    a = os.path.join(base, "seqA")
    for d in ("imgs", "masks"):
        os.makedirs(os.path.join(a, d), exist_ok=True)
    H, W = 72, 96
    rects = {0: [[1, 1, 10, 10], [10, 5, 40, 40], [0, 0, 60, 20], [5, 5, 20, 60]],   # tie at 40: row 1 (first)
             1: [[-10, -6, 50, 50]],                                               # negative x / y
             2: [[40, 30, 60, 70]],                                                # past the right and bottom edges
             3: [[20, 10, 48, 48]],                                                # no mask
             4: [[8, 4, 64, 64]]}                                                  # RGBA
    for i in range(6):
        cv2.imwrite(os.path.join(a, "imgs", "%d.png" % i), _image(H, W, i, ch=4 if i == 4 else 3))
        if i != 3:
            cv2.imwrite(os.path.join(a, "masks", "%d.png" % i), _mask(H, W, 40 + 2 * i, 36, 18, 30))
        if i in rects:                                                             # frame 5: no _rect.txt
            np.savetxt(os.path.join(a, "imgs", "%d_rect.txt" % i), np.array(rects[i]), fmt="%d")
    b = os.path.join(base, "seqB")
    for fold, names in (("0", ["0.png", "1.png"]), ("1", ["2.jpg"])):
        for d in ("imgs", "masks"):
            os.makedirs(os.path.join(b, d, fold), exist_ok=True)
        for j, n in enumerate(names):
            seed = 10 + 3 * int(fold) + j
            cv2.imwrite(os.path.join(b, "imgs", fold, n), _image(64, 48, seed))
            cv2.imwrite(os.path.join(b, "masks", fold, n[:-3] + "png"), _mask(64, 48, 24, 30 + j, 14, 25))
            np.savetxt(os.path.join(b, "imgs", fold, n.split(".")[0] + "_rect.txt"),
                       np.array([[2 + j, -3, 44, 70]]), fmt="%d")
    return {"seqA": os.path.join(a, "imgs"), "seqB": os.path.join(b, "imgs")}


class _StandIn(torch.nn.Module):
    def __init__(self, log):
        super().__init__()
        self.log = log

    def load_state_dict(self, sd, strict=True):
        self.log["loaded_keys"] = sorted(sd)

    def forward(self, x):
        chans = []
        for o in range(3):
            t = x[:, o] * 0.5
            t = t + x[:, (o + 1) % 3] * 0.25
            t = t - x[:, (o + 2) % 3] * 0.125
            t = t + STANDIN_B[o]
            chans.append(torch.round(t * 1024.0) / 1024.0)
        y = torch.stack(chans, 1)
        self.log["calls"].append((x.detach().clone(), y.detach().clone()))
        return y


def run_reference(imgpath, log):
    import cv2
    real_device, real_load, real_imwrite = torch.device, torch.load, cv2.imwrite

    class _Meta(type):
        def __call__(cls, *a, **k):
            return real_device("cpu")

        def __instancecheck__(cls, obj):
            return isinstance(obj, real_device)

    class _CpuDevice(metaclass=_Meta):
        pass

    nets = types.ModuleType("lib.networks")
    nets.define_G = lambda *a, **k: (log.setdefault("define_G", a), _StandIn(log))[1]
    lib = types.ModuleType("lib")
    lib.__path__ = []
    lib.networks = nets

    def imwrite(path, img, *a):
        log["writes"].append((path, img.copy()))
        return real_imwrite(path, img, *a)

    saved = {k: sys.modules.get(k) for k in ("lib", "lib.networks")}
    sys.modules["lib"], sys.modules["lib.networks"] = lib, nets
    torch.device = _CpuDevice
    torch.load = lambda *a, **k: {"model_state_dict": {"netG.netB.model.1.weight": torch.zeros(1)}}
    cv2.imwrite = imwrite
    argv = sys.argv
    sys.argv = ["generate_normals.py", "--imgpath", imgpath]
    try:
        runpy.run_path(os.path.join(REF, "generate_normals.py"), run_name="__main__")
    finally:
        sys.argv = argv
        torch.device, torch.load, cv2.imwrite = real_device, real_load, real_imwrite
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def main(out):
    res = {}
    frames = []
    with tempfile.TemporaryDirectory() as base:
        layouts = write_inputs(base)
        for dirpath, _, files in os.walk(base):
            for f in files:
                p = os.path.join(dirpath, f)
                res["files/" + os.path.relpath(p, base)] = np.frombuffer(open(p, "rb").read(), np.uint8)
        for name, imgpath in layouts.items():
            log = {"calls": [], "writes": []}
            run_reference(imgpath, log)
            assert len(log["calls"]) == len(log["writes"]), name
            res["loaded_keys"] = np.array(log["loaded_keys"], dtype=str)
            assert log["define_G"] == (3, 3, 64, "global", 4, 9, 1, 3, "instance"), log["define_G"]
            root = os.path.dirname(imgpath)
            written = []
            for (x, y), (path, png) in zip(log["calls"], log["writes"]):
                rel = os.path.relpath(path, os.path.join(root, "normals"))
                fold = os.path.dirname(rel) or "."
                key = "%s|%s|%s" % (name, fold, os.path.basename(rel)[:-4])
                frames.append(key)
                res["x_sha256/" + key] = np.array(sha256(x[0]))
                res["y_sha256/" + key] = np.array(sha256(y[0]))
                res["png/" + key] = png
                on_disk = cv2_read(path)
                assert np.array_equal(on_disk, png), key
                written.append(os.path.relpath(path, root))
            res["written/" + name] = np.array(sorted(written), dtype=str)
    res["frames"] = np.array(frames, dtype=str)
    np.savez_compressed(out, **res)
    print(out, os.path.getsize(out), "bytes,", len(frames), "frames:", frames)


def sha256(t):
    a = np.ascontiguousarray(t.numpy(), dtype=np.float32)
    assert a.shape == (3, 512, 512)
    return hashlib.sha256(a.tobytes()).hexdigest()


def cv2_read(p):
    import cv2
    return cv2.imread(p, cv2.IMREAD_UNCHANGED)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "normals_io.npz"))
