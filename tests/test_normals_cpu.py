"""CPU: the host side of the normal-map step (selfreconcode_b200/normals.py) -- the front-normal net's key layout
and the strict loader, the host preprocessing against tests/golden/normals_io.npz (written by the unmodified
generate_normals.py under oracle/make_golden_normals.py, with a stand-in network), crop-box choice, folder walking
and output naming, and the float32 restatement of the unwarp / quantise rule against the script's PNGs."""
import os

import numpy as np
import pytest
import torch

import normal_net_ref as R
from helpers import golden
from selfreconcode_b200 import normals as N

PIFUHD_TABLE = {'model.1': (64, 3, 7, 7), 'model.4': (128, 64, 3, 3), 'model.7': (256, 128, 3, 3),
                'model.10': (512, 256, 3, 3), 'model.13': (1024, 512, 3, 3), 'model.25': (1024, 512, 3, 3),
                'model.28': (512, 256, 3, 3), 'model.31': (256, 128, 3, 3), 'model.34': (128, 64, 3, 3),
                'model.38': (3, 64, 7, 7)}
PIFUHD_TABLE.update({'model.%d.conv_block.%d' % (b, c): (1024, 1024, 3, 3) for b in range(16, 25) for c in (1, 5)})


def _bias_len(name, shape):
    return shape[1] if name in ('model.25', 'model.28', 'model.31', 'model.34') else shape[0]


def test_twin_layout_is_pifuhd_table():
    net = R.GlobalGenerator(**N.PIFUHD_ARCH)
    sd = {k: tuple(v.shape) for k, v in net.state_dict().items()}
    want = {}
    for name, shape in PIFUHD_TABLE.items():
        want[name + '.weight'] = shape
        want[name + '.bias'] = (_bias_len(name, shape),)
    assert len(sd) == 56 and sd == want
    assert dict(N.layer_keys(**N.PIFUHD_ARCH)) == want
    for arch in (R.SMALL, dict(in_nc=3, out_nc=3, ngf=4, n_down=1, n_blocks=0)):
        assert dict(N.layer_keys(**arch)) == {k: tuple(v.shape) for k, v in R.GlobalGenerator(**arch).state_dict().items()}


def test_loader_prefix_and_architecture(tmp_path):
    sd = R.seeded_net(0, **R.SMALL).float().state_dict()
    ck = {'netG.netF.' + k: v for k, v in sd.items()}
    ck.update({'netG.netB.model.1.weight': torch.zeros(2), 'netG.other': torch.zeros(1)})
    p = str(tmp_path / 'pifuhd.pt')
    torch.save({'model_state_dict': ck, 'epoch': 3}, p)
    got = N.read_state_dict(p)
    assert list(got) == list(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    assert N.architecture(got) == R.SMALL
    assert list(N.read_state_dict(sd)) == list(sd)             # a bare state dict
    assert N.architecture(R.GlobalGenerator(**N.PIFUHD_ARCH).state_dict()) == N.PIFUHD_ARCH


def test_loader_rejects_bad_keys():
    sd = dict(R.seeded_net(0, **R.SMALL).float().state_dict())
    bad = dict(sd)
    del bad['model.11.conv_block.5.bias']
    with pytest.raises(KeyError, match="missing key 'model.11.conv_block.5.bias'"):
        N.architecture(bad)
    bad = dict(sd, **{'model.99.weight': torch.zeros(1)})
    with pytest.raises(KeyError, match="unexpected key 'model.99.weight'"):
        N.architecture(bad)
    bad = dict(sd, **{'model.15.weight': torch.zeros(8, 16, 3, 3)})     # an up conv in Conv2d's orientation
    with pytest.raises(ValueError, match="'model.15.weight' has shape"):
        N.architecture(bad)
    bad = dict(sd, **{'model.10.conv_block.1.weight': torch.zeros(32, 32, 1, 1)})
    with pytest.raises(ValueError, match="'model.10.conv_block.1.weight'"):
        N.architecture(bad)
    with pytest.raises(KeyError, match="model.1.weight"):
        N.architecture({k: v for k, v in sd.items() if not k.startswith('model.1.')})


def _golden_tree(tmp_path):
    g = golden("normals_io.npz")
    for k in g.files:
        if k.startswith('files/'):
            p = os.path.join(str(tmp_path), k[6:])
            os.makedirs(os.path.dirname(p), exist_ok=True)
            with open(p, 'wb') as f:
                f.write(g[k].tobytes())
    return g


def _golden_frame(tmp_path, key):
    lay, fold, stem = key.split('|')
    root = os.path.normpath(os.path.join(str(tmp_path), lay, 'imgs', fold))
    return [p for p in N.list_frames(root) if os.path.basename(p).split('.')[0] == stem][0]


def test_host_preprocessing_bitwise_vs_script(tmp_path):
    g = _golden_tree(tmp_path)
    assert len(g['frames']) == 8 and list(g['loaded_keys']) == []
    for key in g['frames']:
        f = N.prepare_frame(_golden_frame(tmp_path, key))
        assert f['x'].dtype == np.float32 and f['x'].shape == (3, 512, 512), key
        assert R.sha256(f['x']) == str(g['x_sha256/' + key]), key        # the script's network input, bit for bit
        assert f['rect_from'] == 'file', key
        assert (f['H'], f['W']) == g['png/' + key].shape[:2]


def test_unwarp_restatement_bitwise_vs_script(tmp_path):
    g = _golden_tree(tmp_path)
    for key in g['frames']:
        f = N.prepare_frame(_golden_frame(tmp_path, key))
        y = R.standin(f['x'])
        assert R.sha256(y) == str(g['y_sha256/' + key]), key             # the stand-in's output the script used
        png = g['png/' + key]
        assert np.array_equal(R.unwarp_f32(y, f['rect'], f['fg'], f['H'], f['W']), png), key
        v, zero = R.unwarp_quantise(y, f['rect'], f['fg'], f['H'], f['W'])
        assert np.abs(v - png).max() < 1 + 1e-3 and (png[zero] == 0).all(), key
    assert (g['png/seqA|.|3'] > 0).any() and (g['png/seqA|.|0'] == 0).any()


def test_rect_choice():
    assert N.choose_rect(np.array([3, 4, 10, 12], np.int32)) == [3, 4, 10, 12]
    rects = np.array([[1, 1, 10, 10], [10, 5, 40, 40], [0, 0, 60, 20], [5, 5, 20, 61], [5, 5, 20, 62]], np.int32)
    assert N.choose_rect(rects[:4]) == [10, 5, 40, 40]                   # ties at (w + h) // 2 = 40: the first
    assert N.choose_rect(rects) == [5, 5, 20, 62]                        # 41
    assert N.choose_rect(np.array([[0, 0, 0, 0], [1, 1, -2, 0]], np.int32)) == [1, 1, -2, 0]   # none positive: last


def test_mask_box_and_fallback():
    H, W = 40, 60
    fg = np.zeros((H, W), bool)
    fg[5:26, 10:21] = True                          # x 10..20 (w 11), y 5..25 (h 21)
    r = int(0.57 * 21)
    assert N.mask_box(fg, H, W) == [15 - r, 15 - r, 2 * r, 2 * r]
    assert N.mask_box(np.zeros((H, W), bool), H, W) == [30 - 30, 20 - 30, 60, 60]
    assert N.mask_box(None, H, W) == [0, -10, 60, 60]
    one = np.zeros((H, W), bool)
    one[3, 4] = True
    assert N.mask_box(one, H, W) == [3, 2, 2, 2]   # radius at least 1


def test_frames_without_rect_use_mask_box(tmp_path):
    _golden_tree(tmp_path)
    f5 = N.prepare_frame(os.path.join(str(tmp_path), 'seqA', 'imgs', '5.png'))
    import cv2
    fg = (cv2.imread(os.path.join(str(tmp_path), 'seqA', 'masks', '5.png')) > 0).all(-1)
    assert f5['rect_from'] == 'mask' and f5['rect'] == N.mask_box(fg, 72, 96)
    os.remove(os.path.join(str(tmp_path), 'seqA', 'masks', '5.png'))
    f5 = N.prepare_frame(os.path.join(str(tmp_path), 'seqA', 'imgs', '5.png'))
    assert f5['rect_from'] == 'centre' and f5['rect'] == [0, -12, 96, 96] and f5['fg'] is None


def test_folders_and_output_naming(tmp_path):
    g = _golden_tree(tmp_path)
    a = os.path.join(str(tmp_path), 'seqA', 'imgs')
    b = os.path.join(str(tmp_path), 'seqB', 'imgs')
    assert N.list_folds(a) == ['.'] and N.list_folds(b) == ['0', '1']
    assert [os.path.basename(p) for p in N.list_frames(a)] == ['%d.png' % i for i in range(6)]
    assert N.mask_path('/d/imgs/0/7.jpg') == '/d/masks/0/7.png' and N.rect_path('/d/imgs/7.png') == '/d/imgs/7_rect.txt'
    open(os.path.join(a, '10.png'), 'wb').write(open(os.path.join(a, '2.png'), 'rb').read())
    assert [os.path.basename(p) for p in N.list_frames(a)][-2:] == ['5.png', '10.png']    # int(stem) order
    # the script's outputs: <imgpath>/../normals/<fold>/<stem>.png, frames without _rect.txt skipped there
    assert list(g['written/seqA']) == ['normals/%d.png' % i for i in range(5)]
    assert list(g['written/seqB']) == ['normals/0/0.png', 'normals/0/1.png', 'normals/1/2.png']


def test_module_imports_no_torchvision_pil_or_oracle(tmp_path):
    import subprocess
    import sys
    from helpers import ROOT
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import selfreconcode_b200.normals as N\n"
            "import numpy as np, cv2\n"
            "p = %r\n"
            "cv2.imwrite(p, np.full((20, 30, 3), 90, np.uint8))\n"
            "f = N.prepare_frame(p)\n"
            "assert f['rect_from'] == 'centre' and f['x'].shape == (3, 512, 512)\n"
            "bad = [m for m in sys.modules if m.split('.')[0] in ('torchvision', 'PIL', 'oracle', 'lib', 'modules')]\n"
            "assert not bad, bad\n") % (ROOT, str(tmp_path / "imgs" / "0.png"))
    os.makedirs(str(tmp_path / "imgs"))
    subprocess.check_call([sys.executable, "-c", code])
