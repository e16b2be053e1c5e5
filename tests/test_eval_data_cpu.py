"""On-disk test-set listing (distributed_sod_project_b200/data.py) follows the reference's rules
(utils/dataset.py:22-69): folder form driven by the masks, .png > .jpg > .bmp when a folder mixes extensions, list-file
form with `prefix`; and the loader packs ragged batches of the decoded originals."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from distributed_sod_project_b200 import data


def _touch(path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    open(path, "wb").close()


def test_folder_form_is_driven_by_the_masks(tmp_path):
    root = tmp_path / "SET"
    for n in ("a", "b", "c", "d"):
        _touch(str(root / "Image" / f"{n}.jpg"))
    for n in ("b", "a", "c"):
        _touch(str(root / "Mask" / f"{n}.png"))
    pairs = data.list_pairs(str(root))
    assert pairs == [(str(root / "Image" / f"{n}.jpg"), str(root / "Mask" / f"{n}.png")) for n in ("a", "b", "c")]


def test_mixed_extensions_choose_png_then_jpg_then_bmp(tmp_path):
    root = tmp_path / "SET"
    for f in ("x.jpg", "x.bmp", "y.jpg", "z.bmp", "notes.txt"):
        _touch(str(root / "Image" / f))
    for f in ("x.png", "x.bmp", "y.png", "z.bmp"):
        _touch(str(root / "Mask" / f))
    pairs = data.list_pairs(str(root))
    # images: .jpg (no .png among them); masks: .png — only masks with the chosen extension make pairs
    assert pairs == [(str(root / "Image" / "x.jpg"), str(root / "Mask" / "x.png")),
                     (str(root / "Image" / "y.jpg"), str(root / "Mask" / "y.png"))]
    assert data._folder_ext(["a.bmp", "b.jpg"]) == ".jpg" and data._folder_ext(["a.bmp", "b.tif"]) == ".bmp"
    assert data._folder_ext(["a.tif"]) == ".tif"
    with pytest.raises(ValueError):
        data._folder_ext(["a.tif", "b.gif"])


def test_list_file_form_uses_the_prefix(tmp_path):
    lst = tmp_path / "test.lst"
    lst.write_text(f"{tmp_path}/DUTS/img_1 extra\n{tmp_path}/DUTS/img_2\n\n")
    pairs = data.list_pairs(str(lst), prefix=(".jpg", ".png"))
    assert pairs == [(f"{tmp_path}/DUTS/Image/img_1.jpg", f"{tmp_path}/DUTS/Mask/img_1.png"),
                     (f"{tmp_path}/DUTS/Image/img_2.jpg", f"{tmp_path}/DUTS/Mask/img_2.png")]
    assert data.list_pairs(str(lst), prefix=(".bmp", ".bmp"))[0][0].endswith("img_1.bmp")


def test_missing_set_is_an_error_naming_it(tmp_path):
    with pytest.raises(FileNotFoundError, match="ecssd"):
        data.open_test_set("ecssd", str(tmp_path / "nowhere"), 4)
    with pytest.raises(FileNotFoundError):
        data.list_pairs(str(tmp_path / "nowhere"))


def test_loader_packs_ragged_batches_of_the_originals(tmp_path):
    rng = np.random.default_rng(0)
    root = tmp_path / "SET"
    os.makedirs(root / "Image")
    os.makedirs(root / "Mask")
    sizes = [(30, 40), (41, 23), (17, 17), (50, 9), (12, 31)]
    want = {}
    for i, (h, w) in enumerate(sizes):
        img = rng.integers(0, 256, (h, w, 3)).astype(np.uint8)
        gt = rng.integers(0, 256, (h, w)).astype(np.uint8)
        Image.fromarray(img, "RGB").save(root / "Image" / f"im{i}.v2.png")      # names stop at the first dot
        Image.fromarray(gt, "L").convert("RGB").save(root / "Mask" / f"im{i}.v2.png")
        want[f"im{i}"] = (img, gt)
    loader, n = data.make_eval_loader(str(root), batch_size=2, indices=range(1, 5, 2))
    assert n == 5
    seen = []
    for b in loader:
        assert isinstance(b, data.EvalBatch)
        o_i = o_g = 0
        for k, name in enumerate(b.names):
            (h, w), (gh, gw) = b.img_hw[k].tolist(), b.gt_hw[k].tolist()
            img, gt = want[name]
            assert (h, w) == img.shape[:2] == (gh, gw)
            assert np.array_equal(b.img[o_i:o_i + h * w * 3].numpy().reshape(h, w, 3), img)
            assert np.array_equal(b.gt[o_g:o_g + h * w].numpy().reshape(h, w), gt)   # RGB mask → "L" of grey = grey
            o_i, o_g = o_i + h * w * 3, o_g + h * w
            seen.append(name)
        assert o_i == b.img.numel() and o_g == b.gt.numel()
    assert seen == ["im1", "im3"]
    assert torch.is_tensor(b.img_hw) and b.img_hw.dtype == torch.int32
