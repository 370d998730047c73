"""Dataset / tile / palette / checkpoint boundary (the API the reference's own tests pin: tests/test_datasets.py,
tests/test_tiles.py) on synthetic slippy-map directories, plus fixtures produced by the real reference."""

import os

import numpy as np
import pytest
import torch
from PIL import Image

from robosat_b200 import colors, synth, tiles as T
from robosat_b200.datasets import BufferedSlippyMapDirectory, SlippyMapTiles, SlippyMapTilesConcatenation
from robosat_b200.transforms import ImageToTensor, JointCompose, JointTransform, MaskToTensor

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _write_grid(root, gold, ext="png"):
    for key in gold.files:
        if key.startswith("tile_"):
            _, x, y = key.split("_")
            os.makedirs(os.path.join(root, "7", x), exist_ok=True)
            Image.fromarray(gold[key]).save(os.path.join(root, "7", x, "%s.%s" % (y, ext)))


def test_tiles_from_slippy_map_and_csv(tmp_path):
    gold = np.load(os.path.join(GOLD, "tiles.npz"))
    _write_grid(str(tmp_path), gold)
    (tmp_path / "7" / "notanumber").mkdir()
    (tmp_path / "README").write_text("ignored")
    found = list(T.tiles_from_slippy_map(str(tmp_path)))
    assert len(found) == 8
    tile, path = found[0]
    assert isinstance(tile, T.Tile) and tile.z == 7 and path.endswith("%d/%d.png" % (tile.x, tile.y))
    csv = tmp_path / "tiles.csv"
    csv.write_text("69623,104945,18\n\n69622,104945,18\n69623,104946,18\n")
    rows = list(T.tiles_from_csv(str(csv)))
    assert len(rows) == 3 and rows[0] == T.Tile(69623, 104945, 18)


def test_buffer_tile_image_matches_reference_fixture(tmp_path):
    gold = np.load(os.path.join(GOLD, "tiles.npz"))
    _write_grid(str(tmp_path), gold)
    tiles = list(T.tiles_from_slippy_map(str(tmp_path)))
    index = dict(tiles)
    centre = T.Tile(11, 21, 7)
    corner = T.Tile(10, 20, 7)
    assert np.array_equal(np.array(T.buffer_tile_image(centre, index, overlap=4, tile_size=16)), gold["buffered_centre_o4"])
    assert np.array_equal(np.array(T.buffer_tile_image(corner, tiles, overlap=4, tile_size=16)), gold["buffered_corner_o4"])  # list form too
    assert np.array_equal(np.array(T.buffer_tile_image(centre, index, overlap=0, tile_size=16)), gold["buffered_centre_o0"])


def test_palettes_match_reference_fixture():
    gold = np.load(os.path.join(GOLD, "tiles.npz"))
    assert colors.continuous_palette_for_color("pink", 256) == gold["palette_pink_256"].tolist()
    assert colors.make_palette("denim", "orange") == gold["palette_denim_orange"].tolist()


def _make_dataset(root, n=3, size=32):
    rng = np.random.RandomState(0)
    for sub, mode in (("images", "RGB"), ("labels", "P")):
        for i in range(n):
            d = os.path.join(root, sub, "18", str(69105 + i))
            os.makedirs(d, exist_ok=True)
            if mode == "RGB":
                Image.fromarray(rng.randint(0, 256, (size, size, 3)).astype(np.uint8)).save(os.path.join(d, "105093.png"))
            else:
                img = Image.fromarray(rng.randint(0, 2, (size, size)).astype(np.uint8), mode="P")
                img.putpalette(colors.make_palette("denim", "orange"))
                img.save(os.path.join(d, "105093.png"))


def test_slippy_map_datasets_api(tmp_path):
    _make_dataset(str(tmp_path))
    ds = SlippyMapTiles(str(tmp_path / "images"))
    assert len(ds) == 3
    image, tile = ds[0]
    assert tile == T.Tile(69105, 105093, 18) and image.size == (32, 32)
    joint = JointCompose([JointTransform(ImageToTensor(), MaskToTensor())])
    cat = SlippyMapTilesConcatenation([str(tmp_path / "images")], str(tmp_path / "labels"), joint)
    assert len(cat) == 3
    images, mask, tiles = cat[0]
    assert tiles[0] == T.Tile(69105, 105093, 18)
    assert isinstance(images, torch.Tensor) and images.shape == (3, 32, 32) and images.dtype == torch.float32
    assert isinstance(mask, torch.Tensor) and mask.dtype == torch.int64 and mask.shape == (32, 32)


def test_buffered_directory_and_unbuffer(tmp_path):
    rng = np.random.RandomState(1)
    for x in (5, 6):
        os.makedirs(str(tmp_path / "3" / str(x)))
        Image.fromarray(rng.randint(0, 256, (256, 256, 3)).astype(np.uint8)).save(str(tmp_path / "3" / str(x) / "2.png"))
    d = BufferedSlippyMapDirectory(str(tmp_path), transform=None, size=256, overlap=32)
    assert len(d) == 2
    image, xyz = d[0]
    assert image.size == (320, 320) and xyz.dtype == torch.int32 and xyz.tolist()[2] == 3
    probs = np.zeros((2, 320, 320), dtype=np.float32)
    assert d.unbuffer(probs).shape == (2, 256, 256)


def test_image_to_tensor_matches_torchvision_semantics():
    rng = np.random.RandomState(2)
    arr = rng.randint(0, 256, (8, 8, 3)).astype(np.uint8)
    t = ImageToTensor()(Image.fromarray(arr))
    assert torch.equal(t, torch.from_numpy(arr).permute(2, 0, 1).float().div(255))


def test_unet_module_state_dict_is_checkpoint_compatible():
    """robosat_b200.unet.UNet wrapped in DataParallel has exactly the reference checkpoint's keys / shapes / dtypes (SURVEY.md F9)."""
    from robosat_b200.unet import UNet

    net = torch.nn.DataParallel(UNet(2, pretrained=False))
    ref = synth.make_state_dict(2, seed=0)
    sd = net.state_dict()
    assert list(sd.keys()) == list(ref.keys())
    assert all(sd[k].shape == ref[k].shape and sd[k].dtype == ref[k].dtype for k in ref)
    net.load_state_dict(ref)  # strict load works
    with pytest.raises(Exception):
        net.module(torch.zeros(1, 3, 64, 64))  # no CPU execution path: must raise, never fall back


def test_adam_state_dict_layout_needs_gpu():
    # the layout itself is covered in tests/test_train_gpu.py; here: module imports without a GPU
    import robosat_b200.optim  # noqa: F401
    import robosat_b200.tools.predict  # noqa: F401
    import robosat_b200.tools.train  # noqa: F401


def test_serve_tool_parser_and_cpu_refusal():
    """`rs serve` keeps the reference's flags (serve.py:76-93); the GPU Predictor refuses a cuda=false config loudly."""
    import argparse

    from robosat_b200 import _lib
    from robosat_b200.serve import Predictor
    from robosat_b200.tools import serve

    parser = argparse.ArgumentParser()
    serve.add_parser(parser.add_subparsers())
    args = parser.parse_args(["serve", "--model", "m.toml", "--dataset", "d.toml", "--checkpoint", "c.pth", "--url", "http://x/{z}/{x}/{y}"])
    assert (args.tile_size, args.host, args.port) == (512, "127.0.0.1", 5000) and args.func is serve.main
    with pytest.raises(_lib.RsbError):
        Predictor({"state_dict": {}}, {"common": {"cuda": False}}, {"common": {"classes": ["a", "b"], "colors": ["denim", "orange"]}})


def test_train_rejects_label_values_outside_the_classes(tmp_path):
    """`rs train` checks every batch's masks on the host, before the upload, and names the tile: through the real dataset and
    DataLoader collation, for the uint8 masks of the device-augment path and the int64 masks of MaskToTensor."""
    from torch.utils.data import DataLoader

    from robosat_b200.tools.train import _MaskToUint8, check_mask_range

    coords = [(10, 20), (10, 21), (11, 20), (11, 21)]
    for sub in ("images", "labels"):
        for x, y in coords:
            os.makedirs(tmp_path / sub / "18" / str(x), exist_ok=True)
    for k, (x, y) in enumerate(coords):
        Image.fromarray(np.zeros((8, 8, 3), np.uint8)).save(tmp_path / "images" / "18" / str(x) / ("%d.png" % y))
        mask = np.zeros((8, 8), np.uint8)
        mask[2:5, 2:5] = 1
        if k == 2:
            mask[7, 7] = 5  # a stray palette index
        img = Image.fromarray(mask, mode="P")
        img.putpalette([0, 0, 0, 255, 255, 255] + [0] * (254 * 3))
        img.save(tmp_path / "labels" / "18" / str(x) / ("%d.png" % y))
    for mask_transform in (_MaskToUint8(), MaskToTensor()):
        transform = JointCompose([JointTransform(ImageToTensor(), mask_transform)])
        ds = SlippyMapTilesConcatenation([str(tmp_path / "images")], str(tmp_path / "labels"), transform)
        (images, masks, tiles), = list(DataLoader(ds, batch_size=4, shuffle=False))
        check_mask_range(masks, tiles, 6)  # 0..5 are all classes of a six-class dataset
        check_mask_range(masks[:2], tiles, 2)
        with pytest.raises(ValueError, match=r"tile 18/11/20 holds the value 5, but the dataset has the 2 classes 0\.\.1"):
            check_mask_range(masks, tiles, 2)
    with pytest.raises(ValueError, match="sample 1 of the batch holds the value -1"):
        check_mask_range(torch.tensor([[[0, 1]], [[-1, 0]]]), None, 2)
