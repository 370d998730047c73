"""`rs train`: same flags, configuration keys, log lines and checkpoint layout as robosat/tools/train.py:42-276.

Everything in the inner loop (train.py:163-201) runs on librsb200.so: the train-mode forward and the backward of the
network (`UNet` -> `UNetTrainEngine`), the losses (sort/scan + closed-form gradient kernels), the metrics (one counting
kernel per batch, one read-back per epoch instead of 4 syncs per sample) and Adam (one fused kernel over a flat arena).
Validation runs on the inference plan.

With several GPUs the tool spawns one process per GPU (the command line is unchanged; `RSB_GPUS` overrides the count):
rank 0's weights are broadcast once, every rank trains on its shard of each epoch (DistributedSampler), the flat fp32
gradient arena is summed with ONE NCCL all-reduce per step (loss pre-scaled by 1/world), BatchNorm statistics stay per
rank like DataParallel's replicas, rank 0 logs and writes the checkpoints (replaces `nn.DataParallel`, train.py:69).
"""

import argparse
import collections
import os
import sys

import torch
from PIL import Image

from robosat_b200.config import load_config
from robosat_b200.datasets import SlippyMapTilesConcatenation
from robosat_b200.log import Log
from robosat_b200.losses import CrossEntropyLoss2d, FocalLoss2d, LovaszLoss2d, mIoULoss2d
from robosat_b200.metrics import Metrics
from robosat_b200.optim import Adam, LossScaler
from robosat_b200.transforms import (ConvertImageMode, ImageToTensor, JointCompose, JointRandomHorizontalFlip, JointRandomRotation,
                                     JointTransform, MaskToTensor)
from robosat_b200.unet import UNet


def add_parser(subparser):
    parser = subparser.add_parser("train", help="trains model on dataset", formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    parser.add_argument("--model", type=str, required=True, help="path to model configuration file")
    parser.add_argument("--dataset", type=str, required=True, help="path to dataset configuration file")
    parser.add_argument("--checkpoint", type=str, required=False, help="path to a model checkpoint (to retrain)")
    parser.add_argument("--resume", type=bool, default=False, help="resume training or fine-tuning (if checkpoint)")  # type=bool quirk kept (train.py:50)
    parser.add_argument("--workers", type=int, default=0, help="number of workers pre-processing images")
    parser.set_defaults(func=main)


def _plot(path, history):
    try:  # matplotlib is optional here; the reference requires it (utils.py)
        import matplotlib

        matplotlib.use("Agg")
        import matplotlib.pyplot as plt
    except ImportError:
        return
    plt.figure()
    n = max(map(len, history.values()))
    plt.xticks(range(n), [v + 1 for v in range(n)])
    plt.grid()
    for values in history.values():
        plt.plot(values)
    plt.xlabel("epoch")
    plt.legend(list(history))
    plt.savefig(path, format="png")
    plt.close()


class _Normalize:
    def __init__(self, mean, std):
        self.mean = torch.tensor(mean).view(3, 1, 1)
        self.std = torch.tensor(std).view(3, 1, 1)

    def __call__(self, t):
        return (t - self.mean) / self.std


class _ResizeCrop:
    """Resize(target, mode) followed by CenterCrop(target) on a PIL image (train.py:250-251)."""

    def __init__(self, size, mode):
        self.size, self.mode = size, mode

    def __call__(self, image):
        if image.size != self.size:
            image = image.resize(self.size, self.mode)
        return image


DEVICE_AUGMENT = os.environ.get("RSB_DEVICE_AUGMENT", "1") != "0"


class _MaskToUint8:
    def __call__(self, image):
        import numpy as np

        return torch.from_numpy(np.array(image, dtype=np.uint8))


def get_dataset_loaders(model, dataset, workers, rank=0, world=1):
    from torch.utils.data import DataLoader
    from torch.utils.data.distributed import DistributedSampler

    target_size = (model["common"]["image_size"],) * 2
    batch_size = model["common"]["batch_size"]
    if world > 1 and os.environ.get("RSB_BATCH_PER_GPU", "0") != "1":
        # `batch_size` of the TOML is the GLOBAL batch, split over the GPUs like nn.DataParallel's scatter does in the reference
        # (train.py:69,180), so lr / logged losses / dropped ragged tails stay comparable for the same configuration;
        # RSB_BATCH_PER_GPU=1 gives every rank the full batch_size instead (BASELINE cfg 5 states its batch per GPU).
        batch_size = max(1, batch_size // world)
    path = dataset["common"]["dataset"]
    mean, std = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
    if DEVICE_AUGMENT:
        # the workers only decode and resize; the random flip / quarter turns (train.py:253-258), ToTensor and Normalize run on the
        # device on the whole uint8 batch (robosat_b200/augment.py, rsb_augment_dihedral, the pre-pass of the network)
        from robosat_b200.transforms import ImageToUint8Tensor

        transform = JointCompose([
            JointTransform(ConvertImageMode("RGB"), ConvertImageMode("P")),
            JointTransform(_ResizeCrop(target_size, Image.BILINEAR), _ResizeCrop(target_size, Image.NEAREST)),
            JointTransform(ImageToUint8Tensor(), _MaskToUint8()),
        ])
    else:
        transform = JointCompose([
            JointTransform(ConvertImageMode("RGB"), ConvertImageMode("P")),
            JointTransform(_ResizeCrop(target_size, Image.BILINEAR), _ResizeCrop(target_size, Image.NEAREST)),
            JointRandomHorizontalFlip(0.5),
            JointRandomRotation(0.5, 90),
            JointRandomRotation(0.5, 90),
            JointRandomRotation(0.5, 90),
            JointTransform(ImageToTensor(), MaskToTensor()),
            JointTransform(_Normalize(mean, std), None),
        ])
    train_dataset = SlippyMapTilesConcatenation([os.path.join(path, "training", "images")], os.path.join(path, "training", "labels"), transform)
    val_dataset = SlippyMapTilesConcatenation([os.path.join(path, "validation", "images")], os.path.join(path, "validation", "labels"), transform)
    assert len(train_dataset) > 0, "at least one tile in training dataset"
    assert len(val_dataset) > 0, "at least one tile in validation dataset"
    if world > 1:
        # Validation sees exactly the tiles the reference's single loader (train.py:265-268: batch_size, drop_last=True) sees:
        # with the TOML batch split over the ranks (batch_size = B / world here) rank r takes tiles r, r + world, ... of the
        # first floor(n / world) * world, and its loader keeps floor(floor(n / world) / (B / world)) = floor(n / B) batches --
        # together the first floor(n / B) * B tiles, each once (tests/test_host_logic.py).
        ts = DistributedSampler(train_dataset, num_replicas=world, rank=rank, shuffle=True, drop_last=True)
        vs = DistributedSampler(val_dataset, num_replicas=world, rank=rank, shuffle=False, drop_last=True)
        train_loader = DataLoader(train_dataset, batch_size=batch_size, sampler=ts, drop_last=True, num_workers=workers)
        val_loader = DataLoader(val_dataset, batch_size=batch_size, sampler=vs, drop_last=True, num_workers=workers)
    else:
        train_loader = DataLoader(train_dataset, batch_size=batch_size, shuffle=True, drop_last=True, num_workers=workers)
        val_loader = DataLoader(val_dataset, batch_size=batch_size, shuffle=False, drop_last=True, num_workers=workers)
    return train_loader, val_loader


def check_mask_range(masks, tiles, num_classes):
    """Reject a batch whose label masks hold a value outside [0, num_classes), naming the first such tile. Runs on the host batch,
    where the bytes already are, before the upload: the loss kernels leave such pixels out instead of failing, so a label PNG with
    a stray palette index would otherwise train on silently (the reference raises "Target ... is out of bounds" there)."""
    flat = masks.reshape(masks.shape[0], -1)
    lo, hi = flat.amin(dim=1), flat.amax(dim=1)
    bad = ((lo < 0) | (hi >= num_classes)).nonzero()
    if bad.numel() == 0:
        return
    i = int(bad[0])
    name = "sample %d of the batch" % i
    try:  # the collated [Tile(x=[...], y=[...], z=[...])] of SlippyMapTilesConcatenation
        tile = tiles[0]
        name = "tile %d/%d/%d" % (int(tile.z[i]), int(tile.x[i]), int(tile.y[i]))
    except (AttributeError, IndexError, KeyError, TypeError):
        pass
    value = int(hi[i]) if int(hi[i]) >= num_classes else int(lo[i])
    raise ValueError("label mask of %s holds the value %d, but the dataset has the %d classes 0..%d" % (name, value, num_classes, num_classes - 1))


def _epoch(loader, num_classes, device, net, criterion, optimizer=None, world=1, scaler=None):
    """One pass of train() (train.py:163-201) or validate() (train.py:204-238): same bookkeeping, batched metrics."""
    from robosat_b200.dist import allreduce_sum_

    training = optimizer is not None
    num_samples, running_loss = 0, torch.zeros((), dtype=torch.float32, device=device)
    metrics = Metrics(range(num_classes))
    net.train() if training else net.eval()
    augmenter = None
    for images, masks, tiles in loader:
        check_mask_range(masks, tiles, num_classes)
        images = images.to(device, non_blocking=True)
        masks = masks.to(device, non_blocking=True)
        if images.dtype == torch.uint8:
            # raw uint8 NHWC tiles + uint8 masks from the workers: flip / rotate the batch on the device (the reference applies
            # the same random transform to the training AND the validation set, train.py:248-268), masks become int64
            if augmenter is None:
                from robosat_b200.augment import DeviceAugmenter

                augmenter = DeviceAugmenter(images.shape[0], images.shape[1], device=device)
            assert images.shape[1:3] == masks.shape[1:], "resolutions for images and masks are in sync"
            images, masks = augmenter.augment(images.contiguous(), masks.contiguous())
            sizes_ok = images.shape[1:3] == masks.shape[1:]
        else:
            sizes_ok = images.size()[2:] == masks.size()[1:]
        assert sizes_ok, "resolutions for images and masks are in sync"
        num_samples += int(images.size(0))
        if training:
            optimizer.zero_grad()
            outputs = net(images)
        else:
            with torch.no_grad():
                outputs = net(images)
        assert outputs.size()[2:] == masks.size()[1:], "resolutions for predictions and masks are in sync"
        assert outputs.size()[1] == num_classes, "classes for predictions and dataset are in sync"
        loss = criterion(outputs, masks)
        if training:
            (loss / world if world > 1 else loss).backward()
            allreduce_sum_(optimizer.flat_grad, world)  # no-op on one GPU
            optimizer.step()  # skipped on the device if the (summed) gradients are not finite: every rank takes the same decision
            if scaler is not None:
                scaler.update()
        running_loss += loss.detach()  # stays on the device: one read-back per epoch instead of one per batch
        metrics.add_batch(masks, outputs.detach())
    if world > 1:
        import torch.distributed as dist

        # epoch totals over all ranks: 4 confusion counts + loss sum + sample count, one small all-reduce per epoch
        counts = torch.tensor(metrics._counts(), dtype=torch.float64, device=device)
        extra = torch.stack([running_loss.double(), torch.tensor(float(num_samples), dtype=torch.float64, device=device)])
        both = torch.cat([counts, extra])
        dist.all_reduce(both)
        metrics._host = [int(v) for v in both[:4].tolist()]
        return {"loss": both[4].item() / both[5].item(), "miou": metrics.get_miou(), "fg_iou": metrics.get_fg_iou(), "mcc": metrics.get_mcc()}
    return {"loss": running_loss.item() / num_samples, "miou": metrics.get_miou(), "fg_iou": metrics.get_fg_iou(), "mcc": metrics.get_mcc()}


def main(args):
    model = load_config(args.model)
    if not model["common"]["cuda"]:
        sys.exit("Error: robosat_b200 runs on CUDA devices only; set cuda = true in the model configuration")
    if not torch.cuda.is_available():
        sys.exit("Error: CUDA requested but not available")
    world = int(os.environ.get("RSB_GPUS", torch.cuda.device_count()))
    world = max(1, min(world, torch.cuda.device_count()))
    if world == 1:
        _run(0, 1, args, 0)
    else:
        import socket

        import torch.multiprocessing as mp

        with socket.socket() as s:
            s.bind(("127.0.0.1", 0))
            port = s.getsockname()[1]
        mp.spawn(_run, args=(world, args, port), nprocs=world, join=True)


def _run(rank, world, args, port):
    model = load_config(args.model)
    dataset = load_config(args.dataset)
    torch.cuda.set_device(rank)
    device = torch.device("cuda", rank)
    if world > 1:
        import torch.distributed as dist

        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", str(port))
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=device)
    os.makedirs(model["common"]["checkpoint"], exist_ok=True)

    num_classes = len(dataset["common"]["classes"])
    net = torch.nn.DataParallel(UNet(num_classes), device_ids=[rank])  # keeps the `module.` checkpoint prefix (train.py:69)
    net = net.to(device)

    try:
        weight = torch.Tensor(dataset["weights"]["values"])
    except KeyError:
        if model["opt"]["loss"] in ("CrossEntropy", "mIoU", "Focal"):
            sys.exit("Error: The loss function used, need dataset weights values")

    optimizer = Adam(net.parameters(), lr=model["opt"]["lr"])
    optimizer.mark_used([not n.startswith("module.resnet.fc.") for n, _ in net.named_parameters()])
    scaler = LossScaler(net, optimizer)

    resume = 0
    if args.checkpoint:
        chkpt = torch.load(args.checkpoint, map_location="cpu")
        net.load_state_dict(chkpt["state_dict"])
        if args.resume:
            optimizer.load_state_dict(chkpt["optimizer"])
            resume = chkpt["epoch"]
    if world > 1:
        # every rank starts from rank 0's weights and buffers: one broadcast of the flat state (the reference re-broadcasts
        # them on every forward through DataParallel.replicate)
        from robosat_b200.dist import broadcast_state_dict

        synced = broadcast_state_dict(net.state_dict() if rank == 0 else None, net.state_dict(), device)
        with torch.no_grad():
            for k, v in net.state_dict().items():
                v.copy_(synced[k])

    loss_name = model["opt"]["loss"]
    if loss_name == "CrossEntropy":
        criterion = CrossEntropyLoss2d(weight=weight).to(device)
    elif loss_name == "mIoU":
        criterion = mIoULoss2d(weight=weight).to(device)
    elif loss_name == "Focal":
        criterion = FocalLoss2d(weight=weight).to(device)
    elif loss_name == "Lovasz":
        criterion = LovaszLoss2d().to(device)
    else:
        sys.exit("Error: Unknown [opt][loss] value !")

    train_loader, val_loader = get_dataset_loaders(model, dataset, args.workers, rank, world)
    num_epochs = model["opt"]["epochs"]
    if resume >= num_epochs:
        sys.exit("Error: Epoch {} set in {} already reached by the checkpoint provided".format(num_epochs, args.model))

    history = collections.defaultdict(list)
    log = Log(os.path.join(model["common"]["checkpoint"], "log" if rank == 0 else "log.rank%d" % rank), out=sys.stdout if rank == 0 else None)
    log.log("--- Hyper Parameters on Dataset: {} ---".format(dataset["common"]["dataset"]))
    log.log("Batch Size:\t {}".format(model["common"]["batch_size"]))
    log.log("Image Size:\t {}".format(model["common"]["image_size"]))
    log.log("Learning Rate:\t {}".format(model["opt"]["lr"]))
    log.log("Loss function:\t {}".format(model["opt"]["loss"]))
    if "weight" in locals():
        log.log("Weights :\t {}".format(dataset["weights"]["values"]))
    log.log("---")

    fg = dataset["common"]["classes"][1]
    for epoch in range(resume, num_epochs):
        log.log("Epoch: {}/{}".format(epoch + 1, num_epochs))
        if world > 1:
            train_loader.sampler.set_epoch(epoch)
        train_hist = _epoch(train_loader, num_classes, device, net, criterion, optimizer, world=world, scaler=scaler)
        if scaler.overflows:
            log.log("loss scale {:g} ({} overflow steps skipped so far)".format(scaler.scale, optimizer.skipped_steps()))
        log.log("Train    loss: {:.4f}, mIoU: {:.3f}, {} IoU: {:.3f}, MCC: {:.3f}".format(
            train_hist["loss"], train_hist["miou"], fg, train_hist["fg_iou"], train_hist["mcc"]))
        for k, v in train_hist.items():
            history["train " + k].append(v)
        val_hist = _epoch(val_loader, num_classes, device, net, criterion, world=world)
        log.log("Validate loss: {:.4f}, mIoU: {:.3f}, {} IoU: {:.3f}, MCC: {:.3f}".format(
            val_hist["loss"], val_hist["miou"], fg, val_hist["fg_iou"], val_hist["mcc"]))
        for k, v in val_hist.items():
            history["val " + k].append(v)
        if rank == 0:
            _plot(os.path.join(model["common"]["checkpoint"], "history-{:05d}-of-{:05d}.png".format(epoch + 1, num_epochs)), history)
            states = {"epoch": epoch + 1, "state_dict": net.state_dict(), "optimizer": optimizer.state_dict()}
            torch.save(states, os.path.join(model["common"]["checkpoint"], "checkpoint-{:05d}-of-{:05d}.pth".format(epoch + 1, num_epochs)))
    if world > 1:
        import torch.distributed as dist

        dist.barrier()
        dist.destroy_process_group()
