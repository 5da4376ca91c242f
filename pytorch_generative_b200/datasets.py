"""Data path of the recipes (reference datasets.py:16-64, 160-187), device side.

The reference binarises / dequantises every image on DataLoader worker processes (`transforms.Compose` over PIL images)
and ships fp32 tensors to the GPU.  Here the loaders deliver the raw uint8 images (4x fewer host->device bytes) and the
stochastic transforms run on the device: `DeviceTransform` wraps a loader and applies, per batch, ToTensor's /255 scaling
followed by dynamic binarisation (Bernoulli(p = pixel), reference datasets.py:16-17), dequantisation
((255 x + U[0,1)) / 256, :20-21), the 28 -> 32 zero padding (:24-25) or CIFAR-10's per-channel normalisation
(transforms.Normalize with the means and standard deviations of :171-173).
"""

import os

import torch
from torch.nn import functional as F
from torch.utils import data

DATA_ROOT = os.environ.get("PG_DATA_ROOT", "/tmp/data")
CIFAR10_MEAN = (0.4914, 0.4822, 0.4465)
CIFAR10_STD = (0.2023, 0.1994, 0.2010)


def dynamically_binarize(x, generator=None):
    """x in [0, 1] -> Bernoulli(x) samples in {0, 1}, on x's device."""
    return torch.bernoulli(x, generator=generator)


def dequantize(x, generator=None):
    return (x * 255 + torch.rand(x.shape, device=x.device, generator=generator)) / 256


def resize_to_32(x):
    return F.pad(x, (2, 2, 2, 2))


def normalize(x, mean=CIFAR10_MEAN, std=CIFAR10_STD):
    """(x - mean[c]) / std[c] per channel of an NCHW batch, as transforms.Normalize computes it."""
    m = torch.tensor(mean, dtype=x.dtype, device=x.device).view(1, -1, 1, 1)
    s = torch.tensor(std, dtype=x.dtype, device=x.device).view(1, -1, 1, 1)
    return (x - m) / s


class DeviceTransform:
    """Iterates `loader`, moving each batch of uint8 (or float) images to `device` and applying the transforms there."""

    def __init__(self, loader, device, binarize=False, dequant=False, pad_to_32=False, seed=None, normalize=False):
        if binarize and dequant:
            raise ValueError("Cannot specify both dynamically_binarize and dequantize.")
        self.loader, self.device = loader, torch.device(device)
        self.binarize, self.dequant, self.pad_to_32, self.normalize = binarize, dequant, pad_to_32, normalize
        self.generator = None
        if seed is not None:
            self.generator = torch.Generator(device=self.device).manual_seed(seed)

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        for batch in self.loader:
            x, y = batch if isinstance(batch, (tuple, list)) else (batch, None)
            x = x.to(self.device, non_blocking=True)
            x = x.float() / 255 if x.dtype == torch.uint8 else x.float()
            if x.dim() == 3:
                x = x.unsqueeze(1)
            if self.binarize:
                x = dynamically_binarize(x, self.generator)
            if self.dequant:
                x = dequantize(x, self.generator)
            if self.pad_to_32:
                x = resize_to_32(x)
            if self.normalize:
                x = normalize(x)
            yield (x, y) if y is not None else x


class _RawImages(data.Dataset):
    """uint8 image tensor + labels as a Dataset (no per-item PIL round trip)."""

    def __init__(self, images, labels):
        self.images, self.labels = images, labels

    def __len__(self):
        return self.images.shape[0]

    def __getitem__(self, i):
        return self.images[i], self.labels[i]


def _torchvision_arrays(name, train, download):
    from torchvision import datasets as tv

    if name == "mnist":
        ds = tv.MNIST(DATA_ROOT, train=train, download=download)
        return ds.data.unsqueeze(1), ds.targets  # [N, 1, 28, 28] uint8
    ds = tv.CIFAR10(DATA_ROOT, train=train, download=download)
    return torch.from_numpy(ds.data).permute(0, 3, 1, 2).contiguous(), torch.tensor(ds.targets)  # [N, 3, 32, 32] uint8


def _loaders(name, batch_size, device, download, **transform):
    out = []
    for train in (True, False):
        images, labels = _torchvision_arrays(name, train, download)
        loader = data.DataLoader(_RawImages(images, labels), batch_size=batch_size, shuffle=train, pin_memory=True)
        out.append(DeviceTransform(loader, device, **transform))
    return tuple(out)


def get_mnist_loaders(batch_size, dynamically_binarize=False, dequantize=False, resize_to_32=False, device="cuda",
                      download=False):
    """(train_loader, test_loader) for MNIST — arguments of reference datasets.py:28-30; the transforms run on `device`.
    The files must already be under $PG_DATA_ROOT unless `download=True`."""
    return _loaders("mnist", batch_size, device, download, binarize=dynamically_binarize, dequant=dequantize,
                    pad_to_32=resize_to_32)


def get_cifar10_loaders(batch_size, device="cuda", download=False, normalize=False):
    """(train_loader, test_loader) for CIFAR-10 scaled to [0, 1] (reference datasets.py:160-187); `normalize`: then
    per-channel zero mean and unit variance, on `device`."""
    return _loaders("cifar10", batch_size, device, download, normalize=normalize)
