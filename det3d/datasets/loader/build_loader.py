"""build_dataloader of the reference (det3d/datasets/loader/build_loader.py), the import path of its tools/train.py:
pillarnext_b200.loader.build_dataloader, with collate_fn scenes.collate.  It takes the reference's arguments with two
differences: memory is pinned whenever CUDA is available, whatever pin_memory says (the trainer's host-to-device
copies are non-blocking), and a DistributedSampler is used when the process group has more than one rank (one rank
sees the whole dataset either way)."""
from pillarnext_b200.loader import build_dataloader

__all__ = ["build_dataloader"]
