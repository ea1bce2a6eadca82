from .nusc import NuScenesDataset

__all__ = ["NuScenesDataset"]
