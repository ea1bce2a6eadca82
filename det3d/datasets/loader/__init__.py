"""Drop-in `det3d.datasets.loader` namespace: the reference's build_dataloader and collate (tools/train.py imports
det3d.datasets.loader.build_loader.build_dataloader)."""
