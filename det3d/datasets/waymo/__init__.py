"""Drop-in `det3d.datasets.waymo` namespace (the reference's configs name det3d.datasets.waymo.waymo.WaymoDataset)."""
