"""Drop-in `det3d.datasets` namespace: the data-pipeline classes the reference's dataset configs name by `_target_`."""
