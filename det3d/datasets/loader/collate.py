"""The collate of the info-file readers: pillarnext_b200.scenes.collate, whose batch the detector takes."""
from pillarnext_b200.scenes import collate

__all__ = ["collate"]
