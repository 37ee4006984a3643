"""sam_road_b200 -- H100-native (sm_90a) implementation of the tiled-inference hot path of
htcr/sam_road behind the reference's own Python API.  See DESIGN.md / INTEGRATION.md."""
from .model import SAMRoad  # noqa: F401

__all__ = ["SAMRoad"]
