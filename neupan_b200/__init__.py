"""neupan_b200 -- H100-native implementation of NeuPAN's PAN hot path.

Mirrors the reference's public names for this path (``neupan.blocks.PAN`` / ``DUNE`` / ``NRMP`` /
``ObsPointNet``, ``neupan.robot.robot``, ``neupan.configuration``, ``neupan.util``) on top of a
C-ABI CUDA library (include/neupan_b200.h, neupan_b200/csrc).  Importing the package does not
need a GPU; running PAN does -- there is no CPU fallback.
"""
from . import configuration, util
from .robot import robot
from .blocks import DUNE, NRMP, PAN, InitialPath, ObsPointNet
from .neupan import neupan
from .scan import scan_to_points
from .ipath import InitialPathBatch
from .planner_batch import PlannerBatch
from .world import MixedPlanner, WorldBatch, pack_maps, rollout, run_episodes

__all__ = ["configuration", "util", "robot", "neupan", "PAN", "DUNE", "NRMP", "ObsPointNet", "InitialPath", "scan_to_points", "InitialPathBatch", "PlannerBatch", "WorldBatch", "MixedPlanner",
           "rollout", "pack_maps", "run_episodes"]
__version__ = "0.1.0"
