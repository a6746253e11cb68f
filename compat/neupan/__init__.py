"""`import neupan` shim: put this directory's parent (``compat/``) on PYTHONPATH and the reference's
entry script runs unchanged on the CUDA implementation:

    PYTHONPATH=/path/to/repo:/path/to/repo/compat python example/run_exp.py -e corridor -d diff

(`from neupan import neupan`, `neupan.blocks.PAN`, `neupan.robot.robot`, `neupan.util`, `neupan.configuration`).
"""
from neupan_b200 import configuration, util  # noqa: F401
from neupan_b200.neupan import neupan  # noqa: F401
