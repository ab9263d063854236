"""cczero-b200: H100-native Xiangqi self-play hot path behind the reference's
CChessPlayer / CChessModelAPI / SelfPlayWorker surface.

The directory name carries the reference's name and is not a Python identifier; import it as
`import cczero_b200` (the shim at the repository root) or via importlib.
"""
from .lib import CzLib, get_lib, CzError  # noqa: F401
