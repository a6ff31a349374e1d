"""Drop-in for the reference's CenterNet.py (ref testcenternet.py)."""
import _odt_path  # noqa: F401
from odt_b200.api import CenterNet  # noqa: F401
