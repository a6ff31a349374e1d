"""Drop-in for the reference's PFPNetR.py (ref testpfpnet.py)."""
import _odt_path  # noqa: F401
from odt_b200.api import PFPNetR  # noqa: F401
