"""Drop-in for the reference's YOLOv2.py (ref testYOLOv2.py:5,74)."""
import _odt_path  # noqa: F401
from odt_b200.api import YOLOv2  # noqa: F401
