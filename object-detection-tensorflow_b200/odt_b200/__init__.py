"""odt_b200: H100-native (sm_90a) detection hot path behind the reference's
model API.  See DESIGN.md."""
from .api import FCOS, SSD300, SSD512, RetinaNet, YOLOv3  # noqa: F401
