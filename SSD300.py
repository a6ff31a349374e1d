"""Drop-in for the reference's SSD300.py: `import SSD300 as net; net.SSD300(config, provider)`
(ref testSSD300.py:7,60).  The implementation lives in
object-detection-tensorflow_b200/odt_b200 (H100 kernels behind a C ABI)."""
import _odt_path  # noqa: F401
from odt_b200.api import SSD300  # noqa: F401
