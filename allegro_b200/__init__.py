"""allegro_b200: an H100 (sm_90a)-native implementation of Allegro's per-edge equivariant
hot path behind the NequIP/Allegro model and operator API.  See DESIGN.md."""
from . import data, o3, systems  # noqa: F401

__version__ = "0.1.0"
