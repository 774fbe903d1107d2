"""Drop-in counterpart of the reference Python binding (binding/python/multiverso/__init__.py:
``from .api import *; from .tables import *``), served by multiverso_b200: HBM tables and
sm_90a kernels when CUDA is present, the C++ host runtime otherwise."""
from .api import *      # noqa: F401,F403
from .tables import *   # noqa: F401,F403
