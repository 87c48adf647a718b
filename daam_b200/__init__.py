"""daam_b200 -- H100-native cross-attention heat-map extraction behind the castorini/daam API.

``from daam_b200 import trace, set_seed`` is the drop-in for ``from daam import trace, set_seed`` on the hot path
(reference export surface: the reference's ``daam/__init__.py:1-6``)."""
from ._version import __version__
from .evaluate import *     # noqa: F401,F403
from .experiment import *   # noqa: F401,F403
from .heatmap import *   # noqa: F401,F403
from .hook import *      # noqa: F401,F403
from .utils import *     # noqa: F401,F403
from .trace import *     # noqa: F401,F403
from .distributed import shard_prompts, gather_heat_maps   # noqa: F401
