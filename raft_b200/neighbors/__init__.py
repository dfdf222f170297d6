"""Mirror of the (removed) ``pylibraft.neighbors`` entry points that sit directly behind the distance path, and
``radius_neighbors`` and ``kernel_density``, project APIs on the same path, and ``ball_cover``, exact low-dimensional
search by the random ball cover."""
from . import ball_cover  # noqa: F401
from . import brute_force  # noqa: F401
from . import epsilon_neighborhood  # noqa: F401
from . import radius  # noqa: F401
from .epsilon_neighborhood import eps_neighbors_l2sq  # noqa: F401
from .kernel_density import kernel_density  # noqa: F401
from .radius import radius_neighbors  # noqa: F401
