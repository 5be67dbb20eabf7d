"""Filter banks of the Chebyshev path (see pygsp/filters/__init__.py:114-136)."""
from .filter import Filter  # noqa: F401
from .heat import Heat  # noqa: F401
from .mexicanhat import MexicanHat  # noqa: F401
from .approximations import (compute_cheby_coeff, cheby_op, cheby_rect,  # noqa: F401
                             compute_jackson_cheby_coeff, lanczos, lanczos_op)
