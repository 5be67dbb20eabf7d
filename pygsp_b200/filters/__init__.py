"""Filter banks of the Chebyshev path (see pygsp/filters/__init__.py:114-136)."""
from .filter import Filter  # noqa: F401
from .abspline import Abspline  # noqa: F401
from .expwin import Expwin  # noqa: F401
from .gabor import Gabor  # noqa: F401
from .halfcosine import HalfCosine  # noqa: F401
from .heat import Heat  # noqa: F401
from .held import Held  # noqa: F401
from .itersine import Itersine  # noqa: F401
from .mexicanhat import MexicanHat  # noqa: F401
from .meyer import Meyer  # noqa: F401
from .modulation import Modulation  # noqa: F401
from .papadakis import Papadakis  # noqa: F401
from .rectangular import Rectangular  # noqa: F401
from .regular import Regular  # noqa: F401
from .simoncelli import Simoncelli  # noqa: F401
from .simpletight import SimpleTight  # noqa: F401
from .wave import Wave  # noqa: F401
from .approximations import (compute_cheby_coeff, cheby_op, cheby_rect,  # noqa: F401
                             compute_jackson_cheby_coeff, lanczos, lanczos_op)
