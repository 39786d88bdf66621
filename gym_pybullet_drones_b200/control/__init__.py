from .BaseControl import BaseControl  # noqa: F401
from .DSLPIDControl import DSLPIDControl  # noqa: F401
from .MRAC import MRAC  # noqa: F401
