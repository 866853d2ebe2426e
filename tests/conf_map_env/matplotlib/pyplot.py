"""TEST INFRASTRUCTURE - `matplotlib.pyplot.get_cmap` of the stand-in (see __init__.py)."""
from . import get_cmap  # noqa: F401
