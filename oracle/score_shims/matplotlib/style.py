"""Stand-in for matplotlib.style (see plotnine/__init__.py next to this package)."""

from plotnine import _INERT  # the same inert stand-in


def __getattr__(name):
  return _INERT
