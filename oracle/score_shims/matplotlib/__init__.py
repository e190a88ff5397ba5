"""Stand-in for matplotlib (see plotnine/__init__.py next to this package): style and pyplot calls do nothing."""

from plotnine import _INERT  # the same inert stand-in

style = _INERT


def __getattr__(name):
  return _INERT
