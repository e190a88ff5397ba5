"""Stand-in for plotnine, which the reference's analysis modules import for their plots.

Scoring draws nothing: every attribute is a callable that accepts anything and returns the stand-in itself, so the
module-level theme calls of utils/plotting.py run and do nothing.  It holds no arithmetic.
"""


class _Inert:

  def __call__(self, *args, **kwargs):
    return self

  def __getattr__(self, name):
    return self

  def __add__(self, other):
    return self

  __radd__ = __add__


_INERT = _Inert()


def __getattr__(name):
  return _INERT
