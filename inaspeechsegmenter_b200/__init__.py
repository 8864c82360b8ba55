"""inaspeechsegmenter_b200 -- H100-native (sm_90a) implementation of the
per-frame hot path of ina-foss/inaSpeechSegmenter behind the reference's own
API (``Segmenter``, ``seg2csv``; inaSpeechSegmenter/__init__.py:26-29).

Importing the package does not need a GPU; creating a ``Segmenter`` does (and
fails loudly without one: there is no CPU fallback).
"""
from .export_funcs import seg2csv, seg2textgrid      # noqa: F401
from .segmenter import Segmenter                      # noqa: F401

__version__ = '0.1.0+b200'
