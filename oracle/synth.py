"""Deterministic synthetic inputs.  The generator lives with the product package
(psam_b200/synth.py) so that bench.py's repo arm never imports anything under oracle/; the oracle-side tests and the
golden-vector generator use it through this re-export."""
import os
import sys

_PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "point-sam_b200")
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)

from psam_b200.synth import make_batch, make_cloud, make_prompts, make_region_masks  # noqa: E402,F401
