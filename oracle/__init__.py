"""CPU oracle for the PySceneDetect content-score hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under `pyscenedetect_b200/` may import this package;
only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline legs use it, as the
checker (or as the timed CPU baseline), never as the product path.

Two layers:

* `oracle.ref_detectors` - a restatement of the reference detectors' `process_frame`
  logic that makes *the same cv2 / numpy calls* as the reference
  (scenedetect/detectors/*.py, scenedetect/detector.py).  The pixel arithmetic of this
  path lives in third-party wheels that are not part of the reference (opencv-python
  4.13.0.92 and numpy 2.3.5 in this image; the reference pins neither,
  pyproject.toml:43-57), so the parity target is "what cv2/numpy in this image compute".
* `oracle.intmath` - a pure numpy/integer restatement of those cv2 primitives
  (BGR->HSV, BGR->Y, INTER_LINEAR resize, Canny, dilate, calcHist, normalize,
  compareHist) documenting the exact fixed-point arithmetic the CUDA kernels
  implement.  It is pinned against cv2 itself in tests/test_oracle_*.py (incl. the
  exhaustive 2^24-colour check).

Pinning: `tests/golden/make_golden.py` imports the real reference from a source checkout
and records per-frame metrics, cut lists and StatsManager CSV text for seeded synthetic
sequences; tests/test_oracle_golden.py checks `ref_detectors` against those fixtures
bit for bit.
"""
