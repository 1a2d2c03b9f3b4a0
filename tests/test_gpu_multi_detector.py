"""Several detectors in one SceneManager against the reference's own SceneManager (tests/golden/multi_detector_v1.json,
recorded by tests/golden/make_multi_detector_golden.py).  The detectors share one fused score pass whose feature mask
is the union of theirs: the cases run masks 5, 6, 11, 13 and 15, and a hash launch next to the fused pass.  Cut
lists and scene lists must be identical, metrics bit-exact (`hist_diff` within 1e-9), the CSV identical where no
`hist_diff` is in it."""

import json
import os

import pytest

from tests.golden_util import case_frames
from tests.test_gpu_parity import _check_stats

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "multi_detector_v1.json")
# the fused pass's feature mask of each case (F_HSV 1, F_BGRSUM 2, F_YHIST 4, F_EDGES 8, F_HASH 16)
MASKS = {"content_threshold_stats": 11, "content_histogram_133x99": 5, "threshold_histogram_stats": 6,
         "adaptive_hist_threshold_hash_360p": 31, "content_adaptive_shared_kernel": 13}


def _cases() -> list:
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def test_cases_cover_the_masks():
    assert {c["name"] for c in _cases()} == set(MASKS)
    assert any((c["gen"][1] * c["gen"][2]) % 16 == 15 for c in _cases())


def _detector(name, kw):
    from tests.test_gpu_parity import _build
    return _build({"det": name, "kw": kw})


@pytest.mark.parametrize("batch", [7, 64])
@pytest.mark.parametrize("name", list(MASKS))
def test_multi_detector_scene_manager_matches_reference(name, batch):
    from pyscenedetect_b200 import StatsManager
    from pyscenedetect_b200.scene_manager import SceneManager
    from pyscenedetect_b200.video import ArrayVideoStream
    case = next(c for c in _cases() if c["name"] == name)
    frames = case_frames(case)
    stats = StatsManager() if case["stats"] else None
    sm = SceneManager(stats, batch_size=batch)
    for det, kw in case["dets"]:
        sm.add_detector(_detector(det, kw))
    sm.auto_downscale = bool(case.get("auto_downscale"))
    if not sm.auto_downscale:
        sm.downscale = case.get("downscale", 1)
    assert sm.detect_scenes(ArrayVideoStream(frames, case["fps"])) == frames.shape[0]
    mask = 0
    for d in sm._detector_list:
        mask |= d.required_features()
    assert mask == MASKS[name]
    assert [c.frame_num for c in sm.get_cut_list()] == case["cuts"]
    assert [[a.frame_num, b.frame_num] for a, b in sm.get_scene_list()] == case["scene_list"]
    if stats is not None:
        _check_stats(case, stats, frames.shape[0])
