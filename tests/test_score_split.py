"""The Python twin of the fused pass's work split (tests/score_split.py) against the kernel source it mirrors, and
the frame counts it chooses for the GPU matrix (tests/test_gpu_score_matrix.py) against the cases they must reach."""

import os
import re

import pytest

from tests import score_split as S

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pyscenedetect_b200", "csrc",
                   "score_kernel.cu")


def _source() -> str:
    with open(SRC) as f:
        return f.read()


def _constexpr(src: str, name: str) -> int:
    m = re.search(rf"constexpr int {name} = (\d+);", src)
    assert m, f"{name} not found in score_kernel.cu"
    return int(m.group(1))


def test_constants_match_the_kernel():
    src = _source()
    assert _constexpr(src, "kWsConsumerWarps") == S.WS_CONSUMER_WARPS
    assert _constexpr(src, "kPxPerThread") == S.PX_PER_THREAD
    assert _constexpr(src, "kWsUnroll") == S.WS_UNROLL
    assert _constexpr(src, "kWsStages") == S.WS_STAGES
    assert "constexpr int kWsStripPx = kWsConsumers * kPxPerThread;" in src
    assert "constexpr int kWsConsumers = kWsConsumerWarps * 32;" in src
    # pick_chunks: the chunk cap, the short-walk cut-off and the cost it minimises
    body = src[src.index("static int pick_chunks("):]
    body = body[:body.index("\n}\n")]
    assert f"const int c_max = n_frames < {S.CHUNK_CAP} ? n_frames : {S.CHUNK_CAP};" in body
    assert f"if (longest < {S.SHORT_WALK} && c > 1) break;" in body
    assert "const long long per_cta = ((long long)n_strips * c + grid - 1) / grid;" in body
    assert "const long long cost = per_cta * (longest + 1);" in body
    assert "if (best_cost < 0 || cost < best_cost)" in body
    # launch_ws: chunks capped at the frame count, one CTA per SM at most
    assert "if (a.n_chunks > a.n_frames) a.n_chunks = a.n_frames;" in src
    assert "const int grid = (int)(items < sm_count ? items : sm_count);" in src
    # ws_item: chunk-fastest item order, halo only for HSV, slots padded to the unroll factor
    item = src[src.index("__device__ __forceinline__ WsItem ws_item("):]
    item = item[:item.index("\n}\n")]
    assert "const int chunk = item % a.n_chunks;" in item
    assert "const int strip = item / a.n_chunks;" in item
    assert "return (int)(((long long)c * n_frames) / n_chunks);" in src
    assert "const bool have_halo = (a.features & PSD_F_HSV) && (w.f0 > 0 || a.prev != nullptr);" in item
    assert "w.slots = (w.walked + kWsUnroll - 1) / kWsUnroll * kWsUnroll;" in item
    assert "for (int item = blockIdx.x; item < n_items; item += gridDim.x)" in src
    # the ws kernel takes P & ~15 pixels in strips, the tail kernel the rest
    assert "(p16 + kWsStripPx - 1) / kWsStripPx" in src


def test_split_known_shapes():
    # 1080p: 168 full strips and one of 9216 pixels (the kernel's own comment)
    s = S.split(1920 * 1080, 1, True, False, 132)
    assert s.n_strips == 169 and 1920 * 1080 - 168 * S.STRIP_PX == 9216
    assert S.split(15, 4, True, False, 132) is None
    one = S.split(128 * 96, 5, True, True, 132)
    assert one.n_strips == 1 and one.n_chunks == 1 and [it.walked for it in one.items] == [6]
    # without HSV no item walks a halo frame
    assert all(not it.halo for it in S.split(640 * 360, 300, False, True, 132).items)
    # chunks cover the frames exactly once and differ by at most one frame
    for n in (1, 7, 17, 100, 2048, 5000):
        s = S.split(1920 * 1080, n, True, False, 132)
        nfs = [it.nf for it in s.items if it.strip == 0]
        assert sum(nfs) == n and max(nfs) - min(nfs) <= 1


@pytest.mark.parametrize("sm_count", [132, 114, 78, 66])
def test_chosen_launches_reach_every_case(sm_count):
    from tests.test_gpu_score_matrix import GEOMETRIES, MIXED_CANDIDATES, MIXED_N_MAX
    reached = set()
    for w, h in GEOMETRIES:
        if w * h >= 16:
            launches = S.choose_launches(w * h, sm_count)
            got = S.coverage(w * h, launches, sm_count)
            assert S.required_cases() <= got, (w, h)
            reached |= got
    assert "few" in reached
    assert any(S.find_mixed_launch(w * h, sm_count, MIXED_N_MAX) for w, h in MIXED_CANDIDATES)


def test_matrix_geometries():
    from tests.test_gpu_score_matrix import GEOMETRIES
    assert {(w * h) % 16 for w, h in GEOMETRIES} == set(range(16))
    for w, h in [(1, 1), (15, 1), (1, 15), (128, 96), (769, 16), (535, 23), (1117, 11), (1920, 1080)]:
        assert (w, h) in GEOMETRIES
    assert any(w < 8 for w, h in GEOMETRIES) and any(h <= 2 for w, h in GEOMETRIES)
    assert any(S.split(w * h, 1, True, False, 132) and S.split(w * h, 1, True, False, 132).n_strips > 2
               for w, h in GEOMETRIES)
