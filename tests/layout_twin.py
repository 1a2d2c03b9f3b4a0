"""numpy twin of psd_gather_bgr: the bytes a psd_frame_layout names, as packed BGR24."""

import numpy as np


def gather_twin(buf: np.ndarray, offset: int, layout, n: int, w: int, h: int) -> np.ndarray:
    """Frames of `layout` (frame, row, pixel, channel byte strides) whose base is byte `offset` of the 1-D uint8
    array `buf` -> (n, h, w, 3) BGR.  Negative and zero strides are read as the kernel reads them."""
    fs, rs, ps, cs = (int(s) for s in layout)
    assert buf.ndim == 1 and buf.dtype == np.uint8 and buf.strides == (1,)
    # every byte the layout names lies inside buf
    lo = offset + sum(min(0, s * (d - 1)) for s, d in zip((fs, rs, ps, cs), (n, h, w, 3)))
    hi = offset + sum(max(0, s * (d - 1)) for s, d in zip((fs, rs, ps, cs), (n, h, w, 3)))
    assert 0 <= lo and hi < buf.size, (lo, hi, buf.size)
    view = np.lib.stride_tricks.as_strided(buf[offset:], shape=(n, h, w, 3), strides=(fs, rs, ps, cs),
                                           writeable=False)
    return np.array(view)
