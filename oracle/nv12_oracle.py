"""CPU oracle of the NV12 input path — TEST INFRASTRUCTURE ONLY (tests/).

An NV12 frame is uint8 [3h/2, w]: h rows of luma Y, then h/2 rows of interleaved chroma U, V at half resolution in both axes.  The
reference's frames are RGB, so an NV12 frame enters it as PreprocessorX.process(cv2.cvtColor(nv12, cv2.COLOR_YUV2RGB_NV12), size);
cvtColor(COLOR_YUV2RGB_NV12) followed by COLOR_RGB2BGR gives the bytes of COLOR_YUV2BGR_NV12.  That conversion is restated here
from OpenCV's published algorithm (modules/imgproc/src/color_yuv.simd.hpp, YUV420sp2RGB8Invoker: BT.601 limited range in 20-bit
fixed point, nearest chroma):
  * Y' = max(0, Y - 16) * 1220542, u = U - 128, v = V - 128, with U, V of pixel (y, x) at chroma row y >> 1, column x & ~1;
  * R = (Y' + 1673527 v + 2^19) >> 20, G = (Y' - 852492 v - 409993 u + 2^19) >> 20, B = (Y' + 2116026 u + 2^19) >> 20, each
    clamped to 0..255;
and the letterbox is preprocess_oracle.letterbox on the BGR frame.  Pinned: tests/test_nv12.py checks it bit for bit against the
cv2 installed in the image (4.13)."""
import numpy as np

import preprocess_oracle as po


def nv12_to_bgr(nv12):
    """cv2.cvtColor(nv12, cv2.COLOR_YUV2BGR_NV12) for uint8 [3h/2, w] (h, w even) -> uint8 [h, w, 3]."""
    h, w = nv12.shape[0] * 2 // 3, nv12.shape[1]
    y = nv12[:h].astype(np.int64)
    uv = nv12[h:].reshape(h // 2, w // 2, 2).astype(np.int64)
    u = np.repeat(np.repeat(uv[..., 0], 2, 0), 2, 1) - 128
    v = np.repeat(np.repeat(uv[..., 1], 2, 0), 2, 1) - 128
    yy = np.maximum(0, y - 16) * 1220542
    half = 1 << 19
    b = (yy + 2116026 * u + half) >> 20
    g = (yy - 852492 * v - 409993 * u + half) >> 20
    r = (yy + 1673527 * v + half) >> 20
    return np.stack([b, g, r], -1).clip(0, 255).astype(np.uint8)


def letterbox_nv12(nv12, input_size, pad=114):
    """-> (uint8 [Hin, Win, 3] BGR, r): the SOT/VOS preprocessor's output for the RGB frame cv2 converts nv12 to."""
    return po.letterbox(nv12_to_bgr(nv12), input_size, swap_rb=False, pad=pad)
