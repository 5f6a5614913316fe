"""Writes turbo_lut.npz: OpenCV's COLORMAP_TURBO table, the last step of the reference's depth colourmap (utils::apply_colormap_to_depth).

    lut_bgr  uint8 [256,3]  cv2.applyColorMap of the values 0..255, as OpenCV returns it (BGR)

The GPU tests compare the frames kernel with tests/render_frames_oracle.py, which reads this table, so the GPU machine needs no OpenCV.
Run from the repository root: python tests/golden/make_turbo_lut.py"""
import os

import cv2
import numpy as np


def turbo_lut_bgr():
    return cv2.applyColorMap(np.arange(256, dtype=np.uint8).reshape(256, 1), cv2.COLORMAP_TURBO).reshape(256, 3)


if __name__ == "__main__":
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "turbo_lut.npz"), lut_bgr=turbo_lut_bgr())
