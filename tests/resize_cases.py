"""Seeded source frames for the raw-frame resize goldens (tests/golden/make_golden_resize.py) and tests.

Each case is (name, seed, (frame_h, frame_w), (y0, x0, h, w), (H, W)): a frame of noise drawn from numpy's legacy RandomState
(bit-stable across numpy versions), the h x w window of it at (y0, x0) that is resized, and the target size.  A window smaller
than its frame is a pitched crop: its rows are frame_w * 3 bytes apart."""
import numpy as np

CASES = [
    ("vga", 101, (480, 640), None, (352, 352)),
    ("fullhd", 102, (1080, 1920), None, (352, 352)),
    ("voc500", 103, (375, 500), None, (352, 352)),
    ("up301", 104, (300, 301), None, (352, 352)),
    ("up90", 105, (100, 90), None, (352, 352)),
    ("hd_640", 106, (720, 1280), None, (640, 640)),
    ("odd_160x96", 107, (333, 517), None, (96, 160)),
    ("exact2x", 108, (704, 704), None, (352, 352)),
    ("w100", 109, (480, 640), None, (100, 100)),
    ("w37", 110, (480, 640), None, (101, 37)),
    ("w35", 111, (200, 300), None, (33, 35)),
    ("w350", 112, (1080, 1920), None, (352, 350)),
    ("w97", 113, (50, 70), None, (96, 97)),
    ("w11", 114, (77, 91), None, (13, 11)),
    ("identity", 115, (352, 352), None, (352, 352)),
    ("row_1xN", 116, (1, 517), None, (352, 352)),
    ("col_Nx1", 117, (333, 1), None, (352, 352)),
    ("pixel_1x1", 118, (1, 1), None, (7, 5)),
    ("upscale_big", 119, (12, 16), None, (960, 1280)),
    ("upscale_odd", 120, (37, 23), None, (500, 301)),
    ("crop", 121, (720, 1280), (97, 213, 401, 623), (352, 352)),
    ("crop_edge", 122, (480, 640), (0, 17, 480, 623), (96, 160)),
]

# the frames of the test.py known answers (img/000139.jpg, img/000004.jpg) as cv2.imread decodes them: tests/golden/frames_modelzoo.npz
MODELZOO_FRAMES = ("000139", "000004")


def frame(seed, shape):
    return np.random.RandomState(seed).randint(0, 256, size=(shape[0], shape[1], 3)).astype(np.uint8)


def case_input(case):
    """(full frame, the window that is resized, as a view into the frame)."""
    _, seed, shape, win, _ = case
    f = frame(seed, shape)
    if win is None:
        return f, f
    y0, x0, h, w = win
    return f, f[y0:y0 + h, x0:x0 + w]
