"""The image-file dataset of the device loader's tests (tests/golden/make_golden_loader.py writes tests/golden/loader_cases.npz).

build(root) writes the dataset into the directory root from the existing fixtures: each listed path is "<group>/<case>.<ext>",
read from
  base/     jpeg_cases.npz "jpg_<case>": cv2's baseline files, EXIF orientations, grey, restart intervals, the 1080p frame;
  unsup/    jpeg_cases.npz "bad_<case>": the files outside the decoder's subset that cv2 reads (the fallback path);
  cut/      jpeg_cases.npz "cut_<case>": a baseline file cut inside its scan (flagged; cv2 reads it);
  prog/     jpeg_progressive.npz "jpg_<case>" (.jpeg): progressive files;
  pdamaged/ jpeg_progressive.npz "jpg_<case>": damaged progressive files that are flagged and that cv2 reads;
  photos/   tests/golden/<case>.jpg: the reference's two photos;
  set.v1/   loader_cases.npz "png" / "bmp": a PNG and a BMP cv2 wrote.
The list file is "list.txt" with these relative paths (the reference's label rule cuts a path at its first '.', so the tests run
from root, whose own path may hold dots).  Label files follow that rule, so both files in "set.v1" share "set.txt".  Labels are
seeded rows "cls cx cy w h"; photos/000139.txt is empty.

The npz holds "names" (the listed paths, in order), "png", "bmp", "frame_<sha256 hex of the file>" (cv2.imdecode's frame of every
file the device does not decode or flags: tests inject them as the fallback reader, since cv2 need not be installed), "sha_<W>x<H>"
([n, 32] SHA-256 of each TensorDataset(..., imgaug=False) item at that size), and per batch size B in BATCHES "targets_b<B>" (the
SHA-256 of each collate_fn targets tensor of the files in order, [nbatches, 32])."""
import hashlib
import os

import numpy as np

SIZES = ((352, 352), (320, 192))    # (W, H)
BATCHES = (16, 7)
LIST = "list.txt"

PROG = ["cv2_q50_420", "cv2_q95_444", "cv2_q50_grey", "cv2_q1_411", "cv2_rst7_420", "cv2_size1x17_422", "cv2_exif6_II",
        "cv2_exif8_MM", "pil_sub2_q50", "pil_grey", "tx_cv2_000004", "tx_seeded_000139", "script_ac_420_0", "enc_eob_past_segment"]
PROG_DAMAGED = ["corrupt_refinement_0", "corrupt_refinement_1", "corrupt_refinement_2", "corrupt_run_past_band",
                "rst_renumbered_in_refinement"]
PHOTOS = ("000004", "000139")
EMPTY_LABEL = "photos/000139"


def sha(b):
    return hashlib.sha256(b).hexdigest()


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def file_bytes(golden_dir, name, loader_npz, jpeg_npz=None, prog_npz=None):
    """The bytes of listed path `name`."""
    group, base = name.split("/", 1)
    case = base.rsplit(".", 1)[0]
    jpeg_npz = jpeg_npz if jpeg_npz is not None else np.load(os.path.join(golden_dir, "jpeg_cases.npz"))
    prog_npz = prog_npz if prog_npz is not None else np.load(os.path.join(golden_dir, "jpeg_progressive.npz"))
    if group == "base":
        return jpeg_npz["jpg_" + case].tobytes()
    if group == "unsup":
        return jpeg_npz["bad_" + case].tobytes()
    if group == "cut":
        return jpeg_npz["cut_" + case].tobytes()
    if group in ("prog", "pdamaged"):
        return prog_npz["jpg_" + case].tobytes()
    if group == "photos":
        with open(os.path.join(golden_dir, case + ".jpg"), "rb") as f:
            return f.read()
    if group == "set.v1":
        return loader_npz[base.rsplit(".", 1)[1]].tobytes()
    raise ValueError(name)


def label_text(rng, stem):
    if stem == EMPTY_LABEL:
        return ""
    rows = []
    for _ in range(int(rng.integers(1, 6))):
        cx, cy, w, h = rng.uniform(0.05, 0.95, 4)
        rows.append("%d %.6f %.6f %.6f %.6f\n" % (int(rng.integers(0, 80)), cx, cy, w, h))
    return "".join(rows)


def build(root, names, golden_dir, loader_npz):
    """Writes the dataset of `names` under root; returns {path: bytes}."""
    jpeg_npz = np.load(os.path.join(golden_dir, "jpeg_cases.npz"))
    prog_npz = np.load(os.path.join(golden_dir, "jpeg_progressive.npz"))
    rng = np.random.default_rng(20261017)
    out, labels = {}, set()
    for name in names:
        data = file_bytes(golden_dir, name, loader_npz, jpeg_npz, prog_npz)
        os.makedirs(os.path.join(root, os.path.dirname(name)), exist_ok=True)
        with open(os.path.join(root, name), "wb") as f:
            f.write(data)
        out[name] = data
        stem = name.split(".")[0]                 # the reference's label rule
        if stem not in labels:
            labels.add(stem)
            with open(os.path.join(root, stem + ".txt"), "w") as f:
                f.write(label_text(rng, stem))
    with open(os.path.join(root, LIST), "w") as f:
        f.write("".join(n + "\n" for n in names))
    return out


def load(golden_dir):
    z = np.load(os.path.join(golden_dir, "loader_cases.npz"))
    return z, [str(n) for n in z["names"]]


def fallback_reader(z):
    """A fallback reader that returns cv2's recorded frame of a file (by its bytes), for runs without cv2.  The frames are read
    out of the npz here, so loader workers forked later share no open file."""
    frames = {k: z[k] for k in z.files if k.startswith("frame_")}

    def read(data):
        key = "frame_" + sha(bytes(data))
        if key not in frames:
            raise KeyError("no recorded cv2 frame for this file (sha256 %s)" % key[6:])
        return frames[key]
    return read
