"""The device loader without a GPU: FileDataset's checks and label rule (utils/device_data.py, after utils/datasets.py:71-129),
collate_files in a worker-like process (no CUDA call; refused files to the fallback reader; collate_fn's targets as the
reference's own, tests/golden/loader_cases.npz), parse_jpeg(strict=False), and the argument checks of yfv2_jpeg_decode_resize."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

import yfv2  # noqa: F401  (registers the package dir)
import loader_cases as lc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden(golden_dir):
    return lc.load(golden_dir)


@pytest.fixture()
def dataset(golden, golden_dir, tmp_path, monkeypatch):
    z, names = golden
    files = lc.build(str(tmp_path), names, golden_dir, z)
    monkeypatch.chdir(tmp_path)
    return z, names, files


def test_file_dataset_items_and_label_rule(dataset):
    from utils.device_data import FileDataset, label_path
    z, names, files = dataset
    ds = FileDataset(lc.LIST, 352, 352)
    assert ds.data_list == names and len(ds) == len(names)
    for i in (0, names.index("set.v1/seeded.png"), names.index(lc.EMPTY_LABEL + ".jpg")):
        data, label = ds[i]
        assert data == files[names[i]]
        assert label.dtype.is_floating_point and str(label.dtype) == "torch.float32"
    assert label_path("set.v1/seeded.png") == "set.txt" and label_path("prog/a.jpeg") == "prog/a.txt"
    assert label_path("./x/y.jpg") == ".txt"                          # the rule cuts at the first '.', wherever it is
    _, empty = ds[names.index(lc.EMPTY_LABEL + ".jpg")]
    assert tuple(empty.shape) == (0,)
    _, rows = ds[names.index("set.v1/seeded.bmp")]
    assert rows.shape[1] == 6 and (rows[:, 0] == 0).all()
    with open("set.txt") as f:
        want = np.array([[0] + line.split() for line in f.read().splitlines()], dtype=np.float32)
    assert np.array_equal(rows.numpy(), want)


def test_file_dataset_refuses_what_tensor_dataset_refuses(dataset, tmp_path):
    from utils.device_data import FileDataset
    for line, what in [("base/missing.jpg", "is not exist"), ("", "is not exist")]:
        (tmp_path / "bad.txt").write_text(line + "\n")
        with pytest.raises(Exception, match=what):
            FileDataset("bad.txt")
    for ext in ("JPG", "gif", "Png"):
        (tmp_path / ("upper." + ext)).write_bytes(b"x")
        (tmp_path / "bad.txt").write_text("upper.%s\n" % ext)
        with pytest.raises(Exception, match="img type error:%s" % ext):
            FileDataset("bad.txt")
    with pytest.raises(AssertionError):
        FileDataset("no_such_list.txt")
    (tmp_path / "nolabel.jpg").write_bytes(b"x")
    (tmp_path / "one.txt").write_text("nolabel.jpg\n")
    ds = FileDataset("one.txt")
    with pytest.raises(Exception, match="nolabel.txt is not exist"):
        ds[0]


_WORKER = r"""
import hashlib, sys, torch
sys.path[:0] = [%(root)r, %(tests)r]
import yfv2
import loader_cases as lc
from utils.device_data import FileDataset, collate_files
z, names = lc.load(%(golden)r)
ds = FileDataset(lc.LIST)
read = lc.fallback_reader(z)
calls = []
def fallback(data):
    calls.append(lc.sha(bytes(data)))
    return read(data)
B = %(B)d
for k in range(0, len(ds), B):
    out = collate_files([ds[i] for i in range(k, min(k + B, len(ds)))], fallback=fallback)
    assert sorted(out["jpeg_slots"] + out["frame_slots"]) == list(range(out["n"]))
    for slot, fr in zip(out["frame_slots"], out["frames"]):
        want = z["frame_" + lc.sha(ds[k + slot][0])]
        assert fr.numpy().tobytes() == want.tobytes() and tuple(fr.shape) == want.shape
    print("BATCH", k, out["n"], bytes(lc.digest(out["targets"].numpy())).hex(), ",".join(names[k + s] for s in out["frame_slots"]))
    if out["jpeg"] is not None:
        infos = out["jpeg"][0]
        assert len(infos) == len(out["jpeg_slots"]) and all(i["status"] == 0 for i in infos)
print("CUDA", torch.cuda.is_initialized())
"""


@pytest.mark.parametrize("B", lc.BATCHES)
def test_collate_files_in_a_process_without_cuda(dataset, golden_dir, B):
    z, names, files = dataset
    code = _WORKER % {"root": ROOT, "tests": os.path.join(ROOT, "tests"), "golden": golden_dir, "B": B}
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=os.getcwd())
    assert r.returncode == 0, r.stderr[-3000:]
    lines = r.stdout.splitlines()
    assert lines[-1] == "CUDA False"
    batches = [ln.split(" ") for ln in lines if ln.startswith("BATCH")]
    want = z["targets_b%d" % B]
    assert len(batches) == len(want) == -(-len(names) // B)
    refused = []
    for (_, k, n, tsha, fb), w in zip(batches, want):
        assert tsha == bytes(w).hex(), k
        refused += [s for s in fb.split(",") if s]
    # every file outside the decoder's subset goes to the fallback with its slot: the PNG, the BMP, the unsupported JPEGs
    assert set(refused) == {n for n in names if n.split("/")[0] in ("unsup", "set.v1")} - {"unsup/progressive.jpg"}


def test_parse_jpeg_strict_false_returns_every_status(dataset):
    import yfv2_engine
    z, names, files = dataset
    pick = ["base/q75_420_opt0.jpg", "set.v1/seeded.png", "prog/cv2_q50_420.jpeg", "unsup/sof9.jpg"]
    data = [files[n] for n in pick]
    with pytest.raises(yfv2_engine.Yfv2Error, match="2 of 4 files refused"):
        yfv2_engine.parse_jpeg(data, pick, progressive=True)
    infos, blob, sizes, _, offsets = yfv2_engine.parse_jpeg(data, pick, blob=True, progressive=True, strict=False)
    assert [i["status"] != 0 for i in infos] == [False, True, False, True]
    assert "PNG" in infos[1]["reason"] and "arithmetic" in infos[3]["reason"]
    assert blob is None and sizes == (0, 0) and offsets[-1] == sum(len(d) for d in data)
    infos, blob, sizes, _, _ = yfv2_engine.parse_jpeg([data[0], data[2]], blob=True, progressive=True, strict=False)
    assert blob is not None and sizes[0] > 0 and all(i["status"] == 0 for i in infos)


def test_decode_resize_refuses_bad_arguments_before_any_launch(dataset):
    import yfv2_engine
    z, names, files = dataset
    L = yfv2_engine.lib()
    infos, blob, (ws, _), host, offsets = yfv2_engine.parse_jpeg([files["base/q75_420_opt0.jpg"]], blob=True)
    meta, fb = blob.numel(), int(offsets[-1])
    mh = ctypes.c_void_p(blob.data_ptr())
    fake = ctypes.c_void_p(16)                                  # never dereferenced: every check comes first

    def call(mh=mh, md=fake, m=meta, files=fake, fbytes=fb, H=192, W=320, dst=fake, err=fake, work=fake, wsb=ws):
        return L.yfv2_jpeg_decode_resize(mh, md, m, files, fbytes, H, W, dst, err, work, wsb, None)

    for kw, what in [({"mh": None}, b"null"), ({"md": None}, b"null"), ({"files": None}, b"null"), ({"dst": None}, b"null"),
                     ({"err": None}, b"null"), ({"work": None}, b"null"), ({"H": 0}, b"target"), ({"W": 0}, b"target"),
                     ({"H": -3}, b"target"), ({"W": 32769}, b"target"), ({"m": meta - 1}, b"blob"),
                     ({"fbytes": fb - 1}, b"files_bytes"), ({"wsb": ws - 1}, b"workspace_bytes")]:
        assert L.yfv2_jpeg_decode_resize is not None
        assert call(**kw) == -1, kw
        assert what in L.yfv2_last_error(), (kw, L.yfv2_last_error())
    junk = (ctypes.c_uint8 * meta)()
    assert call(mh=ctypes.cast(junk, ctypes.c_void_p)) == -1 and b"not a blob" in L.yfv2_last_error()


def test_train_dist_device_decode_needs_device_aug():
    import train_dist
    with pytest.raises(SystemExit) as e:
        train_dist.main(["--device-decode", "--data", "x.data"])
    assert e.value.code == 2
