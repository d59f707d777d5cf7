"""Writes tests/golden/loader_cases.npz and META_loader.json: what the reference's own TensorDataset(imgaug=False) + collate_fn give
for the dataset tests/loader_cases.py builds (run where the reference checkout and cv2 are; see loader_cases.py for the layout).

    python tests/golden/make_golden_loader.py /path/to/reference"""
import importlib.util
import json
import os
import platform
import sys
import tempfile

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import jpeg_cases                  # noqa: E402
import loader_cases as lc          # noqa: E402


def reference_datasets(ref):
    spec = importlib.util.spec_from_file_location("reference_datasets", os.path.join(ref, "utils", "datasets.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
    ds_mod = reference_datasets(ref)
    jz = np.load(os.path.join(HERE, "jpeg_cases.npz"))
    pz = np.load(os.path.join(HERE, "jpeg_progressive.npz"))

    rng = np.random.default_rng(4242)
    img = cv2.GaussianBlur(rng.integers(0, 256, (45, 70, 3), dtype=np.uint8), (5, 5), 0)
    ok_png, png = cv2.imencode(".png", img)
    ok_bmp, bmp = cv2.imencode(".bmp", img[:33, :31])
    assert ok_png and ok_bmp
    store = {"png": png.reshape(-1), "bmp": bmp.reshape(-1)}

    def decodes(b):
        return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR) is not None

    names = ["base/%s.jpg" % c[0] for c in jpeg_cases.CASES]
    unsup = [n for n, _, _ in jpeg_cases.UNSUPPORTED if decodes(jz["bad_" + n].tobytes())]
    names += ["unsup/%s.jpg" % n for n in unsup]
    names += ["cut/%s.jpg" % jpeg_cases.TRUNCATED_SCAN]
    names += ["prog/%s.jpeg" % n for n in lc.PROG]
    pdam = [n for n in lc.PROG_DAMAGED if decodes(pz["jpg_" + n].tobytes())]
    names += ["pdamaged/%s.jpg" % n for n in pdam]
    names += ["photos/%s.jpg" % p for p in lc.PHOTOS]
    names += ["set.v1/seeded.png", "set.v1/seeded.bmp"]
    store["names"] = np.array(names)

    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as root:
        files = lc.build(root, names, HERE, store)
        os.chdir(root)
        try:
            # cv2's frame of every file the device may not decode (refused, or flagged): the tests' fallback reader
            for n in names:
                if n.split("/")[0] in ("unsup", "cut", "pdamaged", "set.v1"):
                    store["frame_" + lc.sha(files[n])] = cv2.imread(n)
            for (W, H) in lc.SIZES:
                ds = ds_mod.TensorDataset(lc.LIST, W, H, imgaug=False)
                assert ds.data_list == names
                items = [ds[i] for i in range(len(ds))]
                store["sha_%dx%d" % (W, H)] = np.stack([lc.digest(im.numpy()) for im, _ in items])
                for i, (im, _) in enumerate(items):        # the reference photos at 352 x 352 are images_modelzoo.npz's
                    if (W, H) == (352, 352) and names[i].startswith("photos/"):
                        u8 = np.load(os.path.join(HERE, "images_modelzoo.npz"))[names[i][7:13] + "_u8"][0]
                        assert np.array_equal(im.numpy(), u8), names[i]
            ds = ds_mod.TensorDataset(lc.LIST, 352, 352, imgaug=False)
            for B in lc.BATCHES:
                dl = torch.utils.data.DataLoader(ds, batch_size=B, shuffle=False, collate_fn=ds_mod.collate_fn, num_workers=0)
                store["targets_b%d" % B] = np.stack([lc.digest(t.numpy()) for _, t in dl])
        finally:
            os.chdir(cwd)
    np.savez_compressed(os.path.join(HERE, "loader_cases.npz"), **store)
    meta = {"generator": "tests/golden/make_golden_loader.py", "opencv": cv2.__version__, "numpy": np.__version__,
            "torch": torch.__version__, "python": platform.python_version(), "files": len(names),
            "fallback_frames": sum(k.startswith("frame_") for k in store), "unsupported_read_by_cv2": unsup,
            "progressive_damaged_read_by_cv2": pdam, "sizes": [list(s) for s in lc.SIZES], "batches": list(lc.BATCHES)}
    with open(os.path.join(HERE, "META_loader.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(meta, indent=1))


if __name__ == "__main__":
    main()
