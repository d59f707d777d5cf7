"""Training and evaluation batches from image files, decoded and resized on the GPU (the input side of utils/datasets.py:71-129).

The reference's TensorDataset reads every image of every batch with cv2.imread and cv2.resize(img, (W, H), INTER_LINEAR) in the
loader workers.  Here the workers only read the files, parse the JPEG headers (yfv2_engine.parse_jpeg, host code, no CUDA call)
and build the targets; DeviceLoader then decodes each batch straight into the [B, 3, H, W] uint8 network input with one
yfv2_jpeg_decode_resize call, on a side stream while the previous batch trains.  Per batch the images are TensorDataset(...,
imgaug=False)'s bytes, in the same order, and the targets collate_fn's; nothing is cached between epochs.

Files the parse refuses (PNG, BMP, JPEGs outside the decoder's subset) are read in the worker by a fallback reader (cv2 by
default) and resized on the device (yfv2_engine.resize_bgr); files whose decode is flagged (corrupt or cut short) are read again
by the fallback in the main process, so they give what cv2 gives."""
import functools
import os

import numpy as np
import torch
from torch.utils.data import DataLoader
from torch.utils.data.distributed import DistributedSampler

import yfv2_engine

IMG_FORMATS = ("bmp", "jpg", "jpeg", "png")      # datasets.py:79, compared case-sensitively


def label_path(img_path):
    """The label file of an image, datasets.py:102's rule: everything before the path's first '.', plus '.txt'."""
    return img_path.split(".")[0] + ".txt"


def read_labels(path):
    """datasets.py:114-126: float32 rows (0, cls, cx, cy, w, h) of a label file (shape (0,) when it is empty); a missing file
    raises."""
    if not os.path.exists(path):
        raise Exception("%s is not exist" % path)
    label = []
    with open(path, "r") as f:
        for line in f.readlines():
            v = line.strip().split(" ")
            label.append([0, v[0], v[1], v[2], v[3], v[4]])
    label = np.array(label, dtype=np.float32)
    if label.shape[0]:
        assert label.shape[1] == 6, "> 5 label columns: %s" % path
    return torch.from_numpy(label)


class FileDataset(torch.utils.data.Dataset):
    """TensorDataset's list file and checks (datasets.py:72-97): every listed path exists and its extension, split(".")[-1], is one
    of bmp jpg jpeg png.  An item is (the file's bytes, its label rows); nothing is decoded here."""

    def __init__(self, path, img_size_width=352, img_size_height=352):
        assert os.path.exists(path), "%s: list file not found" % path
        self.path = path
        self.img_size_width, self.img_size_height = img_size_width, img_size_height
        self.data_list = []
        with open(path, "r") as f:
            for line in f.readlines():
                data_path = line.strip()
                if not os.path.exists(data_path):
                    raise Exception("%s is not exist" % data_path)
                img_type = data_path.split(".")[-1]
                if img_type not in IMG_FORMATS:
                    raise Exception("img type error:%s" % img_type)
                self.data_list.append(data_path)

    def __getitem__(self, index):
        img_path = self.data_list[index]
        with open(img_path, "rb") as f:
            data = f.read()
        return data, read_labels(label_path(img_path))

    def __len__(self):
        return len(self.data_list)


def imread_bytes(data):
    """The fallback reader: cv2.imdecode(data, IMREAD_COLOR), what cv2.imread returns for the file (cv2 imported here only)."""
    import cv2
    return cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)


def collate_targets(labels):
    """collate_fn's targets (datasets.py:70-75): each image's rows get its index in column 0, then all rows concatenated."""
    for i, l in enumerate(labels):
        if l.shape[0] > 0:
            l[:, 0] = i
    return torch.cat(labels, 0)


def collate_files(batch, fallback=None, progressive=True):
    """Runs in the loader worker and makes no CUDA call.  batch: FileDataset items.  Returns a dict of plain tensors, lists and
    numbers (so pin_memory pins the tensors):
      n          the batch size;
      jpeg       parse_jpeg(...)'s (infos, blob, sizes, packed files, offsets) of the files the parse accepts, or None;
      jpeg_slots their places in the batch;
      frames     HWC uint8 BGR tensors the fallback reader gave for the refused files, frame_slots their places;
      targets    collate_fn's targets."""
    data, labels = zip(*batch)
    fallback = fallback or imread_bytes
    out = {"n": len(data), "jpeg": None, "jpeg_slots": [], "frames": [], "frame_slots": [],
           "targets": collate_targets(list(labels))}
    parsed = yfv2_engine.parse_jpeg(data, blob=True, progressive=progressive, strict=False)
    accepted = [i for i, inf in enumerate(parsed[0]) if inf["status"] == 0]
    if len(accepted) < len(data):
        parsed = yfv2_engine.parse_jpeg([data[i] for i in accepted], blob=True, progressive=progressive) if accepted else None
    out["jpeg"], out["jpeg_slots"] = parsed, accepted
    for i in range(len(data)):
        if i not in accepted:
            out["frames"].append(torch.from_numpy(_fallback_frame(fallback, data[i], i)))
            out["frame_slots"].append(i)
    return out


def _fallback_frame(fallback, data, slot):
    img = fallback(data)
    if img is None:                      # cv2.resize would raise on it in the reference's __getitem__
        raise yfv2_engine.Yfv2Error("device_data: the fallback reader could not read the file in batch slot %d" % slot)
    return np.ascontiguousarray(img)


class DeviceLoader:
    """Wraps a DataLoader whose collate_fn is collate_files and yields (imgs, targets): imgs a CUDA uint8 [B, 3, H, W] batch, byte
    for byte torch.stack of TensorDataset(..., imgaug=False) items, targets collate_fn's (CPU, pinned).

    Batch k + 1 is decoded on a side stream while batch k is in use: imgs is ready on the stream that is current when the batch is
    yielded (the stream waits on an event; imgs.record_stream marks its use there), so a consumer that trains on the current
    stream, CUDA graphs included, needs no synchronisation of its own.  Each batch's decode flags are read before it is yielded; a
    flagged file is read again by the fallback reader and resized into its slot."""

    def __init__(self, dataloader, width, height, device=None, fallback=None):
        self.dataloader, self.width, self.height = dataloader, int(width), int(height)
        self.device = torch.device(device if device is not None else torch.device("cuda", torch.cuda.current_device()))
        if self.device.type != "cuda":
            raise yfv2_engine.Yfv2Error("DeviceLoader: runs on CUDA devices only (no CPU fallback)")
        self.fallback = fallback or imread_bytes
        with torch.cuda.device(self.device):
            self.stream = torch.cuda.Stream(self.device)

    def __len__(self):
        return len(self.dataloader)

    @property
    def sampler(self):
        return self.dataloader.sampler

    def __iter__(self):
        pending = None
        for raw in self.dataloader:
            job = self._launch(raw)
            if pending is not None:
                yield self._finish(pending)
            pending = job
        if pending is not None:
            yield self._finish(pending)

    def _launch(self, raw):
        """Enqueues the batch's decode and resizes on the side stream; returns what _finish needs."""
        dev, W, H = self.device, self.width, self.height
        job = {"raw": raw, "batch": None, "flags": None}
        with torch.cuda.device(dev), torch.cuda.stream(self.stream):
            imgs = torch.empty((raw["n"], 3, H, W), dtype=torch.uint8, device=dev)
            if raw["frame_slots"]:              # first: their host-to-device copies wait for the side stream
                self._resize_into(imgs, raw["frames"], raw["frame_slots"])
            slots = raw["jpeg_slots"]
            if slots:
                b = yfv2_engine.JpegBatch(None, dev, parsed=raw["jpeg"])
                if len(slots) == raw["n"]:
                    b.decode_resize(imgs, W, H)
                else:
                    part = b.decode_resize(torch.empty((len(slots), 3, H, W), dtype=torch.uint8, device=dev), W, H)
                    imgs.index_copy_(0, torch.tensor(slots, device=dev), part)
                job["flags"] = torch.empty(len(slots), dtype=torch.int32, pin_memory=True)
                job["flags"].copy_(b.errors, non_blocking=True)
                job["batch"] = b
            job["done"] = torch.cuda.Event()
            job["done"].record(self.stream)
        job["imgs"] = imgs
        return job

    def _resize_into(self, imgs, frames, slots):
        part = yfv2_engine.resize_bgr(frames, self.width, self.height, self.device)
        imgs.index_copy_(0, torch.tensor(slots, device=self.device), part)

    def _finish(self, job):
        """Waits for the batch's decode, repairs flagged slots, and hands imgs to the current stream."""
        raw, imgs = job["raw"], job["imgs"]
        job["done"].synchronize()
        if job["flags"] is not None:
            bad = [j for j, e in enumerate(job["flags"].tolist()) if e]
            if bad:
                _, _, _, host, offsets = raw["jpeg"]
                frames = [torch.from_numpy(_fallback_frame(self.fallback, host[offsets[j]:offsets[j + 1]].numpy().tobytes(),
                                                           raw["jpeg_slots"][j])) for j in bad]
                with torch.cuda.device(self.device), torch.cuda.stream(self.stream):
                    self._resize_into(imgs, frames, [raw["jpeg_slots"][j] for j in bad])
                    job["done"].record(self.stream)
        cur = torch.cuda.current_stream(self.device)
        cur.wait_event(job["done"])
        imgs.record_stream(cur)
        return imgs, raw["targets"]


def device_loader(path, width, height, batch_size, device, *, num_workers, train=False, world=1, rank=0, fallback=None,
                  progressive=True):
    """The loader train_dist.py and evaluation.py build from a list file: FileDataset -> DataLoader (collate_files, pin_memory,
    persistent workers) -> DeviceLoader.  train: a DistributedSampler over `world` ranks with shuffle and drop_last, as
    train_dist.py's host loader (set_epoch through .sampler); otherwise the files in order with the last short batch kept, as
    the reference's validation loader (train.py:50-58, evaluation.py:34-43)."""
    ds = FileDataset(path, width, height)
    collate = functools.partial(collate_files, fallback=fallback, progressive=progressive)
    kw = dict(batch_size=batch_size, collate_fn=collate, num_workers=num_workers, pin_memory=True,
              persistent_workers=num_workers > 0)
    if train:
        sampler = DistributedSampler(ds, num_replicas=world, rank=rank, shuffle=True, drop_last=True)
        dl = DataLoader(ds, sampler=sampler, drop_last=True, **kw)
    else:
        dl = DataLoader(ds, shuffle=False, drop_last=False, **kw)
    return DeviceLoader(dl, width, height, device, fallback)
