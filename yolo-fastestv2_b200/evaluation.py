#!/usr/bin/env python
"""The reference's evaluation.py (--data, --weights): the same two evaluation() passes over cfg["val"] and the same printed line,
with the validation images decoded and resized on the GPU (utils.device_data) instead of by cv2 in the loader workers.

    python yolo-fastestv2_b200/evaluation.py --data data/coco.data --weights modelzoo/coco2017-0.241078ap-model.pth"""
import argparse
import os
import sys

_PKG = os.path.dirname(os.path.abspath(__file__))
if _PKG not in sys.path:
    sys.path.insert(0, _PKG)

import torch                                    # noqa: E402


def main(argv=None, fallback=None):
    """Returns (precision, recall, AP, F1) as printed.  fallback: utils.device_data's reader for files the GPU decoder refuses."""
    parser = argparse.ArgumentParser()
    parser.add_argument("--data", type=str, default="", help="Specify training profile *.data")
    parser.add_argument("--weights", type=str, default="", help="The path of the model")
    opt = parser.parse_args(argv)

    import utils.utils
    import utils.device_data
    import model.detector
    cfg = utils.utils.load_datafile(opt.data)
    assert os.path.exists(opt.weights), "no model at --weights %r" % opt.weights
    if not torch.cuda.is_available():
        raise SystemExit("evaluation.py: runs on CUDA only (no CPU fallback)")

    print("评估配置:")
    print("model_name:%s" % cfg["model_name"])
    print("width:%d height:%d" % (cfg["width"], cfg["height"]))
    print("val:%s" % (cfg["val"]))
    print("model_path:%s" % (opt.weights))

    batch_size = int(cfg["batch_size"] / cfg["subdivisions"])
    nw = min([os.cpu_count(), batch_size if batch_size > 1 else 0, 8])
    device = torch.device("cuda", torch.cuda.current_device())
    val_dataloader = utils.device_data.device_loader(cfg["val"], cfg["width"], cfg["height"], batch_size, device, num_workers=nw,
                                                     fallback=fallback)

    model_ = model.detector.Detector(cfg["classes"], cfg["anchor_num"], True).to(device)
    model_.load_state_dict(torch.load(opt.weights, map_location=device))
    model_.eval()

    print("computer mAP...")
    _, _, AP, _ = utils.utils.evaluation(val_dataloader, cfg, model_, device)
    print("computer PR...")
    precision, recall, _, f1 = utils.utils.evaluation(val_dataloader, cfg, model_, device, 0.3)
    print("Precision:%f Recall:%f AP:%f F1:%f" % (precision, recall, AP, f1))
    return precision, recall, AP, f1


if __name__ == "__main__":
    main()
