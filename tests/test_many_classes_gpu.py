"""GPU: detectors with more than 93 classes (A + C > 96), where the heads' output convolution runs as two 96-column tiles.
Head tensors against the CPU oracle, batch invariance, the post-processing entry points fed by a real forward, and the reference's
train.py -> evaluation() -> test.py sequence with a 150-class cfg."""
import math

import numpy as np
import pytest
import torch

import yfv2  # noqa: F401
import synth
from oracle import net as onet

pytestmark = pytest.mark.gpu
TOL = dict(rtol=1e-4, atol=1e-4)


def make_model(sd, classes, anchors, export_onnx=False):
    import model.detector as det
    m = det.Detector(classes, anchors, True, export_onnx)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval()


def cfg_for(classes, anchors, h, w):
    c = synth.coco_cfg(w, h, classes)
    c["anchor_num"] = anchors
    c["anchors"] = [float(8 + 7 * i) for i in range(4 * anchors)]
    return c


@pytest.mark.parametrize("u8", [False, True], ids=["f32", "u8"])
@pytest.mark.parametrize("A,C,n,h,w,seed", [(3, 94, 2, 64, 96, 1), (3, 150, 3, 352, 352, 2), (3, 189, 1, 640, 640, 3),
                                            (4, 188, 3, 96, 160, 4)])
def test_heads_against_oracle(A, C, n, h, w, seed, u8):
    sd = synth.make_state_dict(300 + seed, classes=C, anchor_num=A)
    x = synth.make_images(400 + seed, n, h, w)
    if u8:
        x8 = (x * 255).to(torch.uint8)
        x, xin = x8.float() / 255.0, x8
    else:
        xin = x
    with torch.no_grad():
        ref = onet.forward(sd, x)
    preds = make_model(sd, C, A)(xin.cuda())
    assert [p.shape[1] for p in preds] == [4 * A, A, C] * 2
    for i, (p, r) in enumerate(zip(preds, ref)):
        np.testing.assert_allclose(p.cpu().numpy(), r.numpy(), err_msg="pred%d" % i, **TOL)


def test_batch_invariance_150_classes():
    """Every image of a batch equals the same image run alone, bit for bit."""
    m = make_model(synth.make_state_dict(51, classes=150), 150, 3)
    x = synth.make_images(52, 5, 352, 352).cuda()
    big = m(x)
    for i in range(5):
        one = m(x[i:i + 1])
        for p, q in zip(big, one):
            assert torch.equal(p[i], q[0]), i


def _forward_150(n=3, side=352, seed=61):
    sd = synth.make_state_dict(seed, classes=150)
    x = synth.make_images(seed + 1, n, side, side)
    preds = make_model(sd, 150, 3)(x.cuda())
    return sd, x, [p.contiguous() for p in preds]


def test_decode_nms_at_150_classes_from_a_forward():
    """Fused decode + NMS is bit-identical to decode -> NMS, and the NMS rows are bit-exact against the oracle on the same decoded
    tensor (the warp-per-cell candidate path: C > 80)."""
    import yfv2_engine as eng
    from oracle import post as opost
    _, _, preds = _forward_150()
    cfg = cfg_for(150, 3, 352, 352)
    cfg["anchors"] = list(synth.COCO_ANCHORS)
    d = eng.decode(preds, cfg)
    assert d.shape == (3, 3 * (22 * 22 + 11 * 11), 155)
    for ct, it in [(0.3, 0.4), (0.01, 0.4), (0.001, 0.45)]:
        out, counts, idx = eng.nms(d, ct, it)
        f_out, f_counts, f_idx = eng.decode_nms(preds, cfg, ct, it, want_idx=True)
        assert torch.equal(counts, f_counts) and torch.equal(out, f_out) and torch.equal(idx, f_idx), (ct, it)
        rows, oidx = opost.nms(d.cpu(), ct, it, return_indices=True)
        for i in range(3):
            c = int(counts[i])
            assert c == rows[i].shape[0], (ct, it, i)
            assert np.array_equal(out[i, :c].cpu().numpy(), rows[i].numpy()), (ct, it, i)
            assert np.array_equal(idx[i, :c].cpu().numpy(), oidx[i]), (ct, it, i)
        assert ct > 0.01 or int(counts.min()) > 0


def test_export_heads_and_ncnn_post_at_150_classes():
    """export_onnx head at 5A + C = 165 channels against the oracle, and the deploy post-process on it bit for bit against
    oracle/ncnn_post.c."""
    import yfv2_engine as eng
    from oracle import ncnn_post as onp
    sd, x, preds = _forward_150(n=2, side=224, seed=71)
    e2, e3 = make_model(sd, 150, 3, export_onnx=True)(x.cuda())
    assert e2.shape == (2, 14, 14, 165) and e3.shape == (2, 7, 7, 165)
    with torch.no_grad():
        r2, r3 = onet.forward_export(sd, x)
    np.testing.assert_allclose(e2.cpu().numpy(), r2.numpy(), **TOL)                       # end to end
    np.testing.assert_allclose(e3.cpu().numpy(), r3.numpy(), **TOL)
    # the export head alone, on the same head tensors: oracle/net.py forward_export's sigmoid | sigmoid | softmax, channel-last
    g2, g3 = eng.export_heads(preds)
    for got, lv in ((g2, 0), (g3, 3)):
        o = [p.cpu() for p in preds[lv:lv + 3]]
        want = torch.cat((o[0].sigmoid(), o[1].sigmoid(), torch.softmax(o[2], dim=1)), 1).permute(0, 2, 3, 1)
        np.testing.assert_allclose(got.cpu().numpy(), want.numpy(), rtol=0, atol=1e-6)
    assert torch.equal(g2, e2) and torch.equal(g3, e3)
    res = eng.ncnn_post(e2, e3, 3, 0.0002, 0.25, (448, 300))
    o2, o3 = e2.cpu().numpy(), e3.cpu().numpy()
    sw, sh = np.float32(448) / np.float32(224), np.float32(300) / np.float32(224)
    total = 0
    for i in range(2):
        b, s, k = onp.ncnn_post(o2[i], o3[i], 3, 150, 224, 224, onp.ANCHORS_COCO, np.float32(0.0002), np.float32(0.25), sw, sh)
        assert len(s) == len(res[i][1])
        assert np.array_equal(b, res[i][0]) and np.array_equal(k, res[i][2])
        assert np.array_equal(s.view(np.uint32), res[i][1].view(np.uint32))
        total += len(s)
    assert total > 20


DATA = ("[name]\nmodel_name=many\n\n[train-configure]\nepochs=1\nsteps=150,250\nbatch_size=8\nsubdivisions=2\nlearning_rate=0.001\n\n"
        "[model-configure]\npre_weights=None\nclasses=150\nwidth=352\nheight=352\nanchor_num=3\n"
        "anchors=12.64,19.39, 37.88,51.48, 55.71,138.31, 126.91,78.23, 131.57,214.55, 279.92,258.87\n\n"
        "[data-configure]\ntrain=/nonexistent/train.txt\nval=/nonexistent/val.txt\nnames=%s\n")


def test_train_evaluate_test_sequence_150_classes(tmp_path):
    """The reference's scripts with a 150-class dataset: three train.py iterations, then evaluation() (what train.py runs every 10
    epochs and evaluation.py runs on the weights), then the test.py flow on the trained model."""
    import model.detector
    import utils.loss
    import utils.utils
    import train_dist
    from torch import optim
    names = tmp_path / "many.names"
    names.write_text("\n".join("c%d" % i for i in range(150)) + "\n")
    data = tmp_path / "many.data"
    data.write_text(DATA % names)
    cfg = utils.utils.load_datafile(str(data))
    assert cfg["classes"] == 150
    device = torch.device("cuda")
    weights = tmp_path / "init.pth"
    torch.save(synth.make_state_dict(81, classes=150), weights)

    # train.py:70-131
    batch_size = int(cfg["batch_size"] / cfg["subdivisions"])
    ds = train_dist.SyntheticDetection(3 * batch_size, cfg["width"], cfg["height"], cfg["classes"])
    train_dataloader = torch.utils.data.DataLoader(ds, batch_size=batch_size, shuffle=True, collate_fn=train_dist.collate_fn,
                                                   num_workers=0, pin_memory=True, drop_last=True)
    model_ = model.detector.Detector(cfg["classes"], cfg["anchor_num"], True).to(device)
    model_.load_state_dict(torch.load(weights, map_location=device), strict=False)
    optimizer = optim.SGD(params=model_.parameters(), lr=cfg["learning_rate"], momentum=0.949, weight_decay=0.0005)
    batch_num, totals = 0, []
    model_.train()
    for imgs, targets in train_dataloader:
        imgs = imgs.to(device).float() / 255.0
        targets = targets.to(device)
        preds = model_(imgs)
        assert preds[2].shape[1] == 150
        iou_loss, obj_loss, cls_loss, total_loss = utils.loss.compute_loss(preds, targets, cfg, device)
        total_loss.backward()
        for g in optimizer.param_groups:
            warmup_num = 5 * len(train_dataloader)
            if batch_num <= warmup_num:
                g["lr"] = cfg["learning_rate"] * math.pow(batch_num / warmup_num, 4)
        if batch_num % cfg["subdivisions"] == 0:
            optimizer.step()
            optimizer.zero_grad()
        totals += [float(iou_loss.detach()), float(obj_loss.detach()), float(cls_loss.detach()), float(total_loss.detach())]
        batch_num += 1
    assert batch_num == 3 and all(np.isfinite(totals))

    # evaluation() (train.py:134-140, evaluation.py:59-64)
    model_.eval()
    val_dataset = train_dist.SyntheticDetection(6, cfg["width"], cfg["height"], cfg["classes"], seed=5)
    val_dataloader = torch.utils.data.DataLoader(val_dataset, batch_size=4, shuffle=False, collate_fn=train_dist.collate_fn,
                                                 num_workers=0, pin_memory=True, drop_last=False)
    r = utils.utils.evaluation(val_dataloader, cfg, model_, device)
    assert r is None or (len(r) == 4 and all(np.all(np.isfinite(np.asarray(v, np.float64))) for v in r))

    # test.py:21-49 on the trained weights
    trained = tmp_path / "trained.pth"
    torch.save(model_.state_dict(), trained)
    model_t = model.detector.Detector(cfg["classes"], cfg["anchor_num"], True).to(device)
    model_t.load_state_dict(torch.load(trained, map_location=device))
    model_t.eval()
    img = synth.make_images(91, 1, cfg["height"], cfg["width"]).to(device)
    preds = model_t(img)
    output = utils.utils.handel_preds(preds, cfg, device)
    assert output.shape[-1] == 155
    output_boxes = utils.utils.non_max_suppression(output, conf_thres=0.01, iou_thres=0.4)
    LABEL_NAMES = [line.strip() for line in open(cfg["names"])]
    for box in output_boxes[0].tolist():
        assert 0 <= int(box[5]) < 150 and LABEL_NAMES[int(box[5])].startswith("c") and np.isfinite(box[:5]).all()
