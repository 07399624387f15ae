"""TEST INFRASTRUCTURE: numpy restatement of gh_render_maps and gh_eval_metrics, written from the reference lines they
replace, in float64 (the replay the GPU results are judged against) or float32 (operation by operation, to pin
rounding-sensitive choices such as save_image's separate multiply and add):

    the dir -> angle epilogue           src/gaussian_renderer/__init__.py:100-105
    vis_orient                          src/utils/image_utils.py:22-37
    psnr                                src/utils/image_utils.py:18-20
    l1_loss, ce_loss, or_loss           src/utils/loss_utils.py:19-47
    save_image's quantisation           torchvision.utils.save_image: x.mul(255).add_(0.5).clamp_(0, 255).to(uint8)
    render_set                          src/render_gaussians.py:50-68
    training_report                     src/train_gaussians.py:254-277, src/train_latent_strands.py:235-258
"""
import numpy as np


def orient_angle(raw, dtype=np.float64):
    c5, c6 = raw[5].astype(dtype), raw[6].astype(dtype)
    den = np.maximum(np.sqrt(c5 * c5 + c6 * c6), dtype(1e-12))
    dx, dy = c5 / den, c6 / den
    mirror = np.where(dx < 0, dtype(-1), dtype(1))
    lo, hi = (np.float32(-1) + np.float32(1e-3), np.float32(1) - np.float32(1e-3)) if dtype == np.float32 else (-0.999, 0.999)
    return (np.arccos(np.clip(dy, dtype(lo), dtype(hi)) * mirror) / dtype(np.pi)).astype(dtype)


def prequant(x, dtype=np.float64):
    """x * 255 + 0.5 before the clamp and the truncation (two rounded operations in float32)."""
    return x.astype(dtype) * dtype(255) + dtype(0.5)


def quant(x, dtype=np.float64):
    return np.clip(np.nan_to_num(prequant(x, dtype), nan=0.0), 0, 255).astype(np.uint8)


def vis_orient(ang, mask, dtype=np.float64):
    deg = ang.astype(dtype) * dtype(180)
    tri = lambda c: np.clip(dtype(1) - np.abs(deg - dtype(c)) / dtype(45), 0, 1)  # noqa: E731
    red, green, magenta, teal = tri(0) + tri(180), tri(90), tri(45), tri(135)
    bgr = [magenta + teal, green + teal, red + magenta]
    return np.stack([bgr[2], bgr[1], bgr[0]]) * mask.astype(dtype)


def render_maps(raw, dtype=np.float64, values=False):
    """The eight maps of gh_render_maps from a raw (10,H,W) array; `values`: the pre-truncation x * 255 + 0.5 of the
    byte maps instead of the bytes."""
    r = raw.astype(dtype)
    q = (lambda x: prequant(x, dtype)) if values else (lambda x: quant(x, dtype))
    hair, head = r[3], r[4]
    ang = orient_angle(raw, dtype)
    conf = r[8] * hair
    hwc = lambda x: np.ascontiguousarray(np.moveaxis(x, 0, -1))  # noqa: E731
    return {"orient_angle": ang[None], "orient_conf_masked": conf[None],
            "render_u8": hwc(q(r[0:3])), "hair_mask_u8": q(hair), "head_mask_u8": q(head), "orient_u8": q(ang * hair),
            "orient_vis_u8": hwc(q(vis_orient(ang, hair, dtype))),
            "orient_conf_vis_u8": hwc(q(vis_orient(ang, dtype(1) - dtype(1) / (conf + dtype(1)), dtype)))}


def eval_metrics(raw, gt_image, gt_mask, gt_angle, gt_conf, stage, dtype=np.float64):
    """gh_eval_metrics' row (l1, mask or ce, or, psnr, ssim = NaN, mse r g b); `stage` 0, 1 (identical) or 2."""
    c01 = lambda x: np.clip(x.astype(dtype), 0, 1)  # noqa: E731
    r = raw.astype(dtype)
    image, mask, ang = c01(r[0:3]), c01(r[3:5]), c01(orient_angle(raw, dtype))
    gi, gm, ga, gc = c01(gt_image), c01(gt_mask), c01(gt_angle[0]), gt_conf[0].astype(dtype)
    if stage == 2:
        image, gi = image * gm[:1], gi * gm[:1]
        p = np.clip(mask[0], dtype(1e-3), dtype(1) - dtype(1e-3))
        m = np.mean(-(gm[0] * np.maximum(np.log(p), -100) + (1 - gm[0]) * np.maximum(np.log(1 - p), -100)), dtype=np.float64)
    else:
        m = np.mean(np.abs(mask - gm), dtype=np.float64)
    d = ang - ga
    lo = np.minimum(np.abs(d), np.minimum(np.abs(d - 1), np.abs(d + 1))) * dtype(np.pi) * gm[0]
    with np.errstate(divide="ignore", invalid="ignore"):
        orient = np.float64(np.sum(lo * gc, dtype=np.float64)) / np.float64(np.sum(gc, dtype=np.float64))
        mse = np.mean(((image - gi) ** 2).reshape(3, -1), axis=1, dtype=np.float64)
        psnr = np.mean(20 * np.log10(1.0 / np.sqrt(mse)))
    return np.array([np.mean(np.abs(image - gi), dtype=np.float64), m, orient, psnr, np.nan, *mse])


def check_bytes(got, raw, name, tol=2e-3):
    """A byte map against the float64 replay of `raw`: equal wherever the replay's x * 255 + 0.5 is further than `tol`
    (the float32 error of the epilogue, in byte levels) from a truncation boundary, at most one level off elsewhere."""
    v = np.clip(render_maps(raw, np.float64, values=True)[name], 0, 255.999)
    want = v.astype(np.uint8)
    got = np.asarray(got)
    assert got.shape == want.shape, f"{name}: shape {got.shape} vs {want.shape}"
    diff = np.abs(got.astype(np.int32) - want.astype(np.int32))
    near = np.abs(v - np.round(v)) <= tol
    assert not np.any(diff[~near]), f"{name}: {int(np.count_nonzero(diff[~near]))} bytes differ away from a boundary"
    assert diff.max(initial=0) <= 1, f"{name}: a byte is {int(diff.max())} levels off"
    return int(np.count_nonzero(diff))
