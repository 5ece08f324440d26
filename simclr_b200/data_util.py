"""Device-side data augmentation of the reference (`tf2/data_util.py`).

`prepare_views` is the fused input stage of `Model.__call__`
(tf2/model.py:250-259): channel split into views, `batch_random_blur`
(tf2/data_util.py:413-440), batch concat (view-major), cast to the activation
dtype and pad 3 -> 4 channels, in two passes over the images.
"""
import torch

from ._lib import lib, stream_ptr
from .engine import get_engine


def draw_blur(num_views, batch, device, blur_probability=0.5, generator=None):
    """The `tf.random` draws of `batch_random_blur`: one sigma ~ U[0.1, 2.0] per view
    shared by the batch (tf2/data_util.py:407, SURVEY Q10) and a Bernoulli(p)
    selector per sample (tf2/data_util.py:425-430)."""
    sigma = torch.empty(num_views, dtype=torch.float32, device=device).uniform_(0.1, 2.0, generator=generator)
    selector = (torch.rand(num_views, batch, device=device, generator=generator) < blur_probability).to(torch.uint8)
    return sigma, selector


def prepare_views(inputs, num_transforms, use_blur, image_size, draws=None):
    """inputs [B,H,W,3*T] fp32 in [0,1] -> [T*B,H,W,4] activation dtype."""
    e = get_engine()
    assert inputs.dtype == torch.float32
    inputs = inputs.contiguous()
    B, H, W, C = inputs.shape
    T = num_transforms
    assert C == 3 * T
    out = e.empty((T * B, H, W, 4))
    sigma = selector = tmp = None
    if use_blur:
        if draws is None:
            sigma, selector = draw_blur(T, B, e.device)
        else:
            sigma, selector = draws
            sigma = torch.as_tensor(sigma, dtype=torch.float32, device=e.device).contiguous()
            selector = torch.as_tensor(selector, device=e.device).to(torch.uint8).contiguous()
        tmp = e.empty((T * B, H, W, 3), torch.float32)
    lib.input_prep(inputs, out, e.code(out.dtype), B, H, W, T, int(use_blur), image_size // 10,
                   sigma, selector, tmp, stream_ptr())
    return out


def batch_random_blur(images_list, height, width, blur_probability=0.5, draws=None):
    """tf2/data_util.py:413-440 on a list of [B,H,W,3] fp32 views; returns fp32 views."""
    e = get_engine()
    T = len(images_list)
    B, H, W, _ = images_list[0].shape
    x = torch.cat(images_list, dim=-1).contiguous()
    if draws is None:
        draws = draw_blur(T, B, e.device, blur_probability)
    sigma = torch.as_tensor(draws[0], dtype=torch.float32, device=e.device).contiguous()
    selector = torch.as_tensor(draws[1], device=e.device).to(torch.uint8).contiguous()
    out = e.empty((T * B, H, W, 4), torch.float32)
    tmp = e.empty((T * B, H, W, 3), torch.float32)
    lib.input_prep(x, out, 0, B, H, W, T, 1, height // 10, sigma, selector, tmp, stream_ptr())
    return [out[t * B:(t + 1) * B, :, :, :3] for t in range(T)]


def preprocess_for_train_batch(images, draws, height, width, out=None, channel_offset=0):
    """`preprocess_for_train` (tf2/data_util.py:443-475) for a batch of uint8 images on device.

    images: list of uint8 tensors [Hs,Ws,3] (any device); draws: list of dicts with keys
    box=(y,x,h,w), flip, color=dict(apply_jitter, perm, brightness, contrast, saturation, hue,
    apply_gray) -- the reference's tf.random draws.  Returns fp32 [n,height,width,3], or writes
    into `out` [n,height,width,C] at `channel_offset` (two views -> [B,H,W,6], tf2/data.py:55-58)."""
    import numpy as np
    e = get_engine()
    offs, hw, total = [], [], 0
    for im in images:
        assert im.dtype == torch.uint8 and im.dim() == 3 and im.shape[2] == 3
        offs.append(total); hw.append([im.shape[0], im.shape[1]]); total += im.numel()
    src = torch.cat([im.reshape(-1) for im in images]).to(e.device)
    return _augment_packed(src, np.asarray(offs, dtype=np.int64), np.asarray(hw, dtype=np.int32), hw, draws, height,
                           width, out, channel_offset)


def _augment_packed(src, src_offset, src_hw, hw, draws, height, width, out, channel_offset):
    """One `simclr_augment` launch over packed images; `hw`: the [n][2] image sizes on the host (box checks)."""
    import numpy as np
    e = get_engine()
    n = len(draws)
    box = np.asarray([d['box'] for d in draws], dtype=np.int32)
    for (y, x, h, w), (Hs, Ws) in zip(box, hw):
        if not (0 <= y and 0 <= x and h > 0 and w > 0 and y + h <= Hs and x + w <= Ws):
            raise ValueError('crop box out of the image')
    flip = np.asarray([1 if d['flip'] else 0 for d in draws], dtype=np.uint8)
    col = np.zeros((n, 8), dtype=np.float32)
    for i, d in enumerate(draws):
        c = d['color']
        code = sum(int(op) << (2 * t) for t, op in enumerate(c['perm']))
        col[i] = [1.0 if c['apply_jitter'] else 0.0, code, c['brightness'], c['contrast'], c['saturation'], c['hue'],
                  1.0 if c['apply_gray'] else 0.0, 0.0]
    t = lambda a: torch.as_tensor(a).to(e.device)
    if out is None:
        out = e.empty((n, height, width, 3), torch.float32)
    assert out.dtype == torch.float32 and out.is_contiguous() and out.shape[:3] == (n, height, width)
    lib.augment(src, t(src_offset).to(torch.int64), t(src_hw).to(torch.int32), t(box), t(flip), t(col),
                out, n, height, width, out.shape[3], channel_offset, stream_ptr())
    return out


def preprocess_for_train_packed(src, src_offset, src_hw, draws, height, width, out=None, channel_offset=0):
    """`preprocess_for_train_batch` over images already packed on the device, as `jpeg.decode_batch` returns them:
    src uint8 HWC images back to back, src_offset int64 [n], src_hw int32 [n][2] (host or device tensors / arrays).
    The same kernel launch and results as the list form."""
    import numpy as np
    hw = src_hw.cpu().numpy() if isinstance(src_hw, torch.Tensor) else np.asarray(src_hw)
    assert src.dtype == torch.uint8 and len(hw) == len(draws) == len(src_offset)
    return _augment_packed(src, src_offset, src_hw, hw.tolist(), draws, height, width, out, channel_offset)


def preprocess_for_eval_packed(src, src_offset, src_hw, height, width, crop=True, out=None, channel_offset=0):
    """`preprocess_for_eval_batch` over packed images (see `preprocess_for_train_packed`)."""
    import numpy as np
    hw = src_hw.cpu().numpy() if isinstance(src_hw, torch.Tensor) else np.asarray(src_hw)
    draws = [dict(box=_eval_box(int(Hs), int(Ws), height, width, crop), flip=False, color=_NO_COLOR) for Hs, Ws in hw]
    return preprocess_for_train_packed(src, src_offset, src_hw, draws, height, width, out=out, channel_offset=channel_offset)


# ---------------------------------------------------------------------------
# The reference's per-image entry point (tf2/data_util.py:497-518) and its random draws
# ---------------------------------------------------------------------------

def draw_train_augmentation(src_h, src_w, color_jitter_strength=1.0, rng=None):
    """Host-side draws of `preprocess_for_train` (tf2/data_util.py:443-475) with the reference's
    distributions: crop via the `sample_distorted_bounding_box` rule (aspect ~ U[3/4, 4/3], area in
    [0.08, 1] of the image, accepted iff it covers >= 10 % (min_object_covered with the whole-image
    box), <= 100 attempts, else the whole image -- SURVEY.md A9), flip ~ B(0.5), colour jitter
    with p 0.8 (brightness / contrast / saturation factors and hue delta from `color_jitter`,
    tf2/data_util.py:53-75, random op order), grayscale with p 0.2."""
    import math
    import random
    rng = rng or random
    box = (0, 0, src_h, src_w)
    area = float(src_h * src_w)
    for _ in range(100):
        aspect = rng.uniform(3. / 4, 4. / 3)
        min_h = int(round(math.sqrt(0.08 * area / aspect)))
        max_h = int(round(math.sqrt(1.0 * area / aspect)))
        if max_h * aspect > src_w:
            max_h = int((src_w + 0.5 - 1e-7) / aspect)
        max_h = min(max_h, src_h)
        h = min(min_h, max_h)
        if h < max_h:
            h += rng.randint(0, max_h - h)
        w = int(round(h * aspect))
        if h <= 0 or w <= 0 or h > src_h or w > src_w:
            continue
        if w * h < 0.1 * area:          # min_object_covered = 0.1 of the whole-image bounding box
            continue
        y = rng.randint(0, src_h - h)
        x = rng.randint(0, src_w - w)
        box = (y, x, h, w)
        break
    s = color_jitter_strength
    perm = [0, 1, 2, 3]
    rng.shuffle(perm)
    color = dict(apply_jitter=(s > 0 and rng.random() < 0.8), perm=tuple(perm),
                 brightness=rng.uniform(max(1.0 - 0.8 * s, 0), 1.0 + 0.8 * s),
                 contrast=rng.uniform(1 - 0.8 * s, 1 + 0.8 * s), saturation=rng.uniform(1 - 0.8 * s, 1 + 0.8 * s),
                 hue=rng.uniform(-0.2 * s, 0.2 * s), apply_gray=(s > 0 and rng.random() < 0.2))
    return dict(box=box, flip=rng.random() < 0.5, color=color)


CROP_PROPORTION = 0.875  # Standard for ImageNet (tf2/data_util.py:22)

_NO_COLOR = dict(apply_jitter=False, perm=(0, 1, 2, 3), brightness=1., contrast=1., saturation=1., hue=0., apply_gray=False)


def _compute_crop_shape(image_height, image_width, aspect_ratio, crop_proportion):
    """tf2/data_util.py:175-213: aspect-ratio-preserving shape of the central crop (fp32 arithmetic, round half
    to even, as `tf.math.rint`)."""
    import numpy as np
    w, h = np.float32(image_width), np.float32(image_height)
    if aspect_ratio > float(w / h):
        crop_height = int(np.rint(np.float32(crop_proportion / aspect_ratio) * w))
        crop_width = int(np.rint(np.float32(crop_proportion) * w))
    else:
        crop_height = int(np.rint(np.float32(crop_proportion) * h))
        crop_width = int(np.rint(np.float32(crop_proportion * aspect_ratio) * h))
    return crop_height, crop_width


def center_crop_box(image_height, image_width, height, width, crop_proportion=CROP_PROPORTION):
    """(y, x, h, w) of `center_crop` (tf2/data_util.py:216-243)."""
    crop_height, crop_width = _compute_crop_shape(image_height, image_width, width / height, crop_proportion)
    return (((image_height - crop_height) + 1) // 2, ((image_width - crop_width) + 1) // 2, crop_height, crop_width)


def preprocess_for_eval_batch(images, height, width, crop=True, out=None, channel_offset=0):
    """`preprocess_for_eval` (tf2/data_util.py:478-494) for a batch of uint8 images: central crop of
    CROP_PROPORTION, bicubic resize, clip -- the crop / resize / clip stages of the augmentation kernel with the
    flip and the colour ops switched off.  Without `crop` the images must already be height x width."""
    draws = [dict(box=_eval_box(im.shape[0], im.shape[1], height, width, crop), flip=False, color=_NO_COLOR)
             for im in images]
    return preprocess_for_train_batch(images, draws, height, width, out=out, channel_offset=channel_offset)


def _eval_box(Hs, Ws, height, width, crop):
    if crop:
        return center_crop_box(Hs, Ws, height, width)
    if (Hs, Ws) != (height, width):
        raise ValueError('preprocess_for_eval(crop=False) needs %dx%d images, got %dx%d' % (height, width, Hs, Ws))
    return (0, 0, Hs, Ws)


def preprocess_image(image, height, width, is_training=False, color_jitter_strength=0., test_crop=True, draws=None):
    """Preprocesses the given image (tf2/data_util.py:497-518; same arguments).

    image: uint8 tensor [Hs,Ws,3].  Training: `preprocess_for_train` on device (`draws` injects the random
    draws); otherwise `preprocess_for_eval` (central crop when `test_crop`)."""
    if not is_training:
        return preprocess_for_eval_batch([image], height, width, crop=test_crop)[0]
    if draws is None:
        draws = draw_train_augmentation(image.shape[0], image.shape[1], color_jitter_strength)
    if color_jitter_strength <= 0:
        draws = dict(draws, color=dict(draws['color'], apply_jitter=False, apply_gray=False))
    return preprocess_for_train_batch([image], [draws], height, width)[0]
