"""Oracle restatement of the train-time parts of `tf2/data_util.py`.

Test infrastructure only.  Every `tf.random.*` draw of the reference is an
explicit argument here (`draws`), so the deterministic arithmetic can be
compared with the CUDA kernels on identical draws.  TF op semantics follow
SURVEY.md Appendix A9.
"""
import torch
import torch.nn.functional as F


# ---------------------------------------------------------------------------
# Gaussian blur (on-device in the reference too: tf2/model.py:255-258)
# ---------------------------------------------------------------------------

def blur_filter(kernel_size, sigma, dtype=torch.float32):
    """tf2/data_util.py:338-343."""
    radius = int(kernel_size / 2)
    x = torch.arange(-radius, radius + 1, dtype=dtype)
    f = torch.exp(-torch.pow(x, 2.0) / (2.0 * torch.pow(torch.tensor(sigma, dtype=dtype), 2.0)))
    return f / f.sum()


def gaussian_blur(image, kernel_size, sigma):
    """tf2/data_util.py:323-361 on [N,H,W,C]; depthwise, zero 'SAME' padding,
    horizontal pass then vertical pass."""
    f = blur_filter(kernel_size, sigma, image.dtype)
    k = f.numel()
    r = k // 2
    c = image.shape[-1]
    x = image.permute(0, 3, 1, 2)
    wh = f.view(1, 1, 1, k).repeat(c, 1, 1, 1)
    wv = f.view(1, 1, k, 1).repeat(c, 1, 1, 1)
    x = F.conv2d(x, wh, padding=(0, r), groups=c)
    x = F.conv2d(x, wv, padding=(r, 0), groups=c)
    return x.permute(0, 2, 3, 1)


def batch_random_blur(images_list, height, width, blur_probability=0.5, draws=None):
    """tf2/data_util.py:413-440.  draws[i] = (sigma, selector[bsz] in {0,1}) for
    view i: one sigma per call shared by the whole batch (SURVEY Q10)."""
    del width
    new_images_list = []
    for i, images in enumerate(images_list):
        if draws is None:
            sigma = float(torch.empty(()).uniform_(0.1, 2.0))
            selector = (torch.rand(images.shape[0]) < blur_probability)
        else:
            sigma, selector = draws[i]
        selector = torch.as_tensor(selector).to(images.dtype).view(-1, 1, 1, 1)
        images_new = gaussian_blur(images, height // 10, sigma)
        images = images_new * selector + images * (1 - selector)
        images = torch.clamp(images, 0., 1.)
        new_images_list.append(images)
    return new_images_list


# ---------------------------------------------------------------------------
# Colour ops (tf.image semantics, SURVEY A9) on [H,W,3] or [N,H,W,3] in [0,1]
# ---------------------------------------------------------------------------

def random_brightness(image, factor):
    """tf2/data_util.py:33-43, impl='simclrv2': multiplicative."""
    return image * factor


def adjust_contrast(image, factor):
    """tf.image.adjust_contrast: (x - mean_hw) * f + mean_hw per channel."""
    mean = image.mean(dim=(-3, -2), keepdim=True)
    return (image - mean) * factor + mean


def rgb_to_hsv(rgb):
    r, g, b = rgb[..., 0], rgb[..., 1], rgb[..., 2]
    v = torch.maximum(torch.maximum(r, g), b)
    mn = torch.minimum(torch.minimum(r, g), b)
    rng = v - mn
    s = torch.where(v > 0, rng / torch.where(v > 0, v, torch.ones_like(v)), torch.zeros_like(v))
    norm = 1.0 / (6.0 * torch.where(rng > 0, rng, torch.ones_like(rng)))
    hr = norm * (g - b)
    hg = norm * (b - r) + 2.0 / 6.0
    hb = norm * (r - g) + 4.0 / 6.0
    h = torch.where(r == v, hr, torch.where(g == v, hg, hb))
    h = torch.where(rng > 0, h, torch.zeros_like(h))
    h = torch.where(h < 0, h + 1.0, h)
    return torch.stack([h, s, v], -1)


def hsv_to_rgb(hsv):
    h, s, v = hsv[..., 0], hsv[..., 1], hsv[..., 2]
    dh = h * 6.0
    dr = torch.clamp(torch.abs(dh - 3.0) - 1.0, 0.0, 1.0)
    dg = torch.clamp(2.0 - torch.abs(dh - 2.0), 0.0, 1.0)
    db = torch.clamp(2.0 - torch.abs(dh - 4.0), 0.0, 1.0)
    oms = 1.0 - s
    return torch.stack([(oms + s * dr) * v, (oms + s * dg) * v, (oms + s * db) * v], -1)


def adjust_saturation(image, factor):
    hsv = rgb_to_hsv(image)
    s = torch.clamp(hsv[..., 1] * factor, 0.0, 1.0)
    return hsv_to_rgb(torch.stack([hsv[..., 0], s, hsv[..., 2]], -1))


def adjust_hue(image, delta):
    hsv = rgb_to_hsv(image)
    h = hsv[..., 0] + delta
    h = h - torch.floor(h)          # mod 1
    return hsv_to_rgb(torch.stack([h, hsv[..., 1], hsv[..., 2]], -1))


def to_grayscale(image):
    """tf2/data_util.py:46-50: rgb_to_grayscale weights, tiled to 3 channels."""
    w = torch.tensor([0.2989, 0.5870, 0.1140], dtype=image.dtype, device=image.device)
    g = (image * w).sum(-1, keepdim=True)
    return g.repeat(*([1] * (image.dim() - 1)), 3)


def color_jitter_rand(image, perm, brightness_f, contrast_f, saturation_f, hue_delta):
    """tf2/data_util.py:119-173 with the draws injected.  perm: order of the
    four ops (0 brightness, 1 contrast, 2 saturation, 3 hue); clip after each."""
    for i in perm:
        if i == 0:
            image = random_brightness(image, brightness_f)
        elif i == 1:
            image = adjust_contrast(image, contrast_f)
        elif i == 2:
            image = adjust_saturation(image, saturation_f)
        else:
            image = adjust_hue(image, hue_delta)
        image = torch.clamp(image, 0., 1.)
    return image


def random_color_jitter(image, draws):
    """tf2/data_util.py:382-390.  draws: dict(apply_jitter, perm, brightness,
    contrast, saturation, hue, apply_gray)."""
    if draws['apply_jitter']:
        image = color_jitter_rand(image, draws['perm'], draws['brightness'],
                                  draws['contrast'], draws['saturation'], draws['hue'])
    if draws['apply_gray']:
        image = to_grayscale(image)
    return image


# ---------------------------------------------------------------------------
# Crop + bicubic resize + flip (tf2/data_util.py:246-320, 364-379, 468-469)
# ---------------------------------------------------------------------------

def _keys_cubic_table(a=-0.5, table_size=1024, dtype=torch.float64):
    """TF's bicubic coefficient table (resize_bicubic_op / scale kernel with
    Keys a=-0.5): entry i holds weights for frac = i / 1024."""
    x = torch.arange(table_size + 1, dtype=dtype) / table_size
    w0 = ((a * (x + 1) - 5 * a) * (x + 1) + 8 * a) * (x + 1) - 4 * a
    w1 = ((a + 2) * x - (a + 3)) * x * x + 1
    w2 = ((a + 2) * (1 - x) - (a + 3)) * (1 - x) * (1 - x) + 1
    w3 = ((a * (2 - x) - 5 * a) * (2 - x) + 8 * a) * (2 - x) - 4 * a
    return torch.stack([w0, w1, w2, w3], -1)


def _bicubic_axis_taps(in_size, out_size):
    """The 4 taps of every output index of one axis of TF's bicubic resize (SURVEY A9).

    TF takes the sample position in fp32, each operation rounded on its own (x86 builds do not contract to FMA):
    `CalculateResizeScale` and `HalfPixelScaler` in tensorflow/core/util/image_resizer_state.h give
    scale = (float)in / (float)out and in_f = ((float)o + 0.5f) * scale - 0.5f; `GetWeightsAndIndices` in
    tensorflow/core/kernels/image/resize_bicubic_op.cc takes in = floor(in_f), delta = in_f - in and the table entry
    lrintf(delta * 1024).  The entry's weights are evaluated here in fp64; out-of-range taps get weight 0 (their index
    is clamped into the axis) and the rest are renormalised unless their sum is below 1000 FLT_MIN, as in TF.

    in_size: an integer or an integer array (broadcast over its leading dimensions).
    Returns (idx int64 [..., out, 4], w float64 [..., out, 4])."""
    import numpy as np
    f32 = np.float32
    n = np.asarray(in_size, dtype=np.int64)[..., None]
    o = np.arange(out_size, dtype=f32)
    scale = n.astype(f32) / f32(out_size)
    src = (o + f32(0.5)) * scale - f32(0.5)
    fl = np.floor(src)
    off = np.rint((src - fl) * f32(1024)).astype(np.int64)           # rint: round half to even, as lrintf
    w = _keys_cubic_table(dtype=torch.float64).numpy()[off]
    idx = fl.astype(np.int64)[..., None] - 1 + np.arange(4)
    n = n[..., None]
    w = np.where((idx >= 0) & (idx < n), w, 0.0)
    tot = w.sum(-1, keepdims=True)
    big = np.abs(tot) >= 1000.0 * 1.17549435e-38                      # std::numeric_limits<float>::min()
    w = np.where(big, w / np.where(big, tot, 1.0), w)
    return np.clip(idx, 0, n - 1), w


def _bicubic_axis_weights(in_size, out_size, dtype):
    """Half-pixel-centre bicubic sampling weights (`_bicubic_axis_taps`) as a dense [out,in] matrix."""
    import numpy as np
    idx, w = _bicubic_axis_taps(in_size, out_size)
    W = np.zeros((out_size, in_size))
    np.add.at(W, (np.arange(out_size)[:, None], idx), w)
    return torch.from_numpy(W).to(dtype)


def crop_and_resize_bicubic(image, box, height, width):
    """`tf.image.crop_to_bounding_box` + `tf.image.resize(BICUBIC)`
    (tf2/data_util.py:289-295, 319-320).  box = (y, x, h, w) integers."""
    y, x, h, w = box
    crop = image[y:y + h, x:x + w, :]
    Wy = _bicubic_axis_weights(h, height, image.dtype).to(image.device)
    Wx = _bicubic_axis_weights(w, width, image.dtype).to(image.device)
    return torch.einsum('oh,hwc,pw->opc', Wy, crop, Wx)


def preprocess_for_train(image, height, width, draws, color_jitter_strength=1.0):
    """tf2/data_util.py:443-475 with draws injected: crop box, flip, colour."""
    image = crop_and_resize_bicubic(image, draws['box'], height, width)
    if draws['flip']:
        image = torch.flip(image, dims=[1])
    if color_jitter_strength > 0:
        image = random_color_jitter(image, draws['color'])
    image = image.reshape(height, width, 3)
    return torch.clamp(image, 0., 1.)


CROP_PROPORTION = 0.875  # tf2/data_util.py:22: standard ImageNet central crop


def _compute_crop_shape(image_height, image_width, aspect_ratio, crop_proportion):
    """tf2/data_util.py:175-213 (tf.math.rint = round half to even on fp32 values)."""
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
    """The (y, x, h, w) box of `center_crop` (tf2/data_util.py:216-243)."""
    crop_height, crop_width = _compute_crop_shape(image_height, image_width, width / height, crop_proportion)
    offset_height = ((image_height - crop_height) + 1) // 2
    offset_width = ((image_width - crop_width) + 1) // 2
    return offset_height, offset_width, crop_height, crop_width


def preprocess_for_eval(image, height, width, crop=True):
    """tf2/data_util.py:478-494 on an fp image [Hs,Ws,3] in [0,1]."""
    if crop:
        image = crop_and_resize_bicubic(image, center_crop_box(image.shape[0], image.shape[1], height, width), height, width)
    image = image.reshape(height, width, 3)
    return torch.clamp(image, 0., 1.)
