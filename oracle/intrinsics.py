"""CPU oracle of demon_b200.images.adjust_intrinsics: the image branch of the reference's `adjust_intrinsics`
(dataset_tools/view_tools.py:97-172) restated with Pillow, `Image.resize` followed by a crop that fills with (127, 127, 127)
where the crop box leaves the resized image.

One deliberate deviation from the reference: for a box that leaves the image, its `safe_crop_image`
(dataset_tools/helpers.py:74-103) pastes the WHOLE resized image at (max(-x0, 0), max(-y0, 0)).  That is the crop only when
x0 <= 0 and y0 <= 0; with x0 > 0 or y0 > 0 the principal point ends up x0 or y0 pixels away from where K_new puts it.
`crop_with_fill` here (and the device kernel) returns the crop, output pixel (u, v) = resized pixel (x0 + u, y0 + v).
`reference_safe_crop` restates what safe_crop_image returns, so that tests can show both sides of that line.
"""
import numpy as np

FILL = 127


def window(K, K_new, w, h):
    """The reference's arithmetic for a w x h image with intrinsics K = (fx, fy, cx, cy) and target K_new, in Python floats:
    -> (rw, rh, x0, y0, bilinear): the size of the resize (int() truncates), the crop offset (round() is half to even) and
    the filter (BILINEAR if scale_x > 1, else LANCZOS, on both axes)."""
    fx, fy, cx, cy = (float(v) for v in K)
    fx_new, fy_new, cx_new, cy_new = (float(v) for v in K_new)
    scale_x, scale_y = fx_new / fx, fy_new / fy
    rw, rh = int(w * scale_x), int(h * scale_y)
    x0, y0 = int(round(cx * scale_x - cx_new)), int(round(cy * scale_y - cy_new))
    return rw, rh, x0, y0, scale_x > 1


def leaves(rw, rh, x0, y0, width_new, height_new):
    """The reference's condition for its warning 'Adjusting intrinsics adds a border to the image'."""
    return x0 < 0 or y0 < 0 or x0 + width_new > rw or y0 + height_new > rh


def crop_with_fill(img, x0, y0, width_new, height_new, fill=FILL):
    """img [h,w,3] uint8 -> [height_new,width_new,3]: pixel (u, v) is img[y0 + v, x0 + u] inside img, `fill` outside."""
    h, w = img.shape[:2]
    out = np.full((height_new, width_new) + img.shape[2:], fill, dtype=img.dtype)
    ya, yb = max(y0, 0), min(y0 + height_new, h)
    xa, xb = max(x0, 0), min(x0 + width_new, w)
    if ya < yb and xa < xb:
        out[ya - y0:yb - y0, xa - x0:xb - x0] = img[ya:yb, xa:xb]
    return out


def reference_safe_crop(img, x0, y0, width_new, height_new, fill=FILL):
    """What the reference's safe_crop_image returns for a box that leaves the image: the whole image pasted at
    (max(-x0, 0), max(-y0, 0)) into a fill-coloured canvas (Pillow's paste clips at the canvas)."""
    out = np.full((height_new, width_new) + img.shape[2:], fill, dtype=img.dtype)
    x, y = max(-x0, 0), max(-y0, 0)
    part = img[:max(height_new - y, 0), :max(width_new - x, 0)]
    out[y:y + part.shape[0], x:x + part.shape[1]] = part
    return out


def adjust_image(img, K, K_new, width_new, height_new):
    """img [h,w,3] uint8, K and K_new (fx, fy, cx, cy) in pixels -> (the adapted image [height_new,width_new,3] uint8,
    status 0, or 1 where the crop left the resized image)."""
    from PIL import Image
    h, w = img.shape[:2]
    rw, rh, x0, y0, bilinear = window(K, K_new, w, h)
    resized = Image.fromarray(np.ascontiguousarray(img)).resize((rw, rh), Image.Resampling.BILINEAR if bilinear else Image.Resampling.LANCZOS)
    return crop_with_fill(np.asarray(resized), x0, y0, width_new, height_new), int(leaves(rw, rh, x0, y0, width_new, height_new))


def reference_safe_crop_image():
    """The reference's own safe_crop_image from its dataset_tools/helpers.py next to DEMON_REF_SRC, or None where that tree
    is absent or the module does not import (it needs Pillow and scipy.ndimage.filters)."""
    import importlib.util
    import os
    from .ref import REF_SRC
    path = os.path.normpath(os.path.join(REF_SRC, "..", "..", "python", "depthmotionnet", "dataset_tools", "helpers.py")) if REF_SRC else ""
    if not os.path.isfile(path):
        return None
    try:
        spec = importlib.util.spec_from_file_location("reference_dataset_helpers", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    except ImportError:
        return None
    return mod.safe_crop_image
