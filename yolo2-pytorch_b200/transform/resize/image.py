"""transform.resize.image -- `rescale(image, height, width)` of the reference (transform/resize/image.py:23-24:
cv2.resize(image, (width, height))) on the GPU, bit-exact for uint8 HWC images."""
import torch

import transform as _t


def rescale(image, height, width):
    """image: uint8 [h, w, 3] tensor or ndarray -> uint8 CUDA tensor [height, width, 3] (channel order unchanged)."""
    if not torch.is_tensor(image):
        image = torch.from_numpy(image)
    return _t.resize_batch([image], height, width, bgr2rgb=False)[0]


class Rescale(object):
    def __call__(self, image, height, width):
        return rescale(image, height, width)


def fixed(image, height, width):
    """reference transform/resize/image.py:36-46: scale by the tighter of (height / h, width / w) into the top-left of a height x width canvas
    (cv2.warpAffine, zero border).  Shrinking uses INTER_AREA, which warpAffine runs as INTER_LINEAR -- yb_warp_affine_u8, bit-exact;
    enlarging would need warpAffine's INTER_CUBIC tables, which are not built (raises)."""
    import transform.augmentation as _aug
    h, w = int(image.shape[0]), int(image.shape[1])
    scale = height / h if h / w > height / width else width / w
    if scale >= 1:
        raise NotImplementedError('transform.resize.image.fixed: the INTER_CUBIC branch (scale >= 1) is not built')
    return _aug.warp_affine(image, [[scale, 0.0, 0.0], [0.0, scale, 0.0]], (width, height), 0)


class Fixed(object):
    def __call__(self, image, height, width):
        return fixed(image, height, width)
