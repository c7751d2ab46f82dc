"""transform -- the part of the reference's `transform/` package that sits immediately upstream of the network input
(SURVEY 8f rank 2), on the GPU: `transform.resize.image.rescale`, `transform.resize.label.rescale`,
`transform.image.BGR2RGB`, and the batched `transform.resize_batch` that does all three for a whole batch of decoded
frames in one launch -- optionally through the horizontal flip and the random-crop window of the reference's training pipeline
(`transform.augmentation.flip_horizontally`, `transform.resize.label.random_crop`), which are index transforms on the source of the same
resize; `transform.augmentation.random_rotate` / `Rotator` and `transform.resize.image.fixed` (shrinking) run cv2.warpAffine's bilinear path in
one kernel.  The photometric augmentations of `transform/image.py` (RandomBlur, BGR2HSV, RandomHue, RandomSaturation, RandomBrightness,
HSV2RGB, RandomGamma) run bit-exactly with cv2 in one launch per chain segment over the resized batch (`transform.image.Compose`);
`parse_transform` / `get_transform` build a configured sequence such as `transform/image_train` the way the reference does.
`TensorTransform` is the tensor chain that follows them (`[transform] tensor`: ToTensor, then per-channel Normalize), compiled into a
per-channel table that the backbones' first-layer kernels read uint8 frames through."""
import inspect

import torch

from b200 import ops as _ops


def parse_transform(config, method):
    """A dotted name such as 'transform.image.RandomBlur' -> an instance, given `config` when its constructor takes one (reference
    transform/__init__.py); anything else is returned as is."""
    if isinstance(method, str):
        import utils
        attr = utils.parse_attr(method)
        return attr(config) if len(inspect.signature(attr).parameters) == 1 else attr()
    return method


def get_transform(config, sequence, compose=None):
    """`sequence` (dotted names or instances) -> `compose(list)`, by default `transform.image.Compose`, which compiles the image ops
    into device launches."""
    if compose is None:
        from transform.image import Compose as compose
    return compose([parse_transform(config, method) for method in sequence])


class TensorTransform(object):
    """The reference's `[transform] tensor` chain, built as `get_transform(config, config.get('transform', 'tensor').split(),
    compose=TensorTransform)`: torchvision.transforms.ToTensor followed by zero or more 3-channel Normalizes (transform.image.Normalize or
    torchvision's own).  Anything else raises ValueError naming the item.

    The chain is compiled by running its own objects once on the CPU over a uint8 image that holds every byte value in every channel, so
    `table[c][v]` (fp32 [3, 256]) is bit for bit what torchvision computes for byte v in channel c.  `lut(device)` is that table on a device
    (cached; a backbone's first-layer `_lut` kernel reads through it), and calling the transform on a uint8 CUDA batch [B, H, W, 3] returns
    the fp32 [B, 3, H, W] image in one launch."""

    def __init__(self, sequence):
        import torchvision
        self.transforms = list(sequence)
        for i, t in enumerate(self.transforms):
            if i == 0:
                if not isinstance(t, torchvision.transforms.ToTensor):
                    raise ValueError('TensorTransform: the chain must start with torchvision.transforms.ToTensor, not %r' % (t,))
            elif not isinstance(t, torchvision.transforms.Normalize):
                raise ValueError('TensorTransform: only 3-channel Normalizes may follow ToTensor, not %r' % (t,))
            elif torch.as_tensor(t.mean).numel() != 3 or torch.as_tensor(t.std).numel() != 3:
                raise ValueError('TensorTransform: %r is not a 3-channel Normalize' % (t,))
        if not self.transforms:
            raise ValueError('TensorTransform: the chain must start with torchvision.transforms.ToTensor, not an empty chain')
        image = torch.arange(256, dtype=torch.uint8).view(256, 1, 1).expand(256, 1, 3).numpy().copy()
        x = image
        for t in self.transforms:
            x = t(x)
        if x.dtype != torch.float32:
            raise ValueError('TensorTransform: the chain yields %s, not float32' % (x.dtype,))
        self.table = x[:, :, 0].contiguous()
        self._luts = {}

    def __repr__(self):
        return 'TensorTransform(%r)' % (self.transforms,)

    def lut(self, device):
        """The table as a CUDA tensor fp32 [3, 256] on `device`, allocated once per device (never inside a CUDA-graph capture: call the
        transform or an eager forward before capturing)."""
        device = torch.device(device)
        t = self._luts.get(device)
        if t is None:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError('TensorTransform: the table for %s is first needed inside a CUDA-graph capture; run once eagerly before '
                                   'capturing' % device)
            t = self._luts[device] = self.table.to(device)
        return t

    def __call__(self, frames_u8):
        """uint8 CUDA tensor [B, H, W, 3] -> float32 [B, 3, H, W], what the chain computes frame by frame (yb_totensor_lut_u8)."""
        if not (isinstance(frames_u8, torch.Tensor) and frames_u8.is_cuda and frames_u8.dtype == torch.uint8 and frames_u8.dim() == 4
                and frames_u8.shape[3] == 3):
            raise RuntimeError('TensorTransform: expected a uint8 CUDA tensor [B, H, W, 3]')
        frames_u8 = frames_u8.contiguous()
        b, h, w, _ = frames_u8.shape
        out = torch.empty(b, 3, h, w, dtype=torch.float32, device=frames_u8.device)
        _ops.call('yb_totensor_lut_u8', frames_u8, self.lut(frames_u8.device), out, b, h, w)
        return out


_TO_TENSOR = None


def to_tensor_transform():
    """TensorTransform([ToTensor()]): the table a backbone reads uint8 frames through when no input transform is set."""
    global _TO_TENSOR
    if _TO_TENSOR is None:
        import torchvision
        _TO_TENSOR = TensorTransform([torchvision.transforms.ToTensor()])
    return _TO_TENSOR


def resize_batch(frames, height, width, bgr2rgb=True, yx_min=None, yx_max=None, flip=None, crop=None, margin=None):
    """frames: list of uint8 [h_i, w_i, 3] tensors (CPU or CUDA; BGR as cv2.imread gives them) -> uint8 CUDA tensor
    [B, height, width, 3], cv2.resize-exact, RGB when `bgr2rgb`.  Optional padded boxes yx_min / yx_max [B, G, 2] (source
    pixels) are returned scaled by (height / h_i, width / w_i) like transform.resize.label.rescale.  One kernel launch;
    the result can be fed straight to the model (`Darknet.forward` accepts uint8 NHWC frames).
    Training form: `flip` (B booleans: cv2.flip(frame, 1) first), `crop` ([B][4] ints (y0, x0, y1, x1): frame[y0:y1, x0:x1] next) and
    `margin` ([B][2] float32: what the reference subtracts from the boxes for that crop) -- see transform.resize.label.random_crop."""
    dev = torch.device('cuda', torch.cuda.current_device())
    sizes, offs, total = [], [], 0
    for f in frames:
        if f.dtype != torch.uint8 or f.dim() != 3 or f.shape[2] != 3:
            raise ValueError('frames must be uint8 [h, w, 3]')
        sizes += [int(f.shape[0]), int(f.shape[1])]
        offs.append(total)
        total += f.numel()
    packed = torch.empty(total, dtype=torch.uint8, device=dev)
    for f, o in zip(frames, offs):
        packed[o:o + f.numel()].copy_(f.reshape(-1), non_blocking=True)
    src_off = torch.tensor(offs, dtype=torch.int64).to(dev, non_blocking=True)
    src_hw = torch.tensor(sizes, dtype=torch.int32).to(dev, non_blocking=True)
    out = torch.empty(len(frames), height, width, 3, dtype=torch.uint8, device=dev)
    slots = 0
    if yx_min is not None:
        yx_min = yx_min.to(device=dev, dtype=torch.float32).contiguous().clone()
        yx_max = yx_max.to(device=dev, dtype=torch.float32).contiguous().clone()
        slots = yx_min.shape[1]
    if flip is None and crop is None:
        _ops.call('yb_resize_batch_u8', packed, src_off, src_hw, out, len(frames), int(height), int(width), int(bool(bgr2rgb)), yx_min, yx_max, slots)
        return (out, yx_min, yx_max) if yx_min is not None else out
    flip_t = crop_t = margin_t = None
    if flip is not None:
        flip_t = torch.tensor([int(bool(f)) for f in flip], dtype=torch.uint8).to(dev, non_blocking=True)
    if crop is not None:
        crop_t = torch.as_tensor(crop, dtype=torch.int32).reshape(len(frames), 4).to(dev, non_blocking=True)
        if margin is None:
            margin = [[c[0], c[1]] for c in crop_t.tolist()]
        margin_t = torch.as_tensor(margin, dtype=torch.float32).reshape(len(frames), 2).to(dev, non_blocking=True)
        for (y0, x0, y1, x1), (h, w) in zip(torch.as_tensor(crop).reshape(-1, 4).tolist(), zip(sizes[0::2], sizes[1::2])):
            if not (0 <= y0 < y1 <= h and 0 <= x0 < x1 <= w):
                raise ValueError('crop window (%d, %d, %d, %d) outside a %d x %d frame' % (y0, x0, y1, x1, h, w))
    _ops.call('yb_resize_aug_batch_u8', packed, src_off, src_hw, crop_t, margin_t, flip_t, out, len(frames), int(height), int(width), int(bool(bgr2rgb)),
              yx_min, yx_max, slots)
    return (out, yx_min, yx_max) if yx_min is not None else out


def to_tensor(frames_u8):
    """uint8 CUDA tensor [B, H, W, 3] -> float32 [B, 3, H, W] in [0, 1] (torchvision ToTensor, one kernel).  The training
    forward needs this form; inference takes the uint8 batch directly."""
    if not (isinstance(frames_u8, torch.Tensor) and frames_u8.is_cuda and frames_u8.dtype == torch.uint8 and frames_u8.dim() == 4 and frames_u8.shape[3] == 3):
        raise RuntimeError('transform.to_tensor: expected a uint8 CUDA tensor [B, H, W, 3]')
    frames_u8 = frames_u8.contiguous()
    b, h, w, _ = frames_u8.shape
    out = torch.empty(b, 3, h, w, dtype=torch.float32, device=frames_u8.device)
    _ops.call('yb_totensor_u8', frames_u8, out, b, h, w)
    return out
