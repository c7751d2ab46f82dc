"""utils.train -- checkpoint files on either side of the GPU path (host code, no kernel).

Same names and on-disk format as the reference's `utils/train.py` (file:line cited per item), so a model directory written by the
reference is read here and vice versa:
  <model_dir>/<step>.pth     torch.save(OrderedDict(name -> CPU tensor))           (train.py:419, utils/train.py:103-111)
  <model_dir>/<step>.epoch   the epoch number as text, optional                    (utils/train.py:108-110)
`load_checkpoint` adds what a torch >= 0.4 process needs to read a torch 0.3.1 file: those files carry no `num_batches_tracked`
buffers (SURVEY 8f rank 1), every other key must match.
"""
import collections
import logging
import os
import time

import torch


class Timer(object):
    """`timer()` is True once every `max` seconds (utils/train.py:26-48); `first` makes the very first call fire."""
    def __init__(self, max, first=True):
        self.max = max
        self.start = 0 if first else time.time()

    def __call__(self):
        now = time.time()
        if now - self.start > self.max:
            self.start = now
            return True
        return False


def _steps(model_dir, ext):
    found = []
    for entry in os.listdir(model_dir):
        name, e = os.path.splitext(entry)
        if e == ext and name.isdigit():
            found.append((int(name), name))
    return sorted(found)


def load_model(model_dir, step=None, ext='.pth', ext_epoch='.epoch', logger=logging.info):
    """(path, step, epoch) of the checkpoint with the largest step, or of `step` (utils/train.py:51-78); epoch is None without an epoch file."""
    if step is None:
        steps = _steps(model_dir, ext)
        if not steps:
            raise FileNotFoundError('no <step>%s checkpoint in %s' % (ext, model_dir))
        step, name = steps[-1]
    else:
        name = str(step)
    prefix = os.path.join(model_dir, name)
    if logger is not None:
        logger('load %s.*' % prefix)
    try:
        with open(prefix + ext_epoch, 'r') as f:
            epoch = int(f.read())
    except (FileNotFoundError, ValueError):
        epoch = None
    path = prefix + ext
    assert os.path.exists(path), path
    return path, step, epoch


class Saver(object):
    """Keeps the `keep` newest checkpoints of a model directory (utils/train.py:81-126)."""
    def __init__(self, model_dir, keep, ext='.pth', ext_epoch='.epoch', logger=logging.info):
        self.model_dir, self.keep, self.ext, self.ext_epoch = model_dir, keep, ext, ext_epoch
        self.logger = (lambda s: s) if logger is None else logger

    def __call__(self, obj, step, epoch=None):
        os.makedirs(self.model_dir, exist_ok=True)
        prefix = os.path.join(self.model_dir, str(step))
        torch.save(obj, prefix + self.ext)
        if epoch is not None:
            with open(prefix + self.ext_epoch, 'w') as f:
                f.write(str(epoch))
        self.logger('model saved into %s.*' % prefix)
        self.tidy()
        return prefix

    def tidy(self):
        steps = _steps(self.model_dir, self.ext)
        for _, name in steps[:max(0, len(steps) - self.keep)]:
            prefix = os.path.join(self.model_dir, name)
            os.remove(prefix + self.ext)
            try:
                os.remove(prefix + self.ext_epoch)
            except FileNotFoundError:
                self.logger(prefix + self.ext_epoch + ' not found')


def load_sizes(config):
    """`[data] sizes = 320,320 416,416 ...` -> [(height, width)] (utils/train.py:129-131)."""
    return [tuple(int(v) for v in pair.split(',')) for pair in config.get('data', 'sizes').split()]


def state_dict_cpu(module):
    """What the reference hands to its Saver (train.py:419): an OrderedDict of CPU tensors."""
    return collections.OrderedDict((key, var.detach().cpu()) for key, var in module.state_dict().items())


def load_checkpoint(path_or_dir, step=None, logger=logging.info):
    """(state_dict, step, epoch) from a checkpoint file or a model directory (detect.py:93-94, train.py:313-314)."""
    epoch = None
    path = path_or_dir
    if os.path.isdir(path_or_dir):
        path, step, epoch = load_model(path_or_dir, step, logger=logger)
    return torch.load(path, map_location='cpu'), step, epoch


def load_state_dict(module, state_dict):
    """`module.load_state_dict(state_dict)` (detect.py:96) that also accepts files written by torch 0.3.1: BatchNorm's `num_batches_tracked`
    (added in torch 0.4) may be absent -- those buffers keep their value; any other missing or unexpected key is an error."""
    result = module.load_state_dict(state_dict, strict=False)
    missing = [k for k in result.missing_keys if not k.endswith('num_batches_tracked')]
    if missing or result.unexpected_keys:
        raise RuntimeError('checkpoint does not match the model: missing %s, unexpected %s' % (missing[:5], list(result.unexpected_keys)[:5]))
    return result
