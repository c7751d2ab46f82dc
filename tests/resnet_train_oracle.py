"""Train-mode restatement of the ResNet plugin (reference model/resnet.py:28-142 under nn.Module.train()) for the training tests and the
`resnet_train.npz` generator: the same arithmetic as `oracle.yolo2_oracle.resnet_forward`, with every BatchNorm on batch statistics (as
nn.BatchNorm2d does in train mode) and each one's batch mean / biased variance recorded, so the running-statistic update of one step can be
restated as (1 - momentum) * old + momentum * batch statistic (unbiased variance)."""
import torch.nn.functional as F

from oracle import yolo2_oracle as O

MOMENTUM = 0.1      # nn.BatchNorm2d's default, which the reference's ResNet keeps


def resnet_train_forward(sd, x, name='resnet18', stats=None, counts=None):
    """x [B,3,H,W] fp32 -> head feature; `stats[bn prefix] = (batch mean, biased batch variance)` and `counts[bn prefix]` = values per channel
    (B x H x W of the BatchNorm's input) when given."""
    def bn(y, prefix):
        if stats is not None:
            stats[prefix] = (y.mean(dim=(0, 2, 3)), y.var(dim=(0, 2, 3), unbiased=False))
        if counts is not None:
            counts[prefix] = y.numel() // y.shape[1]
        return F.batch_norm(y, None, None, sd[prefix + '.weight'], sd[prefix + '.bias'], True, 0.0, 1e-5)

    x = F.relu(bn(F.conv2d(x, sd['conv1.weight'], None, 2, 3), 'bn1'))
    x = F.max_pool2d(x, 3, 2, 1)
    for b in O.resnet_blocks(name):
        p = b['prefix']
        residual = x
        if b['kind'] == 'basic':
            out = F.relu(bn(F.conv2d(x, sd[p + '.conv1.weight'], None, b['stride'], 1), p + '.bn1'))
            out = bn(F.conv2d(out, sd[p + '.conv2.weight'], None, 1, 1), p + '.bn2')
        else:
            out = F.relu(bn(F.conv2d(x, sd[p + '.conv1.weight']), p + '.bn1'))
            out = F.relu(bn(F.conv2d(out, sd[p + '.conv2.weight'], None, b['stride'], 1), p + '.bn2'))
            out = bn(F.conv2d(out, sd[p + '.conv3.weight']), p + '.bn3')
        if b['downsample']:
            residual = bn(F.conv2d(x, sd[p + '.downsample.0.weight'], None, b['stride']), p + '.downsample.1')
        x = F.relu(out + residual)
    return F.conv2d(x, sd['conv.weight'], sd['conv.bias'])


def expected_running(sd0, prefix, mean, var, count):
    """Running mean / variance after one train-mode step from the recorded batch statistics over `count` values per channel."""
    return ((1 - MOMENTUM) * sd0[prefix + '.running_mean'] + MOMENTUM * mean.detach(),
            (1 - MOMENTUM) * sd0[prefix + '.running_var'] + MOMENTUM * var.detach() * count / (count - 1))
