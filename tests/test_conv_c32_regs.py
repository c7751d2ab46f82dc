"""conv_c32_kernel (the Cin = 32 halo tile computed transposed, weights as the register A operand) against its first form
(conv_c32_kernel_v1, selected for the whole process by YB_CONV_C32_V1=1), bit for bit.

The first form's outputs are computed in a child process with that switch set (`python tests/test_conv_c32_regs.py OUT`); both
processes run the same seeded cases and record which kernel ran, so each comparison is known to be between the two forms.  Cases:
layers1.2 at batch 32 (208 x 208, 32 -> 64) plain and pooled; every C32 shape x Cout of test_conv_contract.py (partial tiles, 1 x 2,
1 x 1 x 37, 37 x 1), pooled where H and W are even; channel-slice outputs with sentinels around them and x_ld > 32; and inputs,
weights and scales chosen so that many outputs are negative, +0 or -0, plain and through the pool.
"""
import os
import subprocess
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, 'yolo2-pytorch_b200'), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)

C32_SHAPES = [(2, 16, 8), (3, 21, 19), (1, 1, 37), (2, 37, 1), (1, 2, 2)]
C32_COUTS = [8, 16, 32, 48, 64]
SENTINEL = 0x7BAD


def _inputs(b, h, w, cout, seed, zeros=False):
    import torch
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(b, h, w, 32, generator=gen)
    wt = torch.randn(cout, 32, 3, 3, generator=gen) * (2.0 / 288) ** 0.5
    scale = torch.rand(cout, generator=gen) + 0.5
    shift = torch.randn(cout, generator=gen) * 0.1
    if zeros:
        # exact zeros of both signs in the input, zero filters, negative scales and +-0 shifts: outputs of +0, -0 and negative values
        # in every pattern a 2x2 window can hold
        x = torch.where(torch.rand(x.shape, generator=gen) < 0.6, torch.zeros_like(x), x)
        x = torch.where(torch.rand(x.shape, generator=gen) < 0.5, -x, x)
        wt[::3] = 0.0
        scale = torch.where(torch.arange(cout) % 2 == 0, -scale, scale)
        shift = torch.where(torch.arange(cout) % 4 < 2, torch.zeros(cout), torch.full((cout,), -0.0))
    return x, wt, scale, shift


def compute():
    """Every case's output (raw fp16 bits as int16, on the CPU) and the names of the conv kernels that ran."""
    import torch
    from b200 import ops
    dev = 'cuda'
    out = {}

    def run(name, b, h, w, cout, seed, pool=False, zeros=False):
        x, wt, scale, shift = _inputs(b, h, w, cout, seed, zeros)
        x16, w16 = x.half().to(dev), ops.pack_weight_f16(wt.to(dev))
        sc, sh = scale.to(dev), shift.to(dev)
        y = ops.conv_bn_act(x16, w16, sc, sh, 0.1, flags=ops.CONV_POOL2X2 if pool else 0)
        out[name] = y.view(torch.int16).cpu()
        if pool:
            return
        # the same output as a channel slice of a wider sentinel-filled buffer, read from an x_ld = 40 input
        buf = torch.full((b, h, w, cout + 24), SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)
        xw = torch.full((b, h, w, 40), float('nan'), dtype=torch.float16, device=dev)
        xw[..., :32] = x16
        ops.conv_bn_act(xw, w16, sc, sh, 0.1, out=buf, y_ch_off=8, cin=32)
        out[name + '/slice'] = buf.view(torch.int16).cpu()

    run('layers1.2', 32, 208, 208, 64, 1)
    run('layers1.2/pool', 32, 208, 208, 64, 1, pool=True)
    for b, h, w in C32_SHAPES:
        for cout in C32_COUTS:
            tag = '%dx%dx%d/%d' % (b, h, w, cout)
            run(tag, b, h, w, cout, h * 100 + w + cout)
            if h % 2 == 0 and w % 2 == 0:
                run(tag + '/pool', b, h, w, cout, h * 100 + w + cout, pool=True)
    for b, h, w, cout in ((2, 32, 24, 64), (1, 22, 18, 48)):
        tag = 'zeros/%dx%dx%d/%d' % (b, h, w, cout)
        run(tag, b, h, w, cout, 7, zeros=True)
        run(tag + '/pool', b, h, w, cout, 7, pool=True, zeros=True)

    from torch.profiler import ProfilerActivity, profile
    x, wt, scale, shift = _inputs(1, 16, 8, 64, 0)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ops.conv_bn_act(x.half().to(dev), ops.pack_weight_f16(wt.to(dev)), scale.to(dev), shift.to(dev), 0.1)
        torch.cuda.synchronize()
    kernels = sorted({e.name for e in prof.events() if 'conv_c32' in e.name})
    return out, kernels


@pytest.mark.gpu
def test_c32_register_a_equals_first_form():
    import torch
    from b200 import ops
    torch.cuda.set_device(0)
    assert not os.environ.get('YB_CONV_C32_V1'), 'this test compares the default form against YB_CONV_C32_V1=1'
    ch = ops.conv_choice(32, 208, 208, 32, 64, 3, flags=ops.CONV_POOL2X2, workspace=False)
    assert (ch['kernel'], ch['bk'], ch['bn']) == ('conv_c32_kernel', 32, 64), ch
    new, new_kernels = compute()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, 'v1.pt')
        env = dict(os.environ, YB_CONV_C32_V1='1')
        cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), path]
        r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        old, old_kernels = torch.load(path)
    assert any(k.endswith('conv_c32_kernel_v1') or 'conv_c32_kernel_v1' in k for k in old_kernels), old_kernels
    assert new_kernels and not any('conv_c32_kernel_v1' in k for k in new_kernels), new_kernels
    assert sorted(new) == sorted(old)
    differ = [k for k in new if not torch.equal(new[k], old[k])]
    assert not differ, 'differs from conv_c32_kernel_v1: %s' % differ
    for k in new:
        if k.endswith('/slice'):
            sl = new[k]
            assert bool((sl[..., :8] == SENTINEL).all()) and bool((sl[..., sl.shape[-1] - 24 + 8:] == SENTINEL).all()), k
    # the signed-zero cases really hold both zeros and negative values
    z = new['zeros/2x32x24/64/pool']
    assert bool((z == 0).any()) and bool((z == -32768).any()) and bool((z < 0).any())


if __name__ == '__main__':
    import torch
    torch.cuda.set_device(0)
    torch.save(compute(), sys.argv[1])
