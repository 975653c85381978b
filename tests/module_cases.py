"""Module-level cases of the boundary (SURVEY 8b): ZoneoutLSTMCell / DropoutLSTMCell (modules/layers.py:18-47), Conv1dGenerated /
BatchNorm1dGenerated (modules/generated.py:7-96) and LocationSensitiveAttention (modules/attention.py:6-86).

Each case runs one module class on one device and returns its outputs and gradients.  Parameters and inputs come from seeded
generators, so the same numbers reach the unmodified reference's classes (tests/golden/make_golden_modules.py, CPU fp32, result
stored in tests/golden/modules.npz) and this package's classes on the GPU (tests/test_gpu_modules.py).  Large tensors are stored as a
fixed seeded sample of SAMPLE elements plus the full tensor's largest magnitude (the scale of the absolute tolerances).
"""
import numpy as np
import torch

SAMPLE = 8192


def seeded_params(module, seed, scale=1.0):
    """Every parameter (in name order) ~ U(-scale / sqrt(fan), scale / sqrt(fan)), fan = last dimension (first for vectors)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for _, p in sorted(module.named_parameters()):
            fan = p.shape[-1] if p.dim() > 1 else p.shape[0]
            p.copy_((torch.rand(p.shape, generator=g) * 2 - 1) * (scale / fan ** 0.5))


def sample_index(n):
    return torch.randint(0, n, (SAMPLE,), generator=torch.Generator().manual_seed(n))


def lstm_case(kind, cell, device):
    """Eval mode: one cell step, gradients of <h, gh> + <c, gc>."""
    I, H, B = 544, 1024, 7
    seeded_params(cell, 11)
    cell = cell.to(device).eval()
    g = torch.Generator().manual_seed(3)
    x, h, c = torch.randn(B, I, generator=g), torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)
    gh, gc = torch.randn(B, H, generator=g), torch.randn(B, H, generator=g)
    xo, ho, co = (t.to(device).requires_grad_(True) for t in (x, h, c))
    h1, c1 = cell(xo, ho, co)
    ((h1 * gh.to(device)).sum() + (c1 * gc.to(device)).sum()).backward()
    out = {'h': h1, 'c': c1, 'dx': xo.grad, 'dh': ho.grad, 'dc': co.grad}
    out.update({'d' + n: p.grad for n, p in cell.named_parameters()})
    return {k: v.detach().float().cpu() for k, v in out.items()}


def conv_case(train, conv, bn, device):
    """Grouped generated convolution (valid padding) -> generated batch norm, gradients of <z, gz>, running statistics."""
    G, gd, Cin, k, dil, NB, L = 3, 6, 8, 3, 2, 4, 21
    seeded_params(conv, 21)
    seeded_params(bn, 22)
    conv, bn = conv.to(device).train(train), bn.to(device).train(train)
    g = torch.Generator().manual_seed(5)
    e = torch.randn(G, gd, generator=g)
    x = torch.randn(NB, G * Cin, L + (k - 1) * dil, generator=g)      # the caller pads (ConvBlockGenerated pads before the convolution)
    eo, xo = e.to(device).requires_grad_(True), x.to(device).requires_grad_(True)
    y = conv(eo, xo)
    z = bn(eo, y)
    gz = torch.randn(z.shape, generator=g)
    (z * gz.to(device)).sum().backward()
    out = {'y': y, 'z': z, 'de': eo.grad, 'dx': xo.grad, 'running_mean': bn.running_mean, 'running_var': bn.running_var,
           'num_batches_tracked': bn.num_batches_tracked}
    out.update({'dconv.' + n: p.grad for n, p in conv.named_parameters()})
    out.update({'dbn.' + n: p.grad for n, p in bn.named_parameters()})
    return {k: v.detach().float().cpu() for k, v in out.items()}


ATT_DIMS = dict(B=5, L=37, M=288, D=1024, A=128, C=32, K=31)


def attention_case(att, device):
    """reset + three forward steps with gradients through the carried cumulative weights."""
    B, L, M, D = (ATT_DIMS[k] for k in 'BLMD')
    seeded_params(att, 31, scale=3.0)
    att = att.to(device)
    g = torch.Generator().manual_seed(7)
    lens = torch.tensor([37, 30, 37, 12, 25])
    mask = (torch.arange(L)[None, :] < lens[:, None]).to(device)
    memory = torch.randn(B, L, M, generator=g)
    queries = [torch.randn(B, D, generator=g) for _ in range(3)]
    mo = memory.to(device).requires_grad_(True)
    qo = [q.to(device).requires_grad_(True) for q in queries]
    att.reset(mo, B, L, mo.device)
    out, loss = {}, 0.0
    for step in range(3):
        c, w = att(qo[step], mo, mask, None)
        out[f'context{step}'], out[f'weights{step}'] = c, w
        gc, gw = torch.randn(B, M, generator=g), torch.randn(B, L, generator=g)
        loss = loss + (c * gc.to(device)).sum() + (w * gw.to(device)).sum()
    loss.backward()
    out['dmemory'] = mo.grad
    out.update({f'dquery{s}': qo[s].grad for s in range(3)})
    out.update({'d' + n: p.grad for n, p in att.named_parameters()})
    return {k: v.detach().float().cpu() for k, v in out.items()}


def pack(prefix, result):
    """{prefix.key: full array, or SAMPLE seeded elements} + {prefix.key.absmax: largest magnitude of the full tensor}."""
    out = {}
    for k, v in result.items():
        flat = v.reshape(-1)
        out[f'{prefix}.{k}.absmax'] = np.array([float(flat.abs().max()) if flat.numel() else 0.0], dtype=np.float32)
        out[f'{prefix}.{k}'] = (flat[sample_index(flat.numel())] if flat.numel() > 2 * SAMPLE else flat).numpy().astype(np.float32)
    return out


def unpack_like(stored, prefix, key, tensor):
    """The elements of `tensor` that `pack` stored for prefix.key (same sampling), as a CPU fp32 vector."""
    flat = tensor.detach().float().reshape(-1).cpu()
    ref = torch.from_numpy(stored[f'{prefix}.{key}'])
    return (flat[sample_index(flat.numel())] if flat.numel() > 2 * SAMPLE else flat), ref, float(stored[f'{prefix}.{key}.absmax'][0])
