"""CPU stand-in for kernels.attn_decode_fwd (st5_attn_decode_fwd): the same views in, softmax attention in fp64 out.
Tests install it with monkeypatch to check the host composition around the decode kernel without a GPU."""


def attn_decode_fwd(q, k, v, out, *, H, scale, key_pad=None, probs=None):
    import torch
    B, Tk = k.shape[0], k.shape[1]
    qh = q[:, 0].double().reshape(B, H, 64)
    s = torch.einsum("bhc,bjhc->bhj", qh, k.double().reshape(B, Tk, H, 64)) * scale
    if key_pad is not None:
        s = s.masked_fill(key_pad.bool()[:, None], float("-inf"))
    p = torch.softmax(s, -1)
    out.copy_(torch.einsum("bhj,bjhc->bhc", p, v.double().reshape(B, Tk, H, 64)).reshape(out.shape).to(out.dtype))
    if probs is not None:
        probs.copy_(p.reshape(probs.shape).float())


def install(monkeypatch):
    """Replace the kernel; returns the list every call's argument shapes are appended to."""
    from speecht5_b200 import kernels as K
    calls = []

    def fwd(q, k, v, out, **kw):
        calls.append((tuple(q.shape), tuple(k.shape)))
        attn_decode_fwd(q, k, v, out, **kw)
    monkeypatch.setattr(K, "attn_decode_fwd", fwd)
    return calls
