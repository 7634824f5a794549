"""CPU restatements of the speaker-head kernels (csrc/speaker_head.cu), written the way the kernels compute: row by row,
with the margin logit and its slope as separate closed forms, the smoothing term as N lse - sum z and the gradient
formed from the saved log-sum-exp. `install` puts them (with tests/gemm_emulator.py's GEMM and BatchNorm stand-ins) under
speecht5_b200.kernels, so whole s2c updates run on the CPU."""
import math

import torch

import gemm_emulator

L2_EPS = 1e-12
NONE, AM, AAM = 0, 1, 2


def _margin(margin):
    if margin is None:
        return NONE, 1.0, 0.0, 0
    return int(margin[0]), float(margin[1]), float(margin[2]), int(margin[3])


def margin_logit(c, j, mt, mode, s, m, easy):
    """Row program of margin_logit: c [N] float64 cosines of one row, j column indices, mt the margin column or -1."""
    if mt < 0:
        return c.clone()
    z = s * c
    ct = c[mt]
    if mode == AM:
        z[mt] = s * (ct - m)
    else:
        sine = math.sqrt(min(max(1.0 - ct * ct, 0.0), 1.0))
        phi = ct * math.cos(m) - sine * math.sin(m)
        th, mm = math.cos(math.pi - m), math.sin(math.pi - m) * m
        keep = (ct > 0.0) if easy else (ct > th)
        z[mt] = s * (phi if keep else (ct if easy else ct - mm))
    return z


def margin_slope(c, mt, mode, s, m, easy):
    if mt < 0:
        return torch.ones_like(c)
    d = torch.full_like(c, s)
    if mode == AAM:
        ct = float(c[mt])
        q = 1.0 - ct * ct
        sine = math.sqrt(min(max(q, 0.0), 1.0))
        dsine = -ct / sine if (0.0 <= q <= 1.0 and sine > 0.0) else 0.0
        keep = (ct > 0.0) if easy else (ct > math.cos(math.pi - m))
        d[mt] = s * ((math.cos(m) - dsine * math.sin(m)) if keep else 1.0)
    return d


def margin_ce_fwd(x, mtarget, margin, z_out=None, target=None, eps=0.0, ignore_index=-100, stats=None, lse=None):
    mode, s, m, easy = _margin(margin)
    B, N = x.shape
    j = torch.arange(N)
    for b in range(B):
        c = x[b].double()
        mt = int(mtarget[b]) if mtarget is not None else -1
        z = margin_logit(c, j, mt, mode, s, m, easy)
        if z_out is not None:
            z_out[b] = z.float()
        if target is None:
            continue
        mx = float(z.max())
        ix = int(torch.nonzero(z == mx)[0])
        l = mx + math.log(float(torch.exp(z - mx).sum()))
        t = int(target[b])
        valid = t != ignore_index
        loss = nll = 0.0
        if valid:
            nll = l - float(z[t])
            eps_i = eps / (N - 1)
            loss = (1.0 - eps - eps_i) * nll + eps_i * (N * l - float(z.sum()))
        stats[b] = torch.tensor([loss, nll, float(valid and ix == t), float(valid)])
        lse[b] = l


def margin_ce_bwd(x, mtarget, margin, dx, target=None, eps=0.0, ignore_index=-100, lse=None, gstat=None, dz=None):
    mode, s, m, easy = _margin(margin)
    B, N = x.shape
    j = torch.arange(N)
    for b in range(B):
        c = x[b].double()
        mt = int(mtarget[b]) if mtarget is not None else -1
        if target is not None:
            t = int(target[b])
            if t == ignore_index:
                g = torch.zeros(N, dtype=torch.float64)
            else:
                p = torch.exp(margin_logit(c, j, mt, mode, s, m, easy) - float(lse[b]))
                hit = (j == t).double()
                eps_i = eps / (N - 1)
                g = float(gstat[0]) * ((1.0 - eps - eps_i) * (p - hit) + eps_i * (N * p - 1.0)) + float(gstat[1]) * (p - hit)
        else:
            g = dz[b].double()
        dx[b] = (g * margin_slope(c, mt, mode, s, m, easy)).float()


def l2norm_rows_fwd(x, y, nrm):
    xd = x.double()
    n = xd.norm(dim=1)
    y.copy_((xd / n.clamp_min(L2_EPS)[:, None]).float())
    nrm.copy_(n.float())


def l2norm_rows_bwd(dy, y, nrm, dx, accumulate=False):
    dyd, yd, n = dy.double(), y.double(), nrm.double()
    clamped = n < L2_EPS
    dot = torch.where(clamped, torch.zeros_like(n), (dyd * yd).sum(1))
    g = (dyd - yd * dot[:, None]) / n.clamp_min(L2_EPS)[:, None]
    if accumulate:
        dx.add_(g.to(dx.dtype))
    else:
        dx.copy_(g.to(dx.dtype))


def time_mean_fwd(x, y):
    y.copy_(x.double().mean(1).to(y.dtype))


def time_mean_bwd(dy, dx):
    dx.copy_((dy.double()[:, None, :] / dx.shape[1]).expand(dx.shape).to(dx.dtype))


def batch_norm_act(x, bn, training, act=None, drop_p=0.0):
    """ops.batch_norm_act as a differentiable torch call with BatchNorm1d's running statistics (eval reads them,
    training updates them)."""
    assert drop_p == 0.0 and act is None
    if training and bn.num_batches_tracked is not None:
        bn.num_batches_tracked += 1
    y = torch.nn.functional.batch_norm(x.float(), bn.running_mean, bn.running_var, bn.weight, bn.bias, training,
                                       bn.momentum, bn.eps)
    return y.to(x.dtype)


def install(monkeypatch):
    """The speaker-head kernels + gemm_emulator.install_trainer, BatchNorm with running statistics, and the waveform
    feature extractor without its CUDA guard."""
    gemm_emulator.install_trainer(monkeypatch)
    from speecht5_b200 import frontend, kernels as K, ops
    for name in ("margin_ce_fwd", "margin_ce_bwd", "l2norm_rows_fwd", "l2norm_rows_bwd", "time_mean_fwd",
                 "time_mean_bwd"):
        monkeypatch.setattr(K, name, globals()[name])
    monkeypatch.setattr(ops, "batch_norm_act", batch_norm_act)
    monkeypatch.setattr(frontend.ConvFeatureExtractor, "forward", lambda self, wave: self._layers(wave))
