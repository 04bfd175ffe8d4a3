"""float64 restatement of torch.nn.utils.spectral_norm (n_power_iterations=1, eps=1e-12, dim=0) and of its adjoint,
shared by tests/test_spectral_norm_host.py (against torch's autograd) and tests/test_gpu_spectral_norm.py (against the
kernels)."""
import torch

EPS = 1e-12


def power_iteration64(W, u, v, iterate=True):
    """-> (u, v, sigma, W_bar) in float64.  iterate: v = normalize(W^T u), u = normalize(W v) first (training mode)."""
    Wm = W.double().reshape(W.shape[0], -1)
    u, v = u.double(), v.double()
    if iterate:
        t = Wm.t() @ u
        v = t / max(float(t.norm()), EPS)
        s = Wm @ v
        u = s / max(float(s.norm()), EPS)
    sigma = u @ (Wm @ v)
    return u, v, sigma, W.double() / sigma


def adjoint64(G, W_bar, u, v, sigma):
    """dL/dweight_orig from G = dL/dW_bar, with u and v held constant: (G - <G, W_bar> u v^T) / sigma."""
    Gm = G.double().reshape(G.shape[0], -1)
    d = (Gm * W_bar.double().reshape(Gm.shape)).sum()
    return ((Gm - d * torch.outer(u.double(), v.double())) / sigma).reshape(G.shape)


def sn_config(c_in=80):
    import oracle.ae_oracle as orc
    cfg = orc.default_config(c_in)
    cfg["Decoder"]["sn"] = True
    return cfg


def state_checksum(sd):
    return torch.tensor([float(sum(v.double().sum() for v in sd.values())),
                         float(sum(v.double().abs().sum() for v in sd.values()))])
