import torch


def to_device_tensor(x, device, dtype=None):
    """numpy / tensor -> contiguous CUDA tensor (host arrays go through one H2D copy)."""
    if not torch.is_tensor(x):
        x = torch.as_tensor(x)
    if dtype is not None and x.dtype != dtype:
        x = x.to(dtype)
    if x.device != device:
        x = x.to(device, non_blocking=True)
    return x.contiguous()


def model_device(model):
    try:
        return next(model.parameters()).device
    except StopIteration:
        return torch.device('cuda' if torch.cuda.is_available() else 'cpu')


def ensure_cuda(model, name):
    dev = model_device(model)
    if dev.type != 'cuda':
        if not torch.cuda.is_available():
            raise RuntimeError('%s: parl_b200 algorithms run on the H100 only (no CPU fallback) and no CUDA '
                               'device is visible' % name)
        model.to(torch.device('cuda', torch.cuda.current_device()))
        dev = model_device(model)
    return dev
