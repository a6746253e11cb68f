"""Process-wide defaults mirroring neupan/configuration/__init__.py:25-57.

The reference keeps ``device`` / ``time_print`` / ``tensor_dtype`` as mutable module globals
(set from the yaml at neupan/neupan.py:68-69).  They are kept for API compatibility; this
build additionally carries the device per PAN instance, so two planners on different GPUs can
coexist (the globals only provide the default for helpers called without an instance).
"""
import numpy as np
import torch

device = torch.device("cpu")
time_print = False
tensor_dtype = torch.float32


def np_to_tensor(array, requires_grad=False):
    if np.isscalar(array):
        out = torch.tensor(array, dtype=tensor_dtype).to(device)
    else:
        out = torch.from_numpy(np.asarray(array)).type(tensor_dtype).to(device)
    if requires_grad:
        out.requires_grad_()
    return out


def tensor_to_np(tensor):
    if tensor is None:
        return None
    return tensor.detach().cpu().numpy()


def value_to_tensor(value, requires_grad=False):
    if value is None:
        return None
    if isinstance(value, torch.Tensor):
        value = value.detach().cpu().numpy()
    return torch.tensor(value, dtype=tensor_dtype, requires_grad=requires_grad).to(device)


def to_device(tensor):
    return tensor.to(device)
