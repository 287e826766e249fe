"""Field objects with the small slice of the Taichi field API the reference's callers use
(``.to_numpy()``, ``.from_numpy()``, ``.fill()``, ``[...]`` element access, ``.shape``), backed by
torch CUDA tensors in the reference's public layout (particle_system.py:102-145).

The engine keeps the authoritative state in packed, sorted SoA buffers; a ``Field`` asks its
owner to materialise the public tensors before a read (``owner._pull()``) and tells it about
writes (``owner._touch()``) so the next engine call re-packs them.
"""
from __future__ import annotations

import numpy as np
import torch


class Field:
    def __init__(self, owner, tensor: torch.Tensor, name: str, derived: bool = False):
        self._owner = owner
        self.tensor = tensor
        self.name = name
        self._derived = derived  # engine output only (grid_ids, grid_particles_num)

    @property
    def shape(self):
        s = tuple(self.tensor.shape)
        # a Vector.field(3, ..., shape=n) reports shape (n,)
        return s[:1] if len(s) == 2 else s

    @property
    def dtype(self):
        return self.tensor.dtype

    def to_numpy(self):
        self._owner._pull(self)
        return self.tensor.detach().cpu().numpy()

    def to_torch(self, device=None):
        self._owner._pull(self)
        t = self.tensor.clone()
        return t.to(device) if device is not None else t

    def from_numpy(self, arr):
        self._owner._pull(self)
        src = torch.from_numpy(np.ascontiguousarray(arr)).to(self.tensor.dtype)
        if tuple(src.shape) != tuple(self.tensor.shape):
            raise ValueError(f"{self.name}: shape {tuple(src.shape)} != {tuple(self.tensor.shape)}")
        self.tensor.copy_(src)
        self._owner._touch(self)

    def fill(self, value):
        self._owner._pull(self)
        self.tensor.fill_(value)
        self._owner._touch(self)

    def __getitem__(self, idx):
        self._owner._pull(self)
        if idx is None:
            idx = ()
        out = self.tensor[idx]
        return out.item() if out.dim() == 0 else out.detach().cpu().numpy()

    def __setitem__(self, idx, value):
        self._owner._pull(self)
        if idx is None:
            idx = ()
        self.tensor[idx] = torch.as_tensor(value, dtype=self.tensor.dtype, device=self.tensor.device)
        self._owner._touch(self)

    def __len__(self):
        return self.tensor.shape[0]


class ScalarField:
    """0-d host-side scalar with Taichi's ``f[None]`` access (e.g. ``solver.dt[None]``)."""

    def __init__(self, value=0.0, on_change=None):
        self._value = value
        self._on_change = on_change

    def __getitem__(self, idx):
        if idx is not None and idx != ():
            raise IndexError("0-d field: use field[None]")
        return self._value

    def __setitem__(self, idx, value):
        if idx is not None and idx != ():
            raise IndexError("0-d field: use field[None]")
        self._value = value
        if self._on_change is not None:
            self._on_change(value)

    def to_numpy(self):
        return np.asarray(self._value)

    shape = ()


class ScratchField:
    """Read-only per-particle scratch of a solver's last kernels: argument `which` of the engine method `read`
    (``iisph_read``: a_ii, s_i, a^p; ``pcisph_read``: rho*, p, a^p), in the public fields' order."""

    def __init__(self, solver, read, which, width):
        self._solver, self._read, self._which, self._width = solver, read, which, width

    @property
    def shape(self):
        return (self._solver.ps.particle_max_num,)

    def to_numpy(self):
        ps = self._solver.ps
        ps._push()
        n = ps.particle_max_num
        out = torch.zeros((n, 3) if self._width == 3 else (n,), dtype=torch.float32, device=ps.device)
        args = [None, None, None]
        args[self._which] = out
        getattr(ps._engine, self._read)(*args)
        return out.cpu().numpy()
