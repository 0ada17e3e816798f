"""Host-side mirror of `ark_poly::Radix2EvaluationDomain` (poly/src/domain/radix2/mod.rs:22-153) over the C ABI.

Field elements are (4,) uint64 Montgomery limb arrays, vectors are (n, 4) arrays — numpy on the host path, or
torch CUDA tensors (8-byte dtype) for device-resident data.  The transforms have the reference's semantics:
  fft_in_place / fft  : input shorter than the domain is zero-padded, longer is TRUNCATED (`coeffs.resize`, :144)
  ifft_in_place / ifft: same resize (:151); natural order in and out.
With `curve=` (a B200_CURVE_* id whose scalar field is the domain's field) the coefficients are G1 points instead, the
T = Projective case of the reference's `DomainCoeff` transforms: (len, 3N) uint64 Jacobian Montgomery limbs (x, y, z), padded
with the identity (R, R, 0) or truncated to the domain size; every identity in the output is (R, R, 0)."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib
from .params import CURVES, SCALAR_FIELDS, PrimeField


def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


class Radix2EvaluationDomain:
    def __init__(self, field_id: int, size: int, offset: int = 1):
        # use `new` / `get_coset`
        self.field_id = field_id
        self.F: PrimeField = SCALAR_FIELDS[field_id]
        p = self.F.modulus
        self.size = size
        self.log_size_of_group = size.bit_length() - 1
        # F::get_root_of_unity(size): ff/src/fields/fft_friendly.rs:66-82
        g = self.F.two_adic_root_of_unity
        for _ in range(self.log_size_of_group, self.F.two_adicity):
            g = g * g % p
        self._group_gen = g
        self._group_gen_inv = pow(g, -1, p)
        self._size_inv = pow(size % p, -1, p)
        self._offset = offset % p
        self._offset_inv = pow(self._offset, -1, p)
        self._offset_pow_size = pow(self._offset, size, p)

    # -- constructors (radix2/mod.rs:55-92) -------------------------------------------------------
    @classmethod
    def new(cls, field_id: int, num_coeffs: int):
        size = 1 if num_coeffs <= 1 else 1 << (num_coeffs - 1).bit_length()
        if size.bit_length() - 1 > SCALAR_FIELDS[field_id].two_adicity:
            return None
        return cls(field_id, size)

    @staticmethod
    def compute_size_of_domain(field_id: int, num_coeffs: int):
        size = 1 if num_coeffs <= 1 else 1 << (num_coeffs - 1).bit_length()
        return size if size.bit_length() - 1 <= SCALAR_FIELDS[field_id].two_adicity else None

    def get_coset(self, offset):
        off = self.F.from_limbs(offset) if not isinstance(offset, int) else offset % self.F.modulus
        if off == 0:
            return None  # offset.inverse()? fails
        return Radix2EvaluationDomain(self.field_id, self.size, off)

    # -- getters: Montgomery limbs, like the reference's fields ----------------------------------
    def size_inv(self): return self.F.to_limbs(self._size_inv)
    def group_gen(self): return self.F.to_limbs(self._group_gen)
    def group_gen_inv(self): return self.F.to_limbs(self._group_gen_inv)
    def coset_offset(self): return self.F.to_limbs(self._offset)
    def coset_offset_inv(self): return self.F.to_limbs(self._offset_inv)
    def coset_offset_pow_size(self): return self.F.to_limbs(self._offset_pow_size)
    def size_as_field_element(self): return self.F.to_limbs(self.size)

    def element(self, i: int) -> np.ndarray:
        """offset * g^i  (poly/src/domain/mod.rs:274-280)"""
        return self.F.to_limbs(self._offset * pow(self._group_gen, i, self.F.modulus))

    def elements(self):
        cur, p = self._offset, self.F.modulus
        for _ in range(self.size):
            yield self.F.to_limbs(cur)
            cur = cur * self._group_gen % p

    # -- transforms ---------------------------------------------------------------------------------
    def _offset_ptr(self):
        if self._offset == 1:
            return None, None
        arr = self.F.to_limbs(self._offset)
        return arr, arr.ctypes.data_as(ctypes.c_void_p)

    def _resize(self, x):
        n = self.size
        if _is_torch(x):
            import torch
            x = x.reshape(-1, 4)
            if x.shape[0] == n:
                return x
            out = torch.zeros((n, 4), dtype=x.dtype, device=x.device)
            k = min(n, x.shape[0])
            out[:k] = x[:k]
            return out
        x = np.asarray(x, dtype=np.uint64).reshape(-1, 4)
        if x.shape[0] == n and x.flags["C_CONTIGUOUS"]:
            return x
        out = np.zeros((n, 4), dtype=np.uint64)
        k = min(n, x.shape[0])
        out[:k] = x[:k]
        return out

    @staticmethod
    def _shares(x, orig) -> bool:
        if _is_torch(x):
            return _is_torch(orig) and x.data_ptr() == orig.data_ptr()
        return isinstance(orig, np.ndarray) and np.shares_memory(x, orig)

    def _run(self, x, inverse: bool):
        keep, offp = self._offset_ptr()
        if _is_torch(x):
            import torch
            if not x.is_cuda or not x.is_contiguous():
                raise TypeError("device path needs a contiguous CUDA tensor")
            with torch.cuda.device(x.device):
                st = torch.cuda.current_stream().cuda_stream
                _lib.check(_lib.lib().b200_ntt_fr_dev(self.field_id, x.data_ptr(), self.log_size_of_group, int(inverse), offp, st))
        else:
            assert x.flags["C_CONTIGUOUS"] and x.dtype == np.uint64
            _lib.check(_lib.lib().b200_ntt_fr(self.field_id, x.ctypes.data_as(ctypes.c_void_p), self.log_size_of_group,
                                              int(inverse), offp))
        del keep
        return x

    def _run_padded(self, x, inverse: bool):
        """host input shorter (or longer) than the domain: only the given rows cross PCIe, the resize happens on the device"""
        keep, offp = self._offset_ptr()
        x = np.ascontiguousarray(x, dtype=np.uint64).reshape(-1, 4)
        out = np.empty((self.size, 4), dtype=np.uint64)
        _lib.check(_lib.lib().b200_ntt_fr_padded(self.field_id, x.ctypes.data_as(ctypes.c_void_p), x.shape[0], out.ctypes.data_as(ctypes.c_void_p),
                                                 self.log_size_of_group, int(inverse), offp))
        del keep
        return out

    # -- G1 point coefficients (T = Projective) ----------------------------------------------------
    def _point_width(self, curve: int) -> int:
        if curve not in CURVES or CURVES[curve].ntt_field_id != self.field_id:
            raise ValueError(f"curve {curve} does not have this domain's scalar field ({self.F.name})")
        return 3 * CURVES[curve].N

    def _resize_points(self, x, curve: int):
        w, n = self._point_width(curve), self.size
        zero = np.zeros(w, dtype=np.uint64)   # Projective::zero() = (1, 1, 0) in Montgomery form (group.rs:142-158)
        one = CURVES[curve].fq.to_limbs(1)
        zero[:len(one)] = one
        zero[w // 3:w // 3 + len(one)] = one
        if _is_torch(x):
            import torch
            x = x.reshape(-1, w)
            if x.shape[0] == n:
                return x
            out = torch.from_numpy(np.tile(zero, (n, 1)).view(np.int64)).to(device=x.device, dtype=x.dtype)
            k = min(n, x.shape[0])
            out[:k] = x[:k]
            return out
        x = np.asarray(x, dtype=np.uint64).reshape(-1, w)
        if x.shape[0] == n and x.flags["C_CONTIGUOUS"]:
            return x
        out = np.tile(zero, (n, 1))
        k = min(n, x.shape[0])
        out[:k] = x[:k]
        return out

    def _run_points(self, x, inverse: bool, curve: int):
        keep, offp = self._offset_ptr()
        if _is_torch(x):
            import torch
            if not x.is_cuda or not x.is_contiguous():
                raise TypeError("device path needs a contiguous CUDA tensor")
            with torch.cuda.device(x.device):
                st = torch.cuda.current_stream().cuda_stream
                _lib.check(_lib.lib().b200_ntt_g1_dev(curve, x.data_ptr(), self.log_size_of_group, int(inverse), offp, st))
        else:
            assert x.flags["C_CONTIGUOUS"] and x.dtype == np.uint64
            _lib.check(_lib.lib().b200_ntt_g1(curve, x.ctypes.data_as(ctypes.c_void_p), self.log_size_of_group, int(inverse), offp))
        del keep
        return x

    def _run_points_copy(self, pts, inverse: bool, curve: int):
        x = self._resize_points(pts, curve)
        if self._shares(x, pts):
            x = x.clone() if _is_torch(x) else x.copy()
        return self._run_points(x, inverse, curve)

    def fft(self, coeffs, curve: int | None = None):
        """EvaluationDomain::fft (poly/src/domain/mod.rs:94-98): returns a new vector of `size` evaluations."""
        if curve is not None:
            return self._run_points_copy(coeffs, False, curve)
        if not _is_torch(coeffs):
            return self._run_padded(coeffs, False)
        x = self._resize(coeffs)
        if self._shares(x, coeffs):
            x = x.clone() if _is_torch(x) else x.copy()
        return self._run(x, False)

    def ifft(self, evals, curve: int | None = None):
        if curve is not None:
            return self._run_points_copy(evals, True, curve)
        if not _is_torch(evals):
            return self._run_padded(evals, True)
        x = self._resize(evals)
        if self._shares(x, evals):
            x = x.clone() if _is_torch(x) else x.copy()
        return self._run(x, True)

    def fft_in_place(self, coeffs, curve: int | None = None):
        """Transforms `coeffs` itself when it already has `size` rows (the Vec is resized otherwise, and the new
        vector is returned — Python cannot grow the caller's buffer in place)."""
        if curve is not None:
            return self._run_points(self._resize_points(coeffs, curve), False, curve)
        return self._run(self._resize(coeffs), False)

    def ifft_in_place(self, evals, curve: int | None = None):
        if curve is not None:
            return self._run_points(self._resize_points(evals, curve), True, curve)
        return self._run(self._resize(evals), True)

    def __eq__(self, o):
        return isinstance(o, Radix2EvaluationDomain) and (self.field_id, self.size, self._offset) == (o.field_id, o.size, o._offset)

    def __hash__(self):
        return hash((self.field_id, self.size, self._offset))

    def __repr__(self):
        return f"Radix-2 multiplicative subgroup of size {self.size}"
