"""Thin object layer over the C ABI: Context / FFTGrid / KBlock handles holding torch CUDA tensors.

PyTorch is used only for device memory management and (optionally) torch.distributed plumbing; every
kernel on the hot path is launched by libdftk_b200.
"""
import ctypes
import numpy as np
import torch

from . import _lib
from ._lib import check, c_vp, c_i64, c_int


def _ptr(t):
    """Raw pointer of a torch tensor / numpy array / None."""
    if t is None:
        return None
    if isinstance(t, torch.Tensor):
        assert t.is_contiguous()
        return ctypes.c_void_p(t.data_ptr())
    if isinstance(t, np.ndarray):
        assert t.flags["C_CONTIGUOUS"] or t.flags["F_CONTIGUOUS"]
        return t.ctypes.data_as(ctypes.c_void_p)
    raise TypeError(type(t))


class Context:
    """One per GPU / rank (dftk_b200_ctx)."""

    def __init__(self, device=0, nccl_id=None, rank=0, nranks=1):
        self.L = _lib.lib()
        if not torch.cuda.is_available():
            raise RuntimeError("dftk_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        torch.cuda.set_device(device)
        torch.zeros(1, device=f"cuda:{device}")  # make sure the primary context exists
        h = c_vp()
        if nranks > 1:
            buf = (ctypes.c_char * 128).from_buffer_copy(nccl_id)
            check(self.L.dftk_b200_ctx_create_dist(device, buf, rank, nranks, ctypes.byref(h)))
        else:
            check(self.L.dftk_b200_ctx_create(device, ctypes.byref(h)))
        self.h = h
        self.device = torch.device(f"cuda:{device}")
        self.rank, self.nranks = rank, nranks

    @staticmethod
    def nccl_unique_id():
        buf = ctypes.create_string_buffer(128)
        check(_lib.lib().dftk_b200_nccl_unique_id(buf))
        return buf.raw

    def sync(self):
        check(self.L.dftk_b200_sync(self.h), self.h)

    def set_stream(self, stream):
        """Run all work of this context on `stream` (a torch.cuda.Stream, a raw cudaStream_t integer, or None = default)."""
        raw = 0 if stream is None else getattr(stream, "cuda_stream", stream)
        check(self.L.dftk_b200_ctx_set_stream(self.h, ctypes.c_void_p(raw)), self.h)

    def launch_count(self, reset=False):
        return int(self.L.dftk_b200_launch_count(self.h, 1 if reset else 0))

    def lobpcg_flops(self, reset=False):
        """FP64-equivalent GEMM flops executed by the large-path LOBPCG solves since the last reset."""
        return float(self.L.dftk_b200_lobpcg_flops(self.h, 1 if reset else 0))

    def sync_count(self, reset=False):
        """Scheduler rounds (host synchronisations) of the batched LOBPCG solves."""
        return int(self.L.dftk_b200_sync_count(self.h, 1 if reset else 0))

    def set_option(self, name, value):
        check(self.L.dftk_b200_set_option(self.h, name.encode(), int(value)), self.h)

    def mem_info(self):
        f, t = c_i64(), c_i64()
        check(self.L.dftk_b200_mem_info(self.h, ctypes.byref(f), ctypes.byref(t)), self.h)
        return f.value, t.value

    def allreduce(self, t, op="sum"):
        dt = 0 if t.dtype == torch.float64 else 1
        check(self.L.dftk_b200_allreduce(self.h, _ptr(t), t.numel(), dt, {"sum": 0, "min": 1, "max": 2}[op]), self.h)
        return t

    def allgather(self, send, recv):
        dt = 0 if send.dtype == torch.float64 else 1
        check(self.L.dftk_b200_allgather(self.h, _ptr(send), _ptr(recv), send.numel(), dt), self.h)
        return recv

    def real_gram(self, A, B):
        """A B^T for real (n_a, n) / (n_b, n) float64 device tensors with even n (rows = vectors): one fused launch
        (dftk_b200_tall_gram on the complex-pair view; the real part is the real Gram matrix).  Returns a host array."""
        n = A.shape[1]
        assert n % 2 == 0 and B.shape[1] == n and A.is_contiguous() and B.is_contiguous()
        out = np.zeros((B.shape[0], A.shape[0]), dtype=np.complex128)           # column-major n_a x n_b
        check(self.L.dftk_b200_tall_gram(self.h, _ptr(A), n // 2, A.shape[0], _ptr(B), n // 2, B.shape[0], n // 2, _ptr(out)), self.h)
        return np.ascontiguousarray(out.real.T)

    def zgemm(self, transA, A, B, C, alpha=1.0, beta=0.0):
        """C = alpha op(A) B + beta C on column-major data: tensors are (cols, rows) C-contiguous."""
        al = np.array([np.real(alpha), np.imag(alpha)], dtype=np.float64)
        be = np.array([np.real(beta), np.imag(beta)], dtype=np.float64)
        if transA == "C":
            k, m = A.shape[1], A.shape[0]
            n = B.shape[0]
            check(self.L.dftk_b200_zgemm(self.h, 2, m, n, k, _ptr(al), _ptr(A), k, _ptr(B), k, _ptr(be), _ptr(C), m), self.h)
        else:
            m, k = A.shape[1], A.shape[0]
            n = B.shape[0]
            check(self.L.dftk_b200_zgemm(self.h, 0, m, n, k, _ptr(al), _ptr(A), m, _ptr(B), k, _ptr(be), _ptr(C), m), self.h)
        return C

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.L.dftk_b200_ctx_destroy(self.h)
                self.h = None
        except Exception:
            pass


def lobpcg_multi(kblocks, Xs, tol=1e-6, miniter=1, maxiter=100, n_conv_check=None, prec=True):
    """dftk_b200_lobpcg_multi: all (k, spin) blocks of a rank in one call.  Xs[i]: (n_bands, n_pw_i) device tensors,
    updated in place.  Returns one result dict per block (the fields of `KBlock.lobpcg`)."""
    n = len(kblocks)
    if n == 0:
        return []
    ctx = kblocks[0].ctx
    nb = Xs[0].shape[0]
    assert all(x.shape[0] == nb and x.is_contiguous() for x in Xs)
    kb_arr = (c_vp * n)(*[kb.h.value for kb in kblocks])
    x_arr = (c_vp * n)(*[x.data_ptr() for x in Xs])
    lam, res = np.zeros((n, nb)), np.zeros((n, nb))
    nit, conv, nmv = np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int64)
    check(ctx.L.dftk_b200_lobpcg_multi(n, kb_arr, x_arr, nb, float(tol), int(miniter), int(maxiter),
                                       nb if n_conv_check is None else int(n_conv_check), int(prec), _ptr(lam), _ptr(res),
                                       _ptr(nit), _ptr(nmv), _ptr(conv)), ctx.h)
    return [dict(λ=lam[i].copy(), X=Xs[i], residual_norms=res[i].copy(), n_iter=int(nit[i]), n_matvec=int(nmv[i]),
                 converged=bool(conv[i])) for i in range(n)]


def band_energies_multi(kblocks, psis):
    """dftk_b200_band_energies_multi: per-band <psi|kin|psi> and <psi|P D P'|psi> of all k-blocks in one call.
    Returns two lists of host arrays."""
    n = len(kblocks)
    if n == 0:
        return [], []
    ctx = kblocks[0].ctx
    nbs = np.array([p.shape[0] for p in psis], dtype=np.int32)
    ld = int(nbs.max())
    if ld > 32 or any(kb.n_proj > 96 for kb in kblocks):
        pairs = [kb.band_energies(p) for kb, p in zip(kblocks, psis)]
        return [a for a, _ in pairs], [b for _, b in pairs]
    kb_arr = (c_vp * n)(*[kb.h.value for kb in kblocks])
    x_arr = (c_vp * n)(*[p.data_ptr() for p in psis])
    ek, en = np.zeros((n, ld)), np.zeros((n, ld))
    check(ctx.L.dftk_b200_band_energies_multi(n, kb_arr, x_arr, _ptr(nbs), ld, _ptr(ek), _ptr(en)), ctx.h)
    return [ek[i, :nbs[i]].copy() for i in range(n)], [en[i, :nbs[i]].copy() for i in range(n)]


def density_accumulate_multi(kblocks, psis, weights, rho):
    """dftk_b200_density_accumulate_multi: rho (n_spin, N) += Σ_blocks Σ_n w_n |IFFT psi_n|² / Ω, each block into the channel
    of its spin.  psis[i]: (nb_i, n_pw_i) contiguous device tensors, weights[i]: nb_i host numbers."""
    n = len(kblocks)
    if n == 0:
        return rho
    ctx = kblocks[0].ctx
    nbs = np.array([len(w) for w in weights], dtype=np.int32)
    ld = max(1, int(nbs.max()))
    w = np.zeros((n, ld))
    for i, wi in enumerate(weights):
        w[i, :len(wi)] = wi
    kb_arr = (c_vp * n)(*[kb.h.value for kb in kblocks])
    x_arr = (c_vp * n)(*[p.data_ptr() for p in psis])
    check(ctx.L.dftk_b200_density_accumulate_multi(n, kb_arr, x_arr, _ptr(w), ld, _ptr(nbs), _ptr(rho)), ctx.h)
    return rho


def ldos_accumulate_multi(kblocks, psis, W, ldos):
    """dftk_b200_ldos_accumulate_multi: ldos (n_ε, n_spin, N) += Σ_blocks Σ_n W[j, i, n] |IFFT psi_n|² / Ω, each block into the
    channel of its spin.  psis[i]: (nb_i, n_pw_i) contiguous device tensors, W: (n_ε, n_blocks, ld_w) float64 device tensor;
    a band whose weight is zero at every energy is skipped."""
    n = len(kblocks)
    if n == 0:
        return ldos
    ctx = kblocks[0].ctx
    assert W.is_contiguous() and ldos.is_contiguous() and W.shape[:2] == (ldos.shape[0], n)
    nbs = np.array([p.shape[0] for p in psis], dtype=np.int32)
    kb_arr = (c_vp * n)(*[kb.h.value for kb in kblocks])
    x_arr = (c_vp * n)(*[p.data_ptr() for p in psis])
    check(ctx.L.dftk_b200_ldos_accumulate_multi(n, kb_arr, x_arr, _ptr(nbs), ldos.shape[0], ldos.shape[1], _ptr(W), W.shape[2],
                                                _ptr(ldos)), ctx.h)
    return ldos


def orbital_occupation_multi(kblocks, psis, weights, n_spin, n_orb):
    """dftk_b200_orbital_occupation_multi: Σ_blocks Σ_n w_n (Φ'ψ_n)(Φ'ψ_n)' per spin channel over the Hubbard orbitals of
    the k-blocks.  psis[i]: (nb_i, n_pw_i) contiguous device tensors, weights[i]: nb_i host numbers.  Returns a
    (n_spin, n_orb, n_orb) complex host array."""
    n = len(kblocks)
    out = torch.zeros((n_spin, n_orb, n_orb), dtype=torch.complex128,
                      device=kblocks[0].ctx.device if n else "cpu")
    if n == 0:
        return out.numpy()
    ctx = kblocks[0].ctx
    nbs = np.array([len(w) for w in weights], dtype=np.int32)
    ld = max(1, int(nbs.max()))
    w = np.zeros((n, ld))
    for i, wi in enumerate(weights):
        w[i, :len(wi)] = wi
    kb_arr = (c_vp * n)(*[kb.h.value for kb in kblocks])
    x_arr = (c_vp * n)(*[p.data_ptr() for p in psis])
    check(ctx.L.dftk_b200_orbital_occupation_multi(n, kb_arr, x_arr, _ptr(w), ld, _ptr(nbs), _ptr(out)), ctx.h)
    return out.cpu().numpy().transpose(0, 2, 1).copy()     # column-major per spin -> n[s, i, j]


def random_orbitals_multi(kblocks, n_bands, seed):
    """dftk_b200_random_orbitals: orthonormal random start vectors (n_bands, n_pw_i) for a list of k-blocks."""
    n = len(kblocks)
    if n == 0:
        return []
    ctx = kblocks[0].ctx
    Xs = [kb._new(n_bands) for kb in kblocks]
    kb_arr = (c_vp * n)(*[kb.h.value for kb in kblocks])
    x_arr = (c_vp * n)(*[x.data_ptr() for x in Xs])
    check(ctx.L.dftk_b200_random_orbitals(n, kb_arr, x_arr, int(n_bands), ctypes.c_uint64(int(seed) & (2 ** 64 - 1))), ctx.h)
    return Xs


def _blocks(kblocks, *lists):
    """ctypes arrays of the k-block handles and of the data pointers of each list of (n_bands, n_pw_i) tensors (None: NULL)."""
    n = len(kblocks)
    out = [(c_vp * n)(*[kb.h.value for kb in kblocks])]
    for ts in lists:
        if ts is None:
            out.append(None)
            continue
        assert all(t.is_contiguous() for t in ts)
        out.append((c_vp * len(ts))(*[t.data_ptr() for t in ts]))
    return out


def apply_h_multi(kblocks, psis, outs, scale=None):
    """dftk_b200_apply_h_multi: outs[i] = scale[i] H_i psis[i] for all blocks (potentials already installed)."""
    if not kblocks:
        return outs
    kb, x, o = _blocks(kblocks, psis, outs)
    sc = None if scale is None else np.ascontiguousarray(scale, dtype=np.float64)
    check(kblocks[0].ctx.L.dftk_b200_apply_h_multi(len(kblocks), kb, x, o, psis[0].shape[0], _ptr(sc)), kblocks[0].ctx.h)
    return outs


def stiefel_project_multi(kblocks, X, G):
    """dftk_b200_stiefel_project_multi: G[i] -= X[i] herm(X[i]' G[i]) in place."""
    if kblocks:
        kb, x, g = _blocks(kblocks, X, G)
        check(kblocks[0].ctx.L.dftk_b200_stiefel_project_multi(len(kblocks), kb, x, g, X[0].shape[0]), kblocks[0].ctx.h)
    return G


def stiefel_retract_multi(kblocks, Y):
    """dftk_b200_stiefel_retract_multi: new tensors Y[i] (Y[i]' Y[i])^{-1/2}."""
    out = [torch.empty_like(y) for y in Y]
    if kblocks:
        kb, y, o = _blocks(kblocks, Y, out)
        check(kblocks[0].ctx.L.dftk_b200_stiefel_retract_multi(len(kblocks), kb, y, o, Y[0].shape[0]), kblocks[0].ctx.h)
    return out


def tpa_multi(kblocks, mean_kin, inv_w, use_tpa, X=None, Q=None, S=None):
    """dftk_b200_tpa_multi: X given -> mean_kin (n_blocks, n_bands device tensor) from X; Q given -> S = P \\ Q."""
    if not kblocks:
        return S
    nb = (X if X is not None else Q)[0].shape[0]
    kb, x, q, s = _blocks(kblocks, X, Q, S)
    w = np.ascontiguousarray(inv_w, dtype=np.float64)
    check(kblocks[0].ctx.L.dftk_b200_tpa_multi(len(kblocks), kb, x, q, s, nb, _ptr(w), int(bool(use_tpa)),
                                               _ptr(mean_kin) if use_tpa else None), kblocks[0].ctx.h)
    return S


def real_dots_multi(kblocks, pairs):
    """dftk_b200_real_dots_multi: [Σ_i Re<A[i], B[i]> for (A, B) in pairs] in one reduction and one synchronisation."""
    n = len(kblocks)
    if n == 0:
        return [0.0] * len(pairs)
    A = [a for p in pairs for a in p[0]]
    B = [b for p in pairs for b in p[1]]
    kb, a, b = _blocks(kblocks, A, B)
    out = np.zeros(len(pairs))
    check(kblocks[0].ctx.L.dftk_b200_real_dots_multi(len(pairs), n, kb, a, b, A[0].shape[0], _ptr(out)), kblocks[0].ctx.h)
    return out.tolist()


def axpy_dot_multi(kblocks, Y, X, c, Z=None):
    """dftk_b200_axpy_dot_multi: Y[i] += c X[i] in place, then Σ_i Re<Z[i], Y[i]> (None when Z is None)."""
    if not kblocks:
        return None if Z is None else 0.0
    kb, y, x, z = _blocks(kblocks, Y, X, Z)
    out = ctypes.c_double(0.0)
    check(kblocks[0].ctx.L.dftk_b200_axpy_dot_multi(len(kblocks), kb, y, x, float(c), z, Y[0].shape[0], ctypes.byref(out)),
          kblocks[0].ctx.h)
    return None if Z is None else out.value


class FFTGrid:
    """dftk_b200_grid (FFTGrid of src/fft.jl:57-98)."""

    def __init__(self, ctx, fft_size, unit_cell_volume):
        self.ctx = ctx
        self.fft_size = tuple(int(n) for n in fft_size)
        self.N = int(np.prod(self.fft_size))
        h = c_vp()
        check(ctx.L.dftk_b200_grid_create(ctx.h, *self.fft_size, float(unit_cell_volume), ctypes.byref(h)), ctx.h)
        self.h = h

    def set_potential(self, spin, V):
        """One pre-scaled copy of the total local potential per spin channel, shared by the k-blocks that opt in
        (KBlock.use_grid_potential).  Re-installing the tensor the grid already holds is free."""
        ref = getattr(self, "_pot_ref", None)
        if ref is None:
            ref = self._pot_ref = {}
        cur = ref.get(spin)
        if cur is not None and cur[0] is V and cur[1] == V._version:
            return
        ref[spin] = (V, V._version)
        check(self.ctx.L.dftk_b200_grid_set_potential(self.h, int(spin), _ptr(V)), self.ctx.h)

    def fft_cube(self, data, direction):
        """In-place unnormalised transform of (batch, N) complex data; -1 forward, +1 backward."""
        batch = data.numel() // self.N
        check(self.ctx.L.dftk_b200_fft_cube(self.h, _ptr(data), direction, batch), self.ctx.h)
        return data

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.ctx.L.dftk_b200_grid_destroy(self.h)
                self.h = None
        except Exception:
            pass


class KBlock:
    """dftk_b200_kblock: one (k-point, spin) Hamiltonian block resident on the device.

    Orbitals are stored as torch tensors of shape (n_bands, n_pw) complex128 (= column-major n_pw×n_bands).
    """

    def __init__(self, grid, mapping, kin=None, P=None, D=None, spin=0, kweight=1.0):
        self.grid, self.ctx = grid, grid.ctx
        self.n_pw = int(len(mapping))
        self.n_proj = 0 if P is None else int(P.shape[0])
        self.spin, self.kweight = spin, kweight
        mapping = np.ascontiguousarray(mapping, dtype=np.int64)
        h = c_vp()
        if D is not None:
            D = np.asfortranarray(D, dtype=np.float64)
        if kin is not None and isinstance(kin, np.ndarray):
            kin = np.ascontiguousarray(kin, dtype=np.float64)
        check(self.ctx.L.dftk_b200_kblock_create(grid.h, self.n_pw, _ptr(mapping), _ptr(kin), self.n_proj,
                                                 _ptr(P), _ptr(D), spin, float(kweight), ctypes.byref(h)),
              self.ctx.h)
        self.h = h

    def set_potential(self, V):
        """Install the total local potential.  Re-installing the very tensor the block already holds (same object,
        not modified in place since) is free: Hamiltonian blocks bind their potential before every device call."""
        if isinstance(V, torch.Tensor):
            if V is getattr(self, "_pot_ref", None) and V._version == self._pot_version:
                return
            self._pot_ref, self._pot_version = V, V._version
        else:
            self._pot_ref = None
        self._grid_pot = None
        check(self.ctx.L.dftk_b200_kblock_set_potential(self.h, _ptr(V)), self.ctx.h)

    def use_grid_potential(self, spin):
        """Use the grid's shared potential of `spin` (FFTGrid.set_potential) instead of a per-block copy."""
        if getattr(self, "_grid_pot", None) != spin:
            check(self.ctx.L.dftk_b200_kblock_use_grid_potential(self.h, int(spin)), self.ctx.h)
            self._grid_pot = spin
            self._pot_ref = None

    def _new(self, nb):
        return torch.empty((nb, self.n_pw), dtype=torch.complex128, device=self.ctx.device)

    def set_orbitals(self, Phi):
        """dftk_b200_kblock_set_orbitals: attach Hubbard orbitals Phi ((n_orb, n_pw) complex, a row per orbital) whose
        operator Φ V Φ' every H apply then carries with the nonlocal term; None removes them.  V starts at zero."""
        self.n_orb = 0 if Phi is None else int(Phi.shape[0])
        self._orb_V = None
        check(self.ctx.L.dftk_b200_kblock_set_orbitals(self.h, self.n_orb, _ptr(Phi)), self.ctx.h)

    def fold_size(self):
        """dftk_b200_kblock_fold_size: |H| of the time-reversal fold the projector products take, 0 for complex products."""
        n = c_i64()
        check(self.ctx.L.dftk_b200_kblock_fold_size(self.h, ctypes.byref(n)), self.ctx.h)
        return n.value

    def set_orbital_coefficients(self, V):
        """dftk_b200_kblock_set_orbital_coefficients: the n_orb × n_orb Hermitian orbital block of D (None = zero).
        Re-installing the array the block already holds is free."""
        if V is getattr(self, "_orb_V", False):
            return
        Vc = None if V is None else np.asfortranarray(V, dtype=np.complex128)
        check(self.ctx.L.dftk_b200_kblock_set_orbital_coefficients(self.h, _ptr(Vc)), self.ctx.h)
        self._orb_V = V

    def apply_h(self, psi, out=None):
        out = self._new(psi.shape[0]) if out is None else out
        check(self.ctx.L.dftk_b200_apply_h(self.h, _ptr(psi), _ptr(out), psi.shape[0]), self.ctx.h)
        return out

    def apply_terms(self, psi, parts, out=None, accumulate=False):
        out = self._new(psi.shape[0]) if out is None else out
        check(self.ctx.L.dftk_b200_apply_terms(self.h, _ptr(psi), _ptr(out), psi.shape[0], parts,
                                               1 if accumulate else 0), self.ctx.h)
        return out

    def sphere_to_real(self, psi, normalize=True):
        nb = psi.shape[0]
        out = torch.empty((nb, self.grid.N), dtype=torch.complex128, device=self.ctx.device)
        check(self.ctx.L.dftk_b200_fft_sphere_to_real(self.h, _ptr(psi), _ptr(out), nb, int(normalize)), self.ctx.h)
        return out

    def real_to_sphere(self, f_real, normalize=True):
        nb = f_real.shape[0]
        out = self._new(nb)
        check(self.ctx.L.dftk_b200_fft_real_to_sphere(self.h, _ptr(f_real), _ptr(out), nb, int(normalize)), self.ctx.h)
        return out

    def band_energies(self, psi):
        nb = psi.shape[0]
        ek, en = np.zeros(nb), np.zeros(nb)
        check(self.ctx.L.dftk_b200_band_energies(self.h, _ptr(psi), nb, _ptr(ek), _ptr(en)), self.ctx.h)
        return ek, en

    def lobpcg(self, X, tol=1e-6, miniter=1, maxiter=100, n_conv_check=None, prec=True):
        nb = X.shape[0]
        lam, res = np.zeros(nb), np.zeros(nb)
        nit, conv, nmv = c_int(), c_int(), c_i64()
        check(self.ctx.L.dftk_b200_lobpcg(self.h, _ptr(X), nb, float(tol), miniter, maxiter,
                                          nb if n_conv_check is None else int(n_conv_check), int(prec),
                                          _ptr(lam), _ptr(res), ctypes.byref(nit), ctypes.byref(nmv),
                                          ctypes.byref(conv)), self.ctx.h)
        return dict(λ=lam, X=X, residual_norms=res, n_iter=nit.value, n_matvec=nmv.value,
                    converged=bool(conv.value))

    def trim(self):
        """dftk_b200_kblock_trim: free the scratch this block has grown (solver workspaces, residue-plane pools, FFT
        intermediates); later calls re-grow what they need."""
        check(self.ctx.L.dftk_b200_kblock_trim(self.h), self.ctx.h)

    def lobpcg_slab(self, X, tol=1e-6, miniter=1, maxiter=100, n_conv_check=None, prec=True):
        """dftk_b200_lobpcg_slab: this k-block solved by ALL ranks of the context together (plane-wave slabs; collective).
        X (n_bands, n_pw) must be identical on every rank; it holds the eigenvectors on every rank afterwards."""
        nb = X.shape[0]
        lam, res = np.zeros(nb), np.zeros(nb)
        nit, conv, nmv, xb = c_int(), c_int(), c_i64(), ctypes.c_double()
        check(self.ctx.L.dftk_b200_lobpcg_slab(self.h, _ptr(X), nb, float(tol), miniter, maxiter,
                                               nb if n_conv_check is None else int(n_conv_check), int(prec),
                                               _ptr(lam), _ptr(res), ctypes.byref(nit), ctypes.byref(nmv),
                                               ctypes.byref(conv), ctypes.byref(xb)), self.ctx.h)
        return dict(λ=lam, X=X, residual_norms=res, n_iter=nit.value, n_matvec=nmv.value,
                    converged=bool(conv.value), exchange_bytes=xb.value)

    def density_accumulate(self, psi, occ_w, rho):
        occ_w = np.ascontiguousarray(occ_w, dtype=np.float64)
        check(self.ctx.L.dftk_b200_density_accumulate(self.h, _ptr(psi), _ptr(occ_w), psi.shape[0], _ptr(rho)),
              self.ctx.h)
        return rho

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.ctx.L.dftk_b200_kblock_destroy(self.h)
                self.h = None
        except Exception:
            pass
