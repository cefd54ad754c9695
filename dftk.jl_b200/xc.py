"""Exchange-correlation energy densities and potentials on the device (the XC dispatch point of
ext/DFTKCUDAExt.jl:17-25): one fused CUDA kernel per evaluation (csrc/xc_core.cuh, dual-number closed forms of
Dirac exchange, VWN5, PW92, Teter-Pade, Perdew-Zunger, PBE, PBEsol, revPBE and RPBE with libxc's constants), called
through dftk_b200_xc_evaluate."""
import torch

from ._lib import check
from .device import _ptr

# libxc symbol -> mask bit of the kernel (XC_* in csrc/xc_core.cuh)
FUNCTIONAL_BITS = {"lda_x": 1, "lda_c_vwn": 2, "lda_c_pw": 4, "gga_x_pbe": 8, "gga_c_pbe": 16, "lda_xc_teter93": 32,
                   "lda_c_pz": 64, "gga_x_pbe_sol": 128, "gga_c_pbe_sol": 256, "gga_x_pbe_r": 512, "gga_x_rpbe": 1024}
GGA_BITS = sum(b for f, b in FUNCTIONAL_BITS.items() if f.startswith("gga"))


def evaluate(ctx, functionals, rho, sigma=None):
    """rho: (n_spin, N) device float64; sigma: (1|3, N) or None.  Returns e (N,), Vrho (n_spin, N), Vsigma or None
    -- the quantities libxc returns as zk*rho, vrho, vsigma (src/terms/xc.jl:104-113)."""
    mask = 0
    for f in functionals:
        if f not in FUNCTIONAL_BITS:
            raise NotImplementedError(f"functional {f}")
        mask |= FUNCTIONAL_BITS[f]
    n_spin, N = rho.shape
    is_gga = bool(mask & GGA_BITS)
    if is_gga and sigma is None:
        raise ValueError("GGA functionals need the contracted gradient sigma")
    rho = rho.contiguous()
    e = torch.empty(N, dtype=torch.float64, device=rho.device)
    vr = torch.empty_like(rho)
    vs = None
    if is_gga:
        sigma = sigma.contiguous()
        vs = torch.empty_like(sigma)
    check(ctx.L.dftk_b200_xc_evaluate(ctx.h, mask, n_spin, N, _ptr(rho), _ptr(sigma), _ptr(e), _ptr(vr), _ptr(vs)),
          ctx.h)
    return e, vr, vs
