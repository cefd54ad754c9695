"""ctypes binding of libdftk_b200.so (the C ABI declared in include/dftk_b200.h).

There is deliberately NO fallback: if the CUDA library is missing or a call fails, an exception is
raised.  Nothing in this package imports the CPU oracle.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdftk_b200.so")

c_i64 = ctypes.c_int64
c_int = ctypes.c_int
c_dbl = ctypes.c_double
c_vp = ctypes.c_void_p
P = ctypes.POINTER

# name -> (restype, argtypes); kept in sync with include/dftk_b200.h (tests/test_cabi.py checks it)
SIGNATURES = {
    "dftk_b200_ctx_create": (c_int, [c_int, P(c_vp)]),
    "dftk_b200_ctx_create_dist": (c_int, [c_int, c_vp, c_int, c_int, P(c_vp)]),
    "dftk_b200_nccl_unique_id": (c_int, [c_vp]),
    "dftk_b200_ctx_destroy": (c_int, [c_vp]),
    "dftk_b200_last_error": (ctypes.c_char_p, [c_vp]),
    "dftk_b200_ctx_set_stream": (c_int, [c_vp, c_vp]),
    "dftk_b200_sync": (c_int, [c_vp]),
    "dftk_b200_mem_info": (c_int, [c_vp, P(c_i64), P(c_i64)]),
    "dftk_b200_launch_count": (c_i64, [c_vp, c_int]),
    "dftk_b200_sync_count": (c_i64, [c_vp, c_int]),
    "dftk_b200_lobpcg_flops": (c_dbl, [c_vp, c_int]),
    "dftk_b200_set_option": (c_int, [c_vp, ctypes.c_char_p, c_i64]),
    "dftk_b200_grid_create": (c_int, [c_vp, c_int, c_int, c_int, c_dbl, P(c_vp)]),
    "dftk_b200_grid_destroy": (c_int, [c_vp]),
    "dftk_b200_fft_cube": (c_int, [c_vp, c_vp, c_int, c_i64]),
    "dftk_b200_kblock_create": (c_int, [c_vp, c_i64, c_vp, c_vp, c_i64, c_vp, c_vp, c_int, c_dbl, P(c_vp)]),
    "dftk_b200_kblock_destroy": (c_int, [c_vp]),
    "dftk_b200_kblock_set_orbitals": (c_int, [c_vp, c_i64, c_vp]),
    "dftk_b200_kblock_set_orbital_coefficients": (c_int, [c_vp, c_vp]),
    "dftk_b200_kblock_fold_size": (c_int, [c_vp, P(c_i64)]),
    "dftk_b200_orbital_occupation_multi": (c_int, [c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "dftk_b200_kblock_set_potential": (c_int, [c_vp, c_vp]),
    "dftk_b200_grid_set_potential": (c_int, [c_vp, c_int, c_vp]),
    "dftk_b200_kblock_use_grid_potential": (c_int, [c_vp, c_int]),
    "dftk_b200_kblock_trim": (c_int, [c_vp]),
    "dftk_b200_fft_sphere_to_real": (c_int, [c_vp, c_vp, c_vp, c_i64, c_int]),
    "dftk_b200_fft_real_to_sphere": (c_int, [c_vp, c_vp, c_vp, c_i64, c_int]),
    "dftk_b200_apply_h": (c_int, [c_vp, c_vp, c_vp, c_i64]),
    "dftk_b200_apply_terms": (c_int, [c_vp, c_vp, c_vp, c_i64, c_int, c_int]),
    "dftk_b200_band_energies": (c_int, [c_vp, c_vp, c_i64, c_vp, c_vp]),
    "dftk_b200_band_energies_multi": (c_int, [c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "dftk_b200_density_accumulate_multi": (c_int, [c_i64, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "dftk_b200_ldos_accumulate_multi": (c_int, [c_i64, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp, c_i64, c_vp]),
    "dftk_b200_lobpcg": (c_int, [c_vp, c_vp, c_i64, c_dbl, c_int, c_int, c_i64, c_int, c_vp, c_vp,
                                 P(c_int), P(c_i64), P(c_int)]),
    "dftk_b200_lobpcg_slab": (c_int, [c_vp, c_vp, c_i64, c_dbl, c_int, c_int, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "dftk_b200_lobpcg_multi": (c_int, [c_i64, c_vp, c_vp, c_i64, c_dbl, c_int, c_int, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "dftk_b200_random_orbitals": (c_int, [c_i64, c_vp, c_vp, c_i64, ctypes.c_uint64]),
    "dftk_b200_density_accumulate": (c_int, [c_vp, c_vp, c_vp, c_i64, c_vp]),
    "dftk_b200_allreduce": (c_int, [c_vp, c_vp, c_i64, c_int, c_int]),
    "dftk_b200_allgather": (c_int, [c_vp, c_vp, c_vp, c_i64, c_int]),
    "dftk_b200_xc_evaluate": (c_int, [c_vp, c_int, c_int, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "dftk_b200_symmetrize_fourier": (c_int, [c_vp, c_vp, c_vp, c_int, c_vp, c_vp]),
    "dftk_b200_local_forces": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp]),
    "dftk_b200_nonlocal_force_rows": (c_int, [c_vp, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "dftk_b200_ewald": (c_int, [c_vp, c_vp, c_int, c_vp, c_vp, c_dbl, c_vp, c_vp, c_vp, c_vp]),
    "dftk_b200_structure_factor": (c_int, [c_vp, c_int, c_vp, c_vp, c_vp]),
    "dftk_b200_build_projectors": (c_int, [c_vp, c_i64, c_vp, c_int, c_vp, c_int, c_vp, c_vp]),
    "dftk_b200_radial_transform": (c_int, [c_vp, c_i64, c_vp, c_int, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "dftk_b200_columnwise_dots": (c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_vp]),
    "dftk_b200_tall_gram": (c_int, [c_vp, c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_i64, c_vp]),
    "dftk_b200_zgemm": (c_int, [c_vp, c_int, c_i64, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp,
                                c_vp, c_i64]),
    "dftk_b200_apply_h_multi": (c_int, [c_i64, c_vp, c_vp, c_vp, c_i64, c_vp]),
    "dftk_b200_stiefel_project_multi": (c_int, [c_i64, c_vp, c_vp, c_vp, c_i64]),
    "dftk_b200_stiefel_retract_multi": (c_int, [c_i64, c_vp, c_vp, c_vp, c_i64]),
    "dftk_b200_tpa_multi": (c_int, [c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_int, c_vp]),
    "dftk_b200_real_dots_multi": (c_int, [c_i64, c_i64, c_vp, c_vp, c_vp, c_i64, c_vp]),
    "dftk_b200_axpy_dot_multi": (c_int, [c_i64, c_vp, c_vp, c_vp, c_dbl, c_vp, c_i64, c_vp]),
    "dftk_b200_remap_tables": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp]),
    "dftk_b200_sphere_remap": (c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "dftk_b200_fourier_block_copy": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_int, c_int, c_int, c_i64]),
    "dftk_b200_bspline2_prefilter": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_i64]),
    "dftk_b200_bspline2_evaluate": (c_int, [c_vp, c_vp, c_int, c_int, c_int, c_vp, c_vp, c_int, c_int, c_int, c_i64, c_int]),
    "dftk_b200_overlap_multi": (c_int, [c_vp, c_i64, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
}

_lib = None


class DftkB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libdftk_b200 error {code}: {msg}")
        self.code = code


def lib():
    """Load the shared library (once).  Raises ImportError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'`."
                " dftk_b200 has no CPU fallback.")
        L = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(code, ctx=None):
    if code != 0:
        msg = lib().dftk_b200_last_error(ctx)
        raise DftkB200Error(code, msg.decode() if msg else "?")
