"""Generates tests/golden/golden_ref_r2.npz from the REFERENCE's own code: oracle/_ref/libref_riccati.so is
robotoc's src/riccati/*.cpp + src/core/split_*.cpp compiled unmodified (oracle/Makefile.ref, Eigen / Robot stand-ins
of oracle/shim).  Only runs where a robotoc source tree exists:

    ROBOTOC_REFERENCE=<robotoc source tree> python tests/golden/make_golden_ref.py

Inputs are regenerated from the seeds below by the tests (tests/synth.py); only the reference's outputs are stored:
full Riccati + direction records for the small event schedules (with / without switching-time optimisation) and the iiwa14
recursion, and [P|s|K|k], the STO scalars / policies and the direction records for the BASELINE schedules (trot N=40,
jump STO N=80), each as a fixed, seeded sample of every section of every record (golden_sample.py).
tests/test_golden_ref.py checks the oracle (CPU) and the CUDA path (-m gpu) against this file.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import jump_sto_schedule, small_event_schedule, trot_schedule  # noqa: E402
from robotoc_b200 import ANYMAL  # noqa: E402
from synth import make_kkt, make_unconstr_kkt  # noqa: E402
sys.path.insert(0, HERE)
from golden_sample import groups, layout_bounds, put  # noqa: E402

PATH = os.path.join(HERE, "golden_ref_r2.npz")
FRAC = 0.3  # share of the nonzero entries of every record section that is stored

CASES = {  # name -> (schedule factory, seed, batch, store full records?)
    "small": (lambda: small_event_schedule(False), 201, 1, True),
    "small_sto": (lambda: small_event_schedule(True), 202, 1, True),
    "trot_n40": (lambda: trot_schedule(40), 203, 1, False),
    "jump_sto_n80": (lambda: jump_sto_schedule(80), 204, 1, False),
}
UNCONSTR = dict(nv=7, N=20, dt=0.05, seed=205, batch=2)


def inputs(name, L):
    sched, seed, batch, full = CASES[name]
    td, ev, ctrl = sched()
    kkt, dx0 = make_kkt(ANYMAL, L, ctrl, batch=batch, seed=seed)
    return ctrl, kkt, dx0, full


def trim(L, ric):
    """[P|s|K|k] + {xi, chi, rho, eta, iota} + STOPolicy of every stage."""
    return np.concatenate([ric[..., :L.r_core_size], ric[..., L.r_sc:L.r_sc + 5], ric[..., L.r_dtsdx:L.r_stosc + 2]], axis=-1)


def trim_bounds(L):
    """Sections of a trimmed Riccati record (trim): the [P|s|K|k] fields, the five STO scalars, the STO policy."""
    core = [(o, min(e, L.r_core_size)) for o, e in layout_bounds(L, "r_", L.r_stride) if o < L.r_core_size]
    n_pol = L.r_stosc + 2 - L.r_dtsdx
    return core + [(L.r_core_size, L.r_core_size + 5), (L.r_core_size + 5, L.r_core_size + 5 + n_pol)]


def unconstr_inputs(UL):
    u = UNCONSTR
    return make_unconstr_kkt(u["nv"], UL, u["N"], u["batch"], u["seed"])


if __name__ == "__main__":
    import oracle_lib
    import ref_lib
    from robotoc_b200 import Layout, ULayout
    lib = oracle_lib.load()
    L = Layout(ANYMAL, getter=lib.orc_layout_get)
    out = {}
    for name in CASES:
        ctrl, kkt, dx0, full = inputs(name, L)
        kk, ric, d = ref_lib.riccati_batch(ANYMAL, L, ctrl, kkt, dx0)
        ric = ric if full else trim(L, ric)
        put(out, name + "_ric", ric, groups(ric, layout_bounds(L, "r_", L.r_stride) if full else trim_bounds(L)),
            CASES[name][1], frac=FRAC, k_min=3, k_z=1)
        put(out, name + "_dir", d, groups(d, layout_bounds(L, "d_", L.d_stride)), CASES[name][1] + 1, frac=FRAC, k_min=3, k_z=1)
    UL = ULayout(7, getter=lib.orc_ulayout_get)
    kkt, dx0 = unconstr_inputs(UL)
    kk, ric, d = ref_lib.unconstr_batch(7, UL, UNCONSTR["N"], UNCONSTR["dt"], kkt, dx0)
    put(out, "unconstr_ric", ric, groups(ric, layout_bounds(UL, "r_", UL.r_stride)), UNCONSTR["seed"], frac=FRAC, k_min=3, k_z=1)
    put(out, "unconstr_dir", d, groups(d, layout_bounds(UL, "d_", UL.d_stride)), UNCONSTR["seed"] + 1, frac=FRAC, k_min=3, k_z=1)
    np.savez_compressed(PATH, **out)
    print("wrote", PATH, os.path.getsize(PATH) // 1024, "KiB;", ref_lib.load().ref_version().decode())
