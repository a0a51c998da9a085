"""The reference's own outputs (tests/golden/golden_ref_r2.npz, a seeded sample of every record section, made by tests/golden/make_golden_ref.py from robotoc's
src/riccati compiled unmodified) as the pin:
  CPU:  the oracle (oracle/riccati_oracle.c) reproduces them -- this is what makes the oracle a trustworthy checker;
  CPU:  the oracle equals the reference code on further seeds, every field of every record, on a fixed sample of entries
        (tests/golden/golden_ref_live.npz, made by tests/golden/make_golden_ref_live.py);
  GPU:  the CUDA path reproduces them through the C ABI."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_ref as mg  # noqa: E402
from golden_sample import load, restore  # noqa: E402
import make_golden_ref_live as mgl  # noqa: E402

import oracle_lib  # noqa: E402
from robotoc_b200 import ANYMAL, Layout, ULayout  # noqa: E402

G = load(mg.PATH)
TOL = 1e-10  # relative to the array's scale; measured agreement oracle <-> reference code: 1e-15 .. 3e-15


def _rel(a, b):
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


@pytest.mark.parametrize("name", list(mg.CASES))
def test_oracle_reproduces_reference_golden(name):
    lib = oracle_lib.load()
    L = Layout(ANYMAL, getter=lib.orc_layout_get)
    ctrl, kkt, dx0, full = mg.inputs(name, L)
    kk, ric, d, info = oracle_lib.riccati_batch(ANYMAL, L, ctrl, kkt, dx0)
    assert info == 0
    got = ric if full else mg.trim(L, ric)
    assert _rel(got, restore(G, name + "_ric", got)) < TOL
    assert _rel(d, restore(G, name + "_dir", d)) < TOL


def test_oracle_reproduces_reference_golden_unconstr():
    lib = oracle_lib.load()
    UL = ULayout(7, getter=lib.orc_ulayout_get)
    kkt, dx0 = mg.unconstr_inputs(UL)
    u = mg.UNCONSTR
    kk, ric, d, info = oracle_lib.unconstr_batch(7, UL, u["N"], u["dt"], kkt, dx0)
    assert info == 0
    assert _rel(ric, restore(G, "unconstr_ric", ric)) < TOL and _rel(d, restore(G, "unconstr_dir", d)) < TOL


GL = load(mgl.PATH)


@pytest.mark.parametrize("name,seed", mgl.RICCATI_CASES)
def test_oracle_equals_live_reference_every_field(name, seed):
    """Every field of every Riccati / direction record and the mutated KKT blocks (F, H, G, lu'), batch 3, fresh seeds."""
    from synth import make_kkt
    lib = oracle_lib.load()
    L = Layout(ANYMAL, getter=lib.orc_layout_get)
    td, ev, ctrl = mg.CASES[name][0]()
    kkt, dx0 = make_kkt(ANYMAL, L, ctrl, batch=3, seed=seed)
    kk_o, ric_o, d_o, info = oracle_lib.riccati_batch(ANYMAL, L, ctrl, kkt, dx0)
    assert info == 0
    kk_r, ric_r, d_r = (restore(GL, f"ric_{name}_{k}", a) for k, a in (("kkt", kk_o), ("ric", ric_o), ("dir", d_o)))
    fields = sorted((getattr(L, f), f) for f in mgl.RIC_FIELDS)
    ends = [o for o, _ in fields[1:]] + [L.r_stosc + 2]
    for (o, f), e in zip(fields, ends):
        a, b = ric_o[..., o:e], ric_r[..., o:e]
        scale = np.max(np.abs(b))
        if scale == 0.0:
            assert np.max(np.abs(a)) == 0.0, f
        elif f == "r_W" and any(c.ns == ANYMAL.nu for c in ctrl):
            # ns == nu: W = -(Ginv - SDG^T DG) phi_u with an analytically zero matrix -> pure cancellation noise in both codes
            assert np.max(np.abs(a - b)) < 1e-9 * np.max(np.abs(ric_r[..., L.r_T:L.r_T + ANYMAL.nu])), f
        else:
            assert np.max(np.abs(a - b)) < TOL * scale, f"{f}: {np.max(np.abs(a - b)) / scale:.2e}"
    assert _rel(d_o, d_r) < TOL
    assert _rel(kk_o, kk_r) < TOL  # in-place mutation semantics: Qxx, Qxu, Quu, lu <- F (- K^T G K), H, G, lu'


def test_oracle_equals_live_reference_unconstr():
    from synth import make_unconstr_kkt
    lib = oracle_lib.load()
    UL = ULayout(7, getter=lib.orc_ulayout_get)
    for N, dt, seed in mgl.UNCONSTR_CASES:
        kkt, dx0 = make_unconstr_kkt(7, UL, N, 3, seed)
        kk_o, ric_o, d_o, info = oracle_lib.unconstr_batch(7, UL, N, dt, kkt, dx0)
        kk_r, ric_r, d_r = (restore(GL, f"unconstr_{N}_{k}", a) for k, a in (("kkt", kk_o), ("ric", ric_o), ("dir", d_o)))
        assert info == 0 and _rel(ric_o, ric_r) < TOL and _rel(d_o, d_r) < TOL and _rel(kk_o, kk_r) < TOL


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(mg.CASES))
def test_cuda_reproduces_reference_golden(name):
    from robotoc_b200 import RiccatiRecursion
    L = Layout(ANYMAL)
    ctrl, kkt, dx0, full = mg.inputs(name, L)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), kkt.shape[0])
    rr.setTimeDiscretization(ctrl)
    rr.backwardRiccatiRecursion(kkt)
    rr.forwardRiccatiRecursion(dx0)
    assert int(rr.info().max()) == 0
    ric, d = rr.getRiccatiFactorization(), rr.getDirection()
    ref_ric = restore(G, name + "_ric", ric if full else mg.trim(L, ric))
    if full:
        # stage-conditional sections the reference leaves at their constructor zeros are zero here too; W at ns == nu is noise
        got = ric
        for i, c in enumerate(ctrl):
            if c.ns == ANYMAL.nu:
                got[:, i, L.r_W:L.r_W + ANYMAL.nu] = ref_ric[:, i, L.r_W:L.r_W + ANYMAL.nu]
        assert _rel(got, ref_ric) < 1e-8
    else:
        assert _rel(mg.trim(L, ric), ref_ric) < 1e-8
    assert _rel(d, restore(G, name + "_dir", d)) < 1e-8
    rr.close()


@pytest.mark.gpu
def test_cuda_reproduces_reference_golden_unconstr():
    from robotoc_b200 import UnconstrRiccatiRecursion
    UL = ULayout(7)
    kkt, dx0 = mg.unconstr_inputs(UL)
    u = mg.UNCONSTR
    ur = UnconstrRiccatiRecursion(7, u["N"], u["dt"], u["batch"])
    ur.backwardRiccatiRecursion(kkt)
    ur.forwardRiccatiRecursion(dx0)
    assert int(ur.info().max()) == 0
    ric, d = ur.getRiccatiFactorization(), ur.getDirection()
    assert _rel(ric, restore(G, "unconstr_ric", ric)) < 1e-8
    assert _rel(d, restore(G, "unconstr_dir", d)) < 1e-8
    ur.close()
