"""The stage layer (condensing, expansion, step sizes, slack / dual update: SURVEY.md 8a rows a10-a16) pinned against the
reference's own code.  tests/golden/golden_ref_stage_r2.npz holds (a seeded sample of) one full iteration computed by robotoc's sources
(make_golden_ref_stage.py);
  CPU: the oracle reproduces it; it is also compared with the reference code on the BASELINE trot schedule and further seeds
       (a fixed sample of every record: tests/golden/golden_ref_live.npz, make_golden_ref_live.py);
  GPU: the CUDA path reproduces it through the C ABI."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_ref_stage as mg  # noqa: E402
from golden_sample import load, restore  # noqa: E402
import make_golden_ref_live as mgl  # noqa: E402

import oracle_lib  # noqa: E402
from iteration_check import mask_unread_sto, oracle_iteration, reference_view_of_expansion  # noqa: E402
from robotoc_b200.grid import IMPACT, TERMINAL  # noqa: E402

G = load(mg.PATH)


def _golden(got, impact_cones):
    """The stored reference iteration (a seeded sample of every record section), put into copies of the records under test."""
    pre = "ic_" if impact_cones else ""
    return {k: restore(G, pre + k, got[k]) for k in mg.KEYS if k in got}
TOL = 1e-10


def _cmp_records(S, K, ctrl, got, ref, tol, skip_sol=True, impact_cones=False):
    """Every section the reference's code produces, stage by stage (sections it leaves untouched are not compared)."""
    def rel(name, a, b):
        s = float(np.max(np.abs(b)))
        if s == 0.0:
            assert float(np.max(np.abs(a))) == 0.0, name
            return
        e = float(np.max(np.abs(a - b))) / s
        assert e < tol, f"{name}: {e:.2e}"
    nx, nu, nv = K.nx, K.nu, K.nv
    got, ref = dict(got), dict(ref)
    for dct in (got, ref):  # sections nothing reads on grid points without switching-time optimisation
        dct["kkt"] = mask_unread_sto(K, S, ctrl, kkt=np.array(dct["kkt"]))
        dct["ex_upd"] = mask_unread_sto(K, S, ctrl, ex=np.array(dct["ex_upd"]))
    for i, c in enumerate(ctrl):
        rel(f"Qxx[{i}]", got["kkt"][:, i, K.k_Qxx:K.k_Qxx + nx * nx], ref["kkt"][:, i, K.k_Qxx:K.k_Qxx + nx * nx])
        rel(f"lx[{i}]", got["kkt"][:, i, K.k_lx:K.k_lx + nx], ref["kkt"][:, i, K.k_lx:K.k_lx + nx])
        rel(f"P[{i}]", got["ric"][:, i, K.r_P:K.r_P + nx * nx], ref["ric"][:, i, K.r_P:K.r_P + nx * nx])
        rel(f"dx[{i}]", got["d_upd"][:, i, K.d_dx:K.d_dx + nx], ref["d_upd"][:, i, K.d_dx:K.d_dx + nx])
        rel(f"dlmdgmm[{i}]", got["d_upd"][:, i, K.d_dlmdgmm:K.d_dlmdgmm + nx], ref["d_upd"][:, i, K.d_dlmdgmm:K.d_dlmdgmm + nx])
        if c.type == TERMINAL:
            continue
        nvf = nv + c.nf
        rel(f"kkt[{i}]", got["kkt"][:, i], ref["kkt"][:, i])
        for f, n in (("e_Z", S.nvf * S.nvf), ("e_R", S.nvf * nx), ("e_r", nvf), ("e_Qafqv", S.nvf * nx), ("e_laf", nvf), ("e_Fqqpi", 36)):
            o = getattr(S, f)
            rel(f"{f}[{i}]", got["ex_upd"][:, i, o:o + n], ref["ex_upd"][:, i, o:o + n])
        rel(f"daf[{i}]", got["xd_exp"][:, i, S.x_daf:S.x_daf + nvf], ref["xd_exp"][:, i, S.x_daf:S.x_daf + nvf])
        rel(f"dbetamu[{i}]", got["xd_upd"][:, i, S.x_dbetamu:S.x_dbetamu + nvf], ref["xd_upd"][:, i, S.x_dbetamu:S.x_dbetamu + nvf])
        if c.type == IMPACT:
            if impact_cones:  # the ImpactFrictionCone rows (the box rows do not exist on an impact stage)
                for key, fields in (("cc_cond", ("c_cmpl", "c_cond")), ("cc_exp", ("c_dslack", "c_ddual")), ("cc_upd", ("c_slack", "c_dual"))):
                    for f in fields:
                        o = getattr(S, f)
                        rel(f"impact {f}[{i}]", got[key][:, i, o + S.nbox:o + S.nc], ref[key][:, i, o + S.nbox:o + S.nc])
            continue
        for f, n in (("e_Qafu", S.nvf * nv), ("e_Qxup", nx * S.np), ("e_Quup", S.np * nu), ("e_lup", S.np), ("e_haf", nvf)):
            o = getattr(S, f)
            rel(f"{f}[{i}]", got["ex_upd"][:, i, o:o + n], ref["ex_upd"][:, i, o:o + n])
        rel(f"dnup[{i}]", got["xd_upd"][:, i, S.x_dnup:S.x_dnup + S.np], ref["xd_upd"][:, i, S.x_dnup:S.x_dnup + S.np])
        rel(f"K[{i}]", got["ric"][:, i, K.r_K:K.r_K + nx * nu], ref["ric"][:, i, K.r_K:K.r_K + nx * nu])
        rel(f"du[{i}]", got["d_upd"][:, i, K.d_du:K.d_du + nu], ref["d_upd"][:, i, K.d_du:K.d_du + nu])
        for key, fields in (("cc_cond", ("c_cmpl", "c_cond")), ("cc_exp", ("c_dslack", "c_ddual")), ("cc_upd", ("c_slack", "c_dual"))):
            for f in fields:
                o = getattr(S, f)
                rel(f"{f}[{i}]", got[key][:, i, o:o + S.nc], ref[key][:, i, o:o + S.nc])
    rel("steps", got["steps"], ref["steps"])


@pytest.mark.parametrize("impact_cones", [False, True])
def test_oracle_reproduces_the_reference_iteration_golden(impact_cones):
    lib = oracle_lib.load()
    table, sd, S, K, ctrl, lin, con, sol, dx0 = mg.problem(lib.orc_stage_layout_get, lib.orc_layout_get, impact_cones)
    got = oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0)
    ref = _golden(got, impact_cones)
    if impact_cones:  # the impact cones must matter: the iteration differs from the one without them
        both, a, b = np.intersect1d(G["ic_ric#i"], G["ric#i"], return_indices=True)
        assert np.max(np.abs(G["ic_ric#v"][a] - G["ric#v"][b])) > 1e-6
    _cmp_records(S, K, ctrl, got, ref, TOL, impact_cones=impact_cones)


def _oracle_perf_stage(lib, sd, S, table, ctrl, lin, con):
    """orc_stage_perf_index per grid point: {cost_barrier, primal_feasibility, dual_feasibility, kkt_error}."""
    import ctypes
    lib.orc_stage_perf_index.argtypes = [ctypes.c_void_p] * 6
    out = np.zeros((lin.shape[0], len(ctrl), 4))
    csd = sd.c()
    for b in range(lin.shape[0]):
        for i, c in enumerate(ctrl):
            st = np.zeros(4)
            lib.orc_stage_perf_index(ctypes.byref(csd), ctypes.byref(table), ctypes.byref(c), oracle_lib.ptr(np.ascontiguousarray(lin[b, i])),
                                     oracle_lib.ptr(np.ascontiguousarray(con[b, i])), oracle_lib.ptr(st))
            out[b, i] = st
    return out


@pytest.mark.parametrize("impact_cones", [False, True])
def test_oracle_performance_index_equals_the_reference_evalKKT_summary(impact_cones):
    """PerformanceIndex of every grid point (log barrier, primal / dual feasibility, squared KKT error) as the reference's own
    members compute it before condensing (OCPData / SplitKKTResidual / ConstraintsData / ContactDynamicsData ::KKTError etc.,
    intermediate_stage.cpp:124-132, impact_stage.cpp:104-113, terminal_stage.cpp:94-100) -- golden fixtures."""
    lib = oracle_lib.load()
    table, sd, S, K, ctrl, lin, con, sol, dx0 = mg.problem(lib.orc_stage_layout_get, lib.orc_layout_get, impact_cones)
    got = _oracle_perf_stage(lib, sd, S, table, ctrl, lin, con)
    ref = G["ic_perf_stage" if impact_cones else "perf_stage"]
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=1e-300)
    assert (ref[:, :, 3] > 0).all() and (ref[:, :-1, 0] != 0).any()
    table, ctrl, lin, con, dx0 = mgl.perf_case(sd, S, impact_cones)
    np.testing.assert_allclose(_oracle_perf_stage(lib, sd, S, table, ctrl, lin, con), load(mgl.PATH)[f"perf_icone{int(impact_cones)}"],
                               rtol=1e-12, atol=1e-300)


@pytest.mark.parametrize("which,seed", mgl.STAGE_CASES)
def test_oracle_equals_live_reference_stage_layer(which, seed):
    lib = oracle_lib.load()
    table, sd, S, K, ctrl, lin, con, sol, dx0, icone = mgl.stage_case(which, seed, lib.orc_stage_layout_get, lib.orc_layout_get)
    got = oracle_iteration(sd, S, K, table, ctrl, lin, con, sol, dx0)
    GL = load(mgl.fixture_path(which))
    ref = {k: restore(GL, f"stage_{which}_{k}", got[k]) for k in mgl.STAGE_KEYS}
    _cmp_records(S, K, ctrl, got, ref, TOL, impact_cones=icone)


@pytest.mark.gpu
@pytest.mark.parametrize("impact_cones", [False, True])
def test_cuda_reproduces_the_reference_iteration_golden(impact_cones):
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, RiccatiRecursion
    table, sd, S, K, ctrl, lin, con, sol, dx0 = mg.problem(impact_cones=impact_cones)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), lin.shape[0])
    rr.setTimeDiscretization(ctrl)
    dms = DirectMultipleShooting(rr, sd, table)
    # PerformanceIndex of evalKKT: {cost (not on this path), barrier, primal / dual feasibility, KKT error, sqrt} vs the reference's sums
    perf = dms.evalKKT(lin, con)
    pref = (G["ic_perf_stage"] if impact_cones else G["perf_stage"]).sum(axis=1)
    np.testing.assert_allclose(perf[:, 1:5], pref, rtol=1e-11)
    np.testing.assert_allclose(perf[:, 5], np.sqrt(pref[:, 3]), rtol=1e-11)
    got = _cuda_iteration(rr, dms, S, lin, con, sol, dx0)
    _cmp_records(S, K, ctrl, got, _golden(got, impact_cones), 1e-8, impact_cones=impact_cones)
    rr.close()


def _cuda_iteration(rr, dms, S, lin, con, sol, dx0):
    """One iteration through the C ABI, every record the reference iteration stores."""
    dms.condense(lin, con)
    got = dict(kkt=dms.getKKT(), cc_cond=dms.getConstraintData())
    rr.backwardRiccatiRecursion()
    rr.forwardRiccatiRecursion(dx0)
    assert int(rr.info().max()) == 0
    got["ric"] = rr.getRiccatiFactorization()
    dms.computeStepSizes()
    got["steps"] = np.stack([dms.maxPrimalStepSize(), dms.maxDualStepSize()], axis=1)
    got["cc_exp"], got["xd_exp"] = dms.getConstraintData(), dms.getExpandedDirection()
    dms.integrateSolution(sol)
    got["d_upd"], got["xd_upd"], got["cc_upd"], got["ex_upd"] = (rr.getDirection(), dms.getExpandedDirection(), dms.getConstraintData(),
                                                                 reference_view_of_expansion(S, dms.getExpansionData()))
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("which,seed", [(w, s) for w, s in mgl.STAGE_CASES if w in mgl.GAIT_CASES])
def test_cuda_reproduces_the_reference_iteration_gaits(which, seed):
    """The CUDA iteration against the reference's own on the crawl (with / without switching-time optimisation and impact
    cones) and contact-mask-walk schedules (golden_ref_gaits.npz)."""
    from robotoc_b200 import ANYMAL, DirectMultipleShooting, RiccatiRecursion
    table, sd, S, K, ctrl, lin, con, sol, dx0, icone = mgl.stage_case(which, seed, None, None)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), lin.shape[0])
    rr.setTimeDiscretization(ctrl)
    got = _cuda_iteration(rr, DirectMultipleShooting(rr, sd, table), S, lin, con, sol, dx0)
    GL = load(mgl.GAITS_PATH)
    _cmp_records(S, K, ctrl, got, {k: restore(GL, f"stage_{which}_{k}", got[k]) for k in mgl.STAGE_KEYS if k in got},
                 1e-8, impact_cones=icone)
    rr.close()
