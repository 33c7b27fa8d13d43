"""The loops of one handle, run on the CPU emulation (tests/emu): a call that belongs to another loop either leaves a live loop
exactly as it was or ends it with CPD_ERR_STATE and a message that names the call.

Each row runs a loop's begin and first step on one handle, then one other call, then the rest of the loop.  The loop's results
must be bit-identical to the same loop run alone on a fresh handle, or every loop call after the other call must be refused.
"""
import re

import numpy as np
import pytest

from probreg_b200 import _cabi

M, N, RANK = 100, 90, 16


def _clouds():
    rng = np.random.default_rng(5)
    src = rng.random((M, 3)) * np.array([6.0, 4.0, 3.0])       # about one unit apart: the IMQ inverse stays well conditioned
    c, s = np.cos(0.2), np.sin(0.2)
    rot = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
    tgt = src[rng.permutation(M)[:N]] @ rot.T + 0.3 + 0.02 * rng.standard_normal((N, 3))
    return src, tgt


SRC, TGT = _clouds()
OTHER = SRC[::-1] * 1.01 + 0.05                               # a moved source for the stand-alone E-steps
D2 = ((SRC[:, None] - SRC[None]) ** 2).sum(-1)
GINV = np.linalg.inv(1.0 / np.sqrt(1.0 + D2)).astype(np.float32)
P1T = np.linspace(0.0, 1.0, M)
PXT = TGT[np.arange(M) % N]
X = np.sin(SRC[:, :2] * 1.3)


def _sigma2(h):
    return h.sigma2_init()


# ---- the loops: begin, then the calls that continue them ------------------------------------------------------------------------
def _em_begin(h):
    h.set_state(_cabi.TF_RIGID, True, 0.1, np.eye(3), np.zeros(3), 1.0, _sigma2(h), 0.0)
    h.em_step()


def _nr_begin(h):
    h.nonrigid_begin(2.0, 2.0, _sigma2(h), 0.1)
    h.nonrigid_step()


def _nr_lr_begin(h):
    h.nonrigid_lowrank_begin(2.0, 2.0, _sigma2(h), 0.1, RANK)
    h.nonrigid_step()


def _bc_begin(h):
    h.bcpd_begin(GINV, 2.0, 1e20, 1.0, 0.05)
    h.bcpd_step()


def _bc_lr_begin(h):
    h.bcpd_lowrank_begin(1.0, 2.0, 1e20, 1.0, 0.05, RANK)
    h.bcpd_step()


def _gt_begin(h):
    h.gmmtree_build(1, 1e-3, 1e-3, np.arange(0, M, M // 8)[:8], maxiter=5)


def _nr_rest(lowrank):
    # W and T first: what the loop hands out must not depend on a call placed between its last step and the read
    rest = [("w", lambda h: h.nonrigid_w()), ("moved", lambda h: h.nonrigid_moved()), ("step", lambda h: h.nonrigid_step()),
            ("set_prior", lambda h: h.nonrigid_set_prior(0.5, P1T, PXT)), ("step", lambda h: h.nonrigid_step()),
            ("w", lambda h: h.nonrigid_w()), ("restart", lambda h: h.nonrigid_restart(2.0, 0.5, 0.0)),
            ("step", lambda h: h.nonrigid_step()), ("moved", lambda h: h.nonrigid_moved())]
    if lowrank:
        rest += [("lowrank_get", lambda h: h.nonrigid_lowrank_factors()), ("gram_product", lambda h: h.lowrank_gram_product(X, 1))]
    return rest


def _bc_rest(lowrank):
    rest = [("step", lambda h: h.bcpd_step()), ("get", lambda h: h.bcpd_get(v=True, moved=True, alpha=True, sigma_diag=True)),
            ("step", lambda h: h.bcpd_step())]
    if lowrank:
        rest += [("lowrank_get", lambda h: h.bcpd_lowrank_factors()), ("gram_product", lambda h: h.lowrank_gram_product(X, 1))]
    return rest


LOOPS = {
    "em": (_em_begin, [("step", lambda h: h.em_step()), ("run", lambda h: h.em_run(2, -1.0))]),
    "nonrigid": (_nr_begin, _nr_rest(False)),
    "nonrigid_lowrank": (_nr_lr_begin, _nr_rest(True)),
    "bcpd": (_bc_begin, _bc_rest(False)),
    "bcpd_lowrank": (_bc_lr_begin, _bc_rest(True)),
    "gmmtree": (_gt_begin, [("estep", lambda h: h.gmmtree_estep(np.eye(3), np.full(3, 0.1), 0.01)),
                            ("assign", lambda h: h.gmmtree_assign()), ("nodes", lambda h: h.gmmtree_nodes())]),
}
# what the products of the low-rank factors return depends on whichever set-up ran last, not on the loop
FACTOR_CALLS = {"gram_product"}
# a stopped BCPD loop still hands out its last state (and its factors while they are its own)
READS = {"bcpd": {"get"}, "bcpd_lowrank": {"get", "lowrank_get"}}

# ---- the calls placed inside a loop ------------------------------------------------------------------------------------------------
OTHERS = {
    "set_state": lambda h: h.set_state(_cabi.TF_AFFINE, True, 0.0, np.eye(3), np.zeros(3), 1.0, 0.7, 0.0),
    "em_step": lambda h: (h.set_state(_cabi.TF_RIGID, True, 0.0, np.eye(3), np.zeros(3), 1.0, 0.7, 0.0), h.em_step()),
    "estep": lambda h: h.estep(OTHER, 0.3, 0.1),
    "bcpd_estep": lambda h: h.bcpd_estep(OTHER, 1.1, np.full(M, 1.0 / M), np.ones(M), 0.3, 0.1),
    "mstep": lambda h: h.mstep(_cabi.TF_RIGID, True, *h.estep(OTHER, 0.3, 0.0)),
    "set_source_same_m": lambda h: h.set_source(SRC),
    "set_source_other_m": lambda h: (h.set_source(SRC[:-3]), h.set_source(SRC)),
    "nonrigid_begin": lambda h: h.nonrigid_begin(3.0, 1.0, 0.4, 0.0),
    "nonrigid_lowrank_begin": lambda h: h.nonrigid_lowrank_begin(3.0, 1.0, 0.4, 0.0, RANK + 4),
    "bcpd_begin": lambda h: h.bcpd_begin(GINV, 3.0, 1e20, 0.5, 0.0),
    "bcpd_lowrank_begin": lambda h: h.bcpd_lowrank_begin(2.0, 3.0, 1e20, 0.5, 0.0, RANK + 4),
    "gmmtree_build": lambda h: h.gmmtree_build(1, 1e-3, 1e-3, np.arange(1, M, M // 8)[:8], maxiter=3),
}

ENDED_NR = "{} ended the non-rigid loop of this handle: call cpd_nonrigid_*begin again"
ENDED_EM = "{} ended the rigid/affine EM loop of this handle: call cpd_set_state again"
REPLACED_NR = "cpd_bcpd_lowrank_begin replaced the low-rank factors of this handle: call cpd_nonrigid_*begin again"
REPLACED_BC = "a cpd_nonrigid_*begin replaced the low-rank factors of the BCPD loop: call cpd_bcpd_lowrank_begin again"
NR_NOT_BEGUN = "cpd_nonrigid_begin has not been called"
LOWRANK_NOT_BEGUN = "cpd_nonrigid_lowrank_begin has not been called"
BC_NOT_BEGUN = "cpd_bcpd_begin has not been called since the source was last set"

# (loop, other call) -> the refusal of every later loop call; a pair that is absent leaves the loop as it was.  Pairs in SKIP
# are the loop's own calls, which change it on purpose.
REFUSED = {
    ("em", "nonrigid_begin"): ENDED_EM.format("cpd_nonrigid_begin"),
    ("em", "nonrigid_lowrank_begin"): ENDED_EM.format("cpd_nonrigid_lowrank_begin"),
    ("bcpd", "set_source_same_m"): BC_NOT_BEGUN,
    ("bcpd", "set_source_other_m"): BC_NOT_BEGUN,
    ("bcpd_lowrank", "set_source_same_m"): BC_NOT_BEGUN,
    ("bcpd_lowrank", "set_source_other_m"): BC_NOT_BEGUN,
    ("bcpd_lowrank", "nonrigid_begin"): REPLACED_BC,
    ("bcpd_lowrank", "nonrigid_lowrank_begin"): REPLACED_BC,
}
for _nr in ("nonrigid", "nonrigid_lowrank"):
    REFUSED[(_nr, "set_state")] = ENDED_NR.format("cpd_set_state")
    REFUSED[(_nr, "em_step")] = ENDED_NR.format("cpd_set_state")
    REFUSED[(_nr, "mstep")] = ENDED_NR.format("cpd_mstep")
    REFUSED[(_nr, "set_source_other_m")] = NR_NOT_BEGUN
    REFUSED[(_nr, "bcpd_lowrank_begin")] = REPLACED_NR
SKIP = {("em", "set_state"), ("em", "em_step"), ("em", "mstep"), ("nonrigid", "nonrigid_begin"), ("nonrigid", "nonrigid_lowrank_begin"),
        ("nonrigid_lowrank", "nonrigid_begin"), ("nonrigid_lowrank", "nonrigid_lowrank_begin"), ("bcpd", "bcpd_begin"),
        ("bcpd", "bcpd_lowrank_begin"), ("bcpd_lowrank", "bcpd_begin"), ("bcpd_lowrank", "bcpd_lowrank_begin"),
        ("gmmtree", "gmmtree_build")}
ROWS = [(loop, other) for loop in LOOPS for other in OTHERS if (loop, other) not in SKIP]


def _handle():
    h = _cabi.Handle(3)
    h.set_source(SRC)
    h.set_target(TGT)
    return h


def _run(loop, other=None):
    """[(call, result or CpdError)] of the loop's calls after `other`"""
    begin, rest = LOOPS[loop]
    h = _handle()
    try:
        begin(h)
        if other is not None:
            OTHERS[other](h)
        out = []
        for name, call in rest:
            try:
                out.append((name, call(h)))
            except _cabi.CpdError as e:
                out.append((name, e))
        return out
    finally:
        h.close()


def _flat(x):
    if isinstance(x, (tuple, list)):
        return [y for v in x for y in _flat(v)]
    return [np.asarray(x)]


_alone = {}


@pytest.mark.parametrize("loop,other", ROWS, ids=["%s-%s" % r for r in ROWS])
def test_a_call_inside_a_loop_leaves_it_alone_or_ends_it(emulated, loop, other):
    if loop not in _alone:
        _alone[loop] = _run(loop)
    alone, got = _alone[loop], _run(loop, other)
    refusal = REFUSED.get((loop, other))
    for (name, a), (_, b) in zip(alone, got):
        assert not isinstance(a, Exception), (name, a)
        if refusal is not None and name in READS.get(loop, ()) and not isinstance(b, Exception):
            continue
        if refusal is not None and name not in FACTOR_CALLS:
            assert isinstance(b, _cabi.CpdError), (name, b)
            expect = LOWRANK_NOT_BEGUN if name == "lowrank_get" and refusal == NR_NOT_BEGUN else refusal
            assert re.fullmatch(r"libcpd_b200: %s \(code -3\)" % re.escape(expect), str(b)), (name, str(b))
        elif name not in FACTOR_CALLS or refusal is None:
            assert not isinstance(b, Exception), (name, b)
            for u, v in zip(_flat(a), _flat(b)):
                assert u.shape == v.shape and np.array_equal(u, v), (name, u, v)
