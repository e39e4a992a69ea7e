"""The loop drivers of the engine on the host: how ``SamplerPlan.run_chunked`` (whole loop, noise tape refilled between
chunks) and ``SamplerPlan.run_guided`` (step by step, host callback between denoiser and update) turn one ``sample()`` call
into ``handle.run`` / ``handle.run_range`` calls and noise draws, and what ``_load_resident`` tells the kernels about the tape.

- The chunk schedule as pure host logic, for the noise pattern of a real coefficient table of every sampler family and every
  tape size from one slot to one per draw: the chunks partition the loop, no chunk holds more draws than the tape, draw k
  lands in slot k mod tape_slots, and that is the slot the remapped noise column names for the iteration that reads it, with
  the draw still there when that iteration runs; the draws come in the reference loop's order.
- On the numpy interpreter (tests/emulator.py): one golden case of every family with a tape of one and of three slots gives
  the bits of the all-up-front tape and its golden within the file's interpreter tolerance."""
import types

import pytest
import torch

import cases
import emulator
import loop_cases as lc
from common import tape_of
from test_host_golden import build_agent
from cleandiffuser_b200.diffusion import solvers as S
from cleandiffuser_b200.engine import cabi, runtime
from cleandiffuser_b200.testing import NoiseTape


@pytest.fixture(autouse=True)
def _emulate(monkeypatch):
    emulator.emulate(monkeypatch)      # every operand is bounds-checked against its owner
    monkeypatch.setenv("CDS_BACKEND", "cuda")       # any fallback to the PyTorch loop is a failure here
    monkeypatch.setenv("CDS_MATH", "fp32")
    monkeypatch.delenv("CDS_NOISE_TAPE_MB", raising=False)


def _sample(family, golden, tape_slots=None, monkeypatch=None):
    """x0 and the plan of the family's golden case on the interpreter (tape of ``tape_slots`` slots, None: all draws)"""
    agent, prior, run, draws, want = lc.golden_case(family, golden=golden)
    if tape_slots is not None:
        monkeypatch.setenv("CDS_NOISE_TAPE_MB", lc.tape_mb(tape_slots, prior))
    tape = NoiseTape(draws)
    calls = runtime.STATS["engine_calls"]
    with tape.active():
        x0 = run(prior)
    assert runtime.STATS["engine_calls"] == calls + 1
    assert tape.pos == len(tape.draws)
    (plan,) = agent._engine_plans.values()
    (tab,) = agent._engine_tables.values()
    return x0, plan, tab, want


# ---------------------------------------------------------------------------------------------------------------------------
# the chunk schedule, pure host logic
PATTERNS = {"ddpm": "ddpm", "ddim": None, "sde_dpmsolver": "sde_2m", "consistency": "consistency", "edm_heun": "edm_heun",
            "legacy_ddpm": "legacy", "legacy_edm": "legacy_edm", "rectified_flow": "rf"}


@pytest.fixture(scope="module")
def tables(golden):
    """the coefficient rows of one golden sample() of every family, as the engine cached them"""
    out = {}
    with pytest.MonkeyPatch.context() as mp:
        emulator.emulate(mp)
        mp.setenv("CDS_BACKEND", "cuda")
        mp.setenv("CDS_MATH", "fp32")
        for pattern, family in PATTERNS.items():
            if family is None:                                   # DDIM: the samplers' DDIM case
                agent, inp, kw = build_agent(cases.sampler_cases()["disc_dup_ddim_eps"])
                with NoiseTape(tape_of(golden["samplers"], "disc_dup_ddim_eps")).active():
                    agent.sample(inp["prior"], **kw)
                (tab,) = agent._engine_tables.values()
            else:
                tab = _sample(family, golden)[2]
            out[pattern] = tab.rows.clone()
    return out


class _Recorder:
    """stand-in for a cabi.Plan: every iteration it is asked to run reads the tape slot its (remapped) coefficient row names,
    the way the update and PREP kernels do, and checks that the draw in it is the one the reference loop takes there"""

    def __init__(self, plan, expect, log):
        self.plan, self.expect, self.log = plan, expect, log

    def _iterate(self, it):
        slot = int(self.plan.coef[it, S.R_NOISE]) - 1
        if self.expect[it] is None:
            assert slot < 0, (it, slot)
        else:
            assert 0 <= slot < self.plan.noise.shape[0], (it, slot, self.plan.noise.shape[0])
            assert int(self.plan.noise[slot, 0, 0]) == self.expect[it], \
                f"iteration {it} reads slot {slot} holding draw {int(self.plan.noise[slot, 0, 0])}, not draw {self.expect[it]}"
        self.log.append(("iter", it))

    def run(self, first, count, stream, use_graph=True):
        self.log.append(("run", first, count))
        for it in range(first, first + count):
            self._iterate(it)

    def run_range(self, it, op_first, op_count, stream):
        if op_first + op_count == len(self.plan.program.ops):          # the update is the last operator
            self._iterate(it)

    def launches_per_iter(self):
        return 1


def _host_plan(rows, tape_slots, monkeypatch):
    """a plan with nothing but what the drivers touch, its coefficient rows loaded by the real _load_resident"""
    n_slots = int((rows[:, S.R_NOISE] > 0).sum())
    plan = types.SimpleNamespace(
        x=torch.zeros(1, 1), coef=torch.zeros_like(rows), mask=None, x_min=None, x_max=None, device=torch.device("cpu"),
        noise=torch.full((tape_slots, 1, 1), -1.0) if tape_slots else None, n_iters=rows.shape[0], batch=1, x_shape=(1,),
        n_branches=1, pred=torch.zeros(1), program=types.SimpleNamespace(ops=[cabi.Op(), cabi.Op()]),
        fill_tables=lambda *a, **k: None)
    plan.program.ops[-1].kind = cabi.OP_UPDATE
    runtime._load_resident(None, plan, torch.zeros(1, 1), None, runtime._Table(rows, n_slots, None, None), tape_slots)
    draws = []

    def draw(dst, like):
        slot = (dst.data_ptr() - plan.noise.data_ptr()) // (4 * plan.noise[0].numel())
        draws.append(slot)
        dst.fill_(float(len(draws) - 1))                       # the k-th draw of the call carries k
    monkeypatch.setattr(runtime, "_draw_noise", draw)
    return plan, draws


@pytest.mark.parametrize("pattern", list(PATTERNS))
def test_chunk_schedule(tables, pattern, monkeypatch):
    rows = tables[pattern]
    n = rows.shape[0]
    noise_rows = (rows[:, S.R_NOISE] > 0).tolist()
    n_draws = sum(noise_rows)
    k_of = [sum(noise_rows[:it]) if noise_rows[it] else None for it in range(n)]       # reference loop: draw k at iteration it
    for tape_slots in range(1, n_draws + 1) if n_draws else [0]:
        where = f"{pattern}, tape of {tape_slots} of {n_draws} slots"
        # the whole-loop driver
        plan, draws = _host_plan(rows, tape_slots, monkeypatch)
        log = []
        plan.handle = _Recorder(plan, k_of, log)
        runtime.SamplerPlan.run_chunked(plan, None, None, torch.zeros(1, 1), noise_rows)
        chunks = [(e[1], e[2]) for e in log if e[0] == "run"]
        assert [f for f, _ in chunks] == [0] + [f + c for f, c in chunks[:-1]] and sum(c for _, c in chunks) == n, where
        assert all(c > 0 for _, c in chunks), where
        assert [e[1] for e in log if e[0] == "iter"] == list(range(n)), where
        for f, c in chunks:
            assert sum(noise_rows[f:f + c]) <= tape_slots, (where, f, c)
        assert draws == [k % tape_slots for k in range(n_draws)], (where, draws)
        if 0 < tape_slots < n_draws:
            assert len(chunks) == -(-n_draws // tape_slots), where
        # the step-by-step driver of the guidance callback, on the same remapped rows
        plan, draws = _host_plan(rows, tape_slots, monkeypatch)
        log = []
        plan.handle = _Recorder(plan, k_of, log)
        guided = []
        runtime.SamplerPlan.run_guided(plan, None, None, torch.zeros(1, 1), plan.coef[:, S.R_NOISE].tolist(),
                                       lambda i, x, p: guided.append(i))
        assert guided == list(range(n)) and [e[1] for e in log if e[0] == "iter"] == list(range(n)), where
        assert draws == [k % tape_slots for k in range(n_draws)], (where, draws)


def test_noise_patterns_of_the_tables(tables):
    """the tables above draw where each family's loop draws: DDPM on every step but the last, the legacy DDPM on every step
    before t = 0 (not on the t = 0 step nor on the extra steps of sample_x), the SDE DPM-Solvers on every step, consistency on every re-noise (all evaluations but the first), DDIM, the EDM samplers (Heun correctors included) and
    rectified flow never"""
    draws = {k: (v[:, S.R_NOISE] > 0).tolist() for k, v in tables.items()}
    assert draws["ddpm"] == [True] * (len(draws["ddpm"]) - 1) + [False]
    n = sum(draws["legacy_ddpm"])
    assert n > 1 and draws["legacy_ddpm"] == [True] * n + [False] * (len(draws["legacy_ddpm"]) - n) and not draws["legacy_ddpm"][-1]
    assert all(draws["sde_dpmsolver"])
    assert draws["consistency"] == [False] + [True] * (len(draws["consistency"]) - 1)
    for k in ("ddim", "edm_heun", "legacy_edm", "rectified_flow"):
        assert not any(draws[k]), (k, draws[k])


# ---------------------------------------------------------------------------------------------------------------------------
# every family on the interpreter with a short tape
@pytest.mark.parametrize("slots", [1, 3])
@pytest.mark.parametrize("family", list(lc.GOLDEN))
def test_short_tape_gives_the_bits_of_the_whole_tape(golden, family, slots, monkeypatch):
    x_all, plan_all, tab, want = _sample(family, golden)
    x0, plan, _, _ = _sample(family, golden, slots, monkeypatch)
    if tab.n_slots:
        assert plan.noise.shape[0] == min(slots, tab.n_slots) and plan_all.noise.shape[0] == tab.n_slots
    else:
        assert plan.noise is None
    assert torch.equal(x0, x_all), float((x0 - x_all).abs().max())
    file = lc.GOLDEN[family][0]
    frac = lc.INTERP_TOL[file](x0.numpy(), want)
    assert frac <= 1.0, (family, frac)
