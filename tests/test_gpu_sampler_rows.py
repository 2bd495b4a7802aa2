"""The sampler's per-row mode (`vv_sampler_per_row` / `vv_set_row_sampler`): B = 4 rows with their own step counts, CFG scales and solvers
in one program.  Each row's latent must match the same row sampled alone with its own settings through `set_diffusion_steps` and the
oracle sampler; rows on equal settings match the same settings given to every row by `set_diffusion_steps`; changing one row's settings
leaves the others alone and builds no program; a non-finite row does not reach the others; a 1-step row among rows of
max_diffusion_steps steps gives its 1-step result."""
import os

import pytest
import torch

from vibevoice_b200.configuration import preset_config
from vibevoice_b200.schedule import DPMSolverMultistepScheduler
from vibevoice_b200.synth import SynthTokenizer, synth_state_dict

pytestmark = pytest.mark.gpu

ODE, SDE = "dpmsolver++", "sde-dpmsolver++"
MIXED = [(1, 1.0, ODE), (5, 1.3, SDE), (10, 3.0, ODE), (30, 1.3, SDE)]     # (steps, cfg_scale, solver) of rows 0..3
ORACLE_TOL = 2e-4         # test_gpu_parity.py::test_diffusion_sampler_vs_oracle
TIE_TOL = 2e-5            # two runs of the same program: the stream kernel's fp32 atomics are not reproducible (test_gpu_sampler_steps.py)


def rel_l2(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


_MODELS = {}


def model(preset):
    if preset not in _MODELS:
        from vibevoice_b200.modeling import VibeVoiceForConditionalGenerationInference
        for m, _, _ in _MODELS.values():
            m.engine.close()
        _MODELS.clear()
        cfg = preset_config(preset)
        tok = SynthTokenizer(cfg.decoder_config.vocab_size)
        sd = synth_state_dict(cfg, 1234, torch.bfloat16)
        m = VibeVoiceForConditionalGenerationInference(cfg, tok, max_batch=4)
        m.load_state_dict(sd, tok)
        _MODELS[preset] = (m, cfg, sd)
    return _MODELS[preset]


def inputs(cfg, seed):
    g = torch.Generator().manual_seed(seed)
    cond = torch.randn(8, cfg.decoder_config.hidden_size, generator=g)
    noise = torch.randn(4, 64, generator=g)
    step_noise = [torch.randn(64, 64, generator=g) for _ in range(4)]      # row r's step i: step_noise[r][i]
    return cond, noise, step_noise


def scheduler(eng, solver):
    return DPMSolverMultistepScheduler.from_config(eng.scheduler.config, algorithm_type=solver)


def global_row(eng, cond, noise, step_noise, r, steps, cfg_scale, solver):
    """Row r alone with `set_diffusion_steps` (the other rows inactive)."""
    eng.sampler_per_row(0)
    eng.set_scheduler(scheduler(eng, solver))
    eng.set_diffusion_steps(steps)
    with torch.cuda.stream(eng.stream):
        eng.hidden.copy_(cond.to(eng.device))
    eng.upload_frame_inputs(noise[r:r + 1], [r])
    if solver == SDE:
        eng.upload_step_noise(lambda i: step_noise[r][i:i + 1], [r])
    eng.diffusion_sample(cfg_scale)
    eng.sync()
    return eng.latent[r].cpu().clone()


def per_row(eng, cond, noise, step_noise, settings, n_max=None, reset=True):
    """All rows in the per-row mode with settings[r] = (steps, cfg_scale, solver)."""
    if reset:
        eng.sampler_per_row(n_max or max(s for s, _, _ in settings))
    for r, (steps, cs, solver) in enumerate(settings):
        eng.set_row_sampler(r, steps, solver, cs)
        if solver == SDE:
            eng.upload_row_step_noise(r, step_noise[r][:steps])
    with torch.cuda.stream(eng.stream):
        eng.hidden.copy_(cond.to(eng.device))
    eng.upload_frame_inputs(noise, list(range(4)))
    eng.diffusion_sample(123.0)                          # ignored in the per-row mode
    eng.sync()
    return eng.latent.cpu().clone()


def oracle_row(sd, cond, noise, step_noise, r, steps, cfg_scale, solver):
    from oracle import vv_oracle as O
    kw = dict(algorithm_type=solver, step_noise=[step_noise[r][i:i + 1] for i in range(steps)]) if solver == SDE else {}
    return O.sample_speech_tokens(sd, cond[r:r + 1], cond[4 + r:5 + r], cfg_scale, steps, torch.cat([noise[r:r + 1], torch.zeros(1, 64)]),
                                  **kw)[0]


@pytest.mark.parametrize("preset", ["tiny", "1.5b-l2", "7b-l2"])
def test_mixed_rows_match_solo_and_oracle(preset):
    m, cfg, sd = model(preset)
    eng = m.engine
    cond, noise, sn = inputs(cfg, 11)
    solo = [global_row(eng, cond, noise, sn, r, *MIXED[r]) for r in range(4)]
    got = per_row(eng, cond, noise, sn, MIXED)
    eng.sampler_per_row(0)
    for r in range(4):
        want = oracle_row(sd, cond, noise, sn, r, *MIXED[r])
        assert rel_l2(got[r], solo[r]) < ORACLE_TOL, (r, rel_l2(got[r], solo[r]))
        assert rel_l2(got[r], want) < ORACLE_TOL, (r, rel_l2(got[r], want))


def test_equal_settings_match_global_mode():
    m, cfg, sd = model("tiny")
    eng = m.engine
    cond, noise, sn = inputs(cfg, 12)
    eng.sampler_per_row(0)
    eng.set_scheduler(scheduler(eng, ODE))
    eng.set_diffusion_steps(10)
    with torch.cuda.stream(eng.stream):
        eng.hidden.copy_(cond.to(eng.device))
    eng.upload_frame_inputs(noise, list(range(4)))
    eng.diffusion_sample(1.3)
    eng.sync()
    want = eng.latent.cpu().clone()
    got = per_row(eng, cond, noise, sn, [(10, 1.3, ODE)] * 4)
    eng.sampler_per_row(0)
    assert rel_l2(got, want) < 1e-5, rel_l2(got, want)


def test_row_change_is_isolated_and_builds_nothing(capfd):
    m, cfg, sd = model("tiny")
    eng = m.engine
    cond, noise, sn = inputs(cfg, 13)
    base = per_row(eng, cond, noise, sn, MIXED)
    os.environ["VV_VERBOSE"] = "1"                       # a program build prints "[vv] stream program: ..."
    try:
        capfd.readouterr()
        changed = [MIXED[0], MIXED[1], (3, 1.5, SDE), MIXED[3]]
        got = per_row(eng, cond, noise, sn, changed, n_max=30, reset=False)
        err = capfd.readouterr().err
    finally:
        del os.environ["VV_VERBOSE"]
    eng.sampler_per_row(0)
    assert "stream program" not in err, err
    for r in (0, 1, 3):
        assert rel_l2(got[r], base[r]) < TIE_TOL, (r, rel_l2(got[r], base[r]))
    want = oracle_row(sd, cond, noise, sn, 2, 3, 1.5, SDE)
    assert rel_l2(got[2], want) < ORACLE_TOL


def test_nonfinite_row_stays_in_its_row():
    m, cfg, sd = model("tiny")
    eng = m.engine
    cond, noise, sn = inputs(cfg, 14)
    base = per_row(eng, cond, noise, sn, MIXED)
    bad_cond, bad_noise = cond.clone(), noise.clone()
    bad_cond[1], bad_cond[5] = float("nan"), float("nan")         # row 1: positive and negative condition
    bad_noise[2] = 1e4                                             # row 2: huge initial noise
    bad_sn = [s.clone() for s in sn]
    bad_sn[1][:] = float("nan")
    got = per_row(eng, bad_cond, bad_noise, bad_sn, MIXED)
    eng.sampler_per_row(0)
    assert not torch.isfinite(got[1]).all()
    for r in (0, 3):
        assert rel_l2(got[r], base[r]) < TIE_TOL, (r, rel_l2(got[r], base[r]))


def test_one_step_row_among_max_step_rows():
    m, cfg, sd = model("tiny")
    eng = m.engine
    n_max = m._max_steps
    cond, noise, sn = inputs(cfg, 15)
    settings = [(1, 1.3, ODE), (n_max, 1.3, ODE), (n_max, 2.0, SDE), (1, 3.0, SDE)]
    got = per_row(eng, cond, noise, sn, settings)
    eng.sampler_per_row(0)
    for r in (0, 3):
        solo = global_row(eng, cond, noise, sn, r, *settings[r])
        want = oracle_row(sd, cond, noise, sn, r, *settings[r])
        assert rel_l2(got[r], solo) < ORACLE_TOL and rel_l2(got[r], want) < ORACLE_TOL, (r, rel_l2(got[r], solo), rel_l2(got[r], want))
    eng.set_scheduler(scheduler(eng, ODE))


def teardown_module():
    for m, _, _ in _MODELS.values():
        m.engine.close()
    _MODELS.clear()
