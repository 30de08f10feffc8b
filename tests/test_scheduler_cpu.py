"""Scheduler mirror vs the reference scheduler's tables (tests/golden/scheduler.pt, made by oracle/pin/make_golden.py)."""
import torch

from pyramid_flow_b200.scheduler import B200FlowMatchScheduler


def test_scheduler_tables_match_reference(golden_dir):
    g = torch.load(golden_dir / "scheduler.pt", weights_only=False)
    s = B200FlowMatchScheduler(shift=1.0, stages=3, stage_range=[0, 1 / 3, 2 / 3, 1], gamma=1 / 3)
    for k in (0, 1, 2):
        assert s.start_sigmas[k] == g["start_sigmas"][k]
        assert s.end_sigmas[k] == g["end_sigmas"][k]
        assert s.ori_start_sigmas[k] == g["ori_start_sigmas"][k]
        assert list(s.timestep_ratios[k]) == list(g["timestep_ratios"][k])
        # the reference's np.linspace over 0-d torch scalars yields float32 here (numpy/torch-version dependent); the
        # mirror computes the same line in float64: equal to float32 resolution
        assert torch.allclose(s.timesteps_per_stage[k].float(), g["timesteps_per_stage"][k].float(), rtol=0, atol=2e-4)
        assert torch.equal(s.sigmas_per_stage[k], g["sigmas_per_stage"][k])
    for n in (10, 20):
        for st in range(3):
            s.set_timesteps(n, st)
            assert torch.allclose(s.timesteps, g[f"timesteps_{n}_{st}"], rtol=0, atol=2e-4)
            # what the DiT actually sees is the bf16-rounded timestep (pipeline P:750): identical
            assert torch.equal(s.timesteps.bfloat16(), g[f"timesteps_{n}_{st}"].bfloat16())
            assert torch.equal(s.sigmas, g[f"sigmas_{n}_{st}"])
    # published stage boundaries start sigmas {1.0, 0.80024, 0.50075}, end {0.667, 0.334, 0}
    assert abs(s.start_sigmas[1] - 0.80024) < 1e-5 and abs(s.start_sigmas[2] - 0.50075) < 1e-5


def test_euler_step_matches_reference(golden_dir):
    g = torch.load(golden_dir / "scheduler.pt", weights_only=False)
    s = B200FlowMatchScheduler()
    s.set_timesteps(10, 1)
    out = s.step(model_output=g["step_v"], timestep=s.timesteps[0], sample=g["step_x"]).prev_sample
    assert torch.equal(out, g["step_out"])
    assert s.step_index == 1
