"""TEST INFRASTRUCTURE ONLY -- generate tests/golden/sa_*.pt by running the UNMODIFIED reference SA-Solver sampler
(`diffusion.SASolverSampler` from the reference checkout that oracle/refshim.py locates and imports) on seeded inputs with
the deterministic toy denoiser of oracle/dpm_oracle.py.  Needs the reference checkout:  python oracle/gen_golden_sa.py

Two things are wrapped, none of the reference's arithmetic is touched:
  * `SASolverSampler.register_buffer` keeps `alphas_cumprod` on the CPU (the reference moves it to CUDA, sa_sampler.py:24-28);
  * `torch.randn_like` records every draw (one at init, one per step: diffusion/model/sa_solver.py:785,850), and
    `SASolver.adams_moulton_update_few_steps` records the first corrected x (x_1).
Each file holds the case, the inputs, all S + 1 draws, the model times, x_1 and the output.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import dpm_oracle as do               # noqa: E402
from oracle.refshim import install_reference_shims  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
CASES = {"sa_s25_eta1": dict(steps=25, eta=1.0, n=2, hw=(8, 8), cfg=4.5),       # scripts/inference.py:119-133's own call
         "sa_s5_eta0": dict(steps=5, eta=0.0, n=1, hw=(8, 8), cfg=4.5),         # deterministic
         "sa_s2": dict(steps=2, eta=1.0, n=1, hw=(8, 8), cfg=4.5),              # the minimum S
         "sa_s7_eta05": dict(steps=7, eta=0.5, n=2, hw=(8, 12), cfg=4.5),       # non-square latents
         "sa_s6_cfg1": dict(steps=6, eta=1.0, n=1, hw=(8, 8), cfg=1.0)}         # unguided: one conditional evaluation


def inputs(case, seed=0):
    g = torch.Generator().manual_seed(seed)
    n, (h, w) = case["n"], case["hw"]
    x_T = torch.randn(n, 4, h, w, generator=g)
    cond = torch.randn(n, 1, 6, 8, generator=g) * 0.5
    uncond = (torch.randn(1, 1, 6, 8, generator=g) * 0.5).repeat(n, 1, 1, 1)
    return x_T, cond, uncond


def main():
    install_reference_shims()
    import tqdm as _tqdm  # noqa: F401  (the reference's loop wraps its range in tqdm)
    import diffusion.model.sa_solver as sa_solver
    from diffusion import SASolverSampler

    def keep_on_cpu(self, name, attr):
        setattr(self, name, attr)
    SASolverSampler.register_buffer = keep_on_cpu

    os.makedirs(OUT, exist_ok=True)
    randn_like = torch.randn_like
    moulton = sa_solver.SASolver.adams_moulton_update_few_steps
    for name, case in CASES.items():
        x_T, cond, uncond = inputs(case)
        draws, times, corrected = [], [], []

        def recording_randn_like(x, *a, **k):
            r = randn_like(x, *a, **k)
            draws.append(r.clone())
            return r

        def recording_moulton(self, *a, **k):
            r = moulton(self, *a, **k)
            corrected.append(r.clone())
            return r

        def spy(x, t, c, **kw):
            times.append(float(t[0]))
            return do.toy_model(x, t, c, **kw)

        torch.manual_seed(1000 + case["steps"])
        torch.randn_like, sa_solver.SASolver.adams_moulton_update_few_steps = recording_randn_like, recording_moulton
        try:
            out, extra = SASolverSampler(spy, device="cpu").sample(
                S=case["steps"], batch_size=case["n"], shape=(4,) + case["hw"], conditioning=cond, eta=case["eta"],
                x_T=x_T.clone(), unconditional_guidance_scale=case["cfg"], unconditional_conditioning=uncond,
                model_kwargs={})
        finally:
            torch.randn_like, sa_solver.SASolver.adams_moulton_update_few_steps = randn_like, moulton
        assert extra is None and len(draws) == case["steps"] + 1 and len(times) == case["steps"]
        torch.save(dict(case=case, x_T=x_T, cond=cond, uncond=uncond, draws=torch.stack(draws), model_times=torch.tensor(times),
                        x_1=corrected[0], out=out), os.path.join(OUT, name + ".pt"))
        print(name, tuple(out.shape), "times", [round(v, 3) for v in times[:3]], "...", "draws", len(draws))


if __name__ == "__main__":
    main()
