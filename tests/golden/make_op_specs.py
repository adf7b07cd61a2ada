#!/usr/bin/env python
"""Every distinct normalisation, glue and optimiser launch of the real training steps, as pointer-free specs.

One eager step per configuration is dry-run on the CPU (nothing launches) through tests/op_spec.py's
recording(); each `ops._call` launch of a covered op is reduced to a spec, and the first spec of every
launch class (op_spec.launch_class) is kept.  tests/test_op_prod_gpu.py runs each of them on the GPU against
a float64 reference; tests/test_op_specs_cpu.py re-records and compares, so a change to the launch plan
fails on the CPU until the fixture, and with it the GPU suite, holds the new launch.

    python tests/golden/make_op_specs.py        -> tests/golden/op_specs.json.gz
"""
import dataclasses
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import make_gemm_specs  # noqa: E402
import op_spec  # noqa: E402

FIXTURE = os.path.join(HERE, "op_specs.json.gz")

# the GEMM fixture's configurations, plus a step with an EMA target and a two-substep teacher
CONFIGS = dict(make_gemm_specs.CONFIGS)
CONFIGS["SD15_ema"] = ("SD15", {}, dict(ema_decay=0.95, teacher_substeps=2), 8, 64)


def record_trace(name):
    """The whole launch trace (every `_call` record, GEMMs included) of one configuration's eager step."""
    from pcm_b200 import config, weights
    from pcm_b200.step import PCMTrainStep
    cfg_name, over, step_kw, batch, hw = CONFIGS[name]
    cfg = dataclasses.replace(getattr(config, cfg_name), **over)
    sd = weights.synthetic_state_dict(cfg, 0)
    with op_spec.recording() as rec:
        st = PCMTrainStep(cfg, sd, "cpu", batch=batch, height=hw, width=hw, multiphase=4, **step_kw)
        rec.trace.clear()
        st.run_eager()
        return rec.trace


def main():
    specs = {}
    for name in CONFIGS:
        specs[name] = op_spec.distinct_specs(record_trace(name))
        print(f"{name}: {len(specs[name])} launch classes")
    op_spec.trace.dump(specs, FIXTURE)
    print(f"wrote {FIXTURE} ({os.path.getsize(FIXTURE)} bytes)")


if __name__ == "__main__":
    main()
