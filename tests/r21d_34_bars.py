"""Bars of the R(2+1)D-34 engine (the IG65M models' network on tests/r21d_34_ref.py's stand_in_state_dict_34) against a
float64 forward of the same network, held by test_r21d_34_gpu.py.  Worst row (clip for a stage, feature row for the
features); (rel-L2, max-abs / max|ref|), as split_engine_bars.R21D_BARS for R(2+1)D-18.

Each bar sits 1.6x .. 2x above the worst value measured on one H100 80GB HBM3 (700 W power limit) over T = 32 (two
clips, two chunks), 8 and 7 (four clips, two chunks) and the controls' rounded-operand runs; the engine is
deterministic, so a rerun gives the same values.  Measured, rel-L2 / max-abs÷max:
  stem 2.1e-6 / 2.5e-6, layer1 8.0e-6 / 8.3e-6, layer2 2.3e-5 / 1.8e-5, layer3 1.01e-4 / 1.03e-4 (T = 32; 5.4e-5 / 6.2e-5
  at T = 8 and 7), layer4 2.3e-4 / 2.8e-4 (T = 32; 1.1e-4 / 9.0e-5 at T = 8 and 7), features 1.5e-4 / 1.8e-4 (T = 32;
  5.3e-5 / 9.9e-5 at T = 8 and 7).
From layer3 on that is about twice R(2+1)D-18's (split_engine_bars.R21D_BARS) and, at T = 32, twice T = 8's.  The
operands account for little of it: the float64 emulation of the split scheme (scripts/precision/emulate_r21d.py
--depth 34) measures 1.3e-7 at the features, so as for R(2+1)D-18 it is the GEMMs' fp32 accumulation (not measured conv
by conv at depth 34).  The controls with a lost lo half (fp16 weights, fp16 input) measure 4.3e-4 / 3.4e-4 rel-L2 at
the stem (107x / 84x its bar) and 1.3e-3 / 6.7e-4 at the features (5x / 2.7x)."""

R21D_34_STAGES = ("stem", "layer1", "layer2", "layer3", "layer4", "features")

R21D_34_BARS = {"stem": (4e-6, 5e-6), "layer1": (1.5e-5, 1.5e-5), "layer2": (4e-5, 3.5e-5), "layer3": (1.8e-4, 1.8e-4),
                "layer4": (4e-4, 4.5e-4), "features": (2.5e-4, 3e-4)}

# fp32-oracle test: per-stage rel-L2 of read_stage against the fp32 oracle's taps (test_r21d_gpu.STAGE_BAR's role);
# the features' bar is the project's 1e-3 / 1e-3 per row.  Measured: stem 2.1e-6, layer1 7.8e-6, layer2 2.2e-5,
# layer3 9.8e-5, layer4 2.3e-4 (T = 32).
STAGE_BAR_FP32 = {"stem": 1e-5, "layer1": 3e-5, "layer2": 1e-4, "layer3": 3e-4, "layer4": 1e-3}
