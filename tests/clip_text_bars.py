"""Bars of the CLIP text tower against float64 (tests/test_clip_text_gpu.py, tests/test_extract_clip_zero_shot_gpu.py),
about 2x the worst values an H100 80GB HBM3 measured on the synthetic towers at 512 / 8, 640 / 10 and 768 / 12 with
every GEMM weight a split-fp16 pair (DESIGN.md §4.16)."""
# attention output against float64 from the same fp16 q / k / v: |err| <= ATTENTION_REL |ref| + ATTENTION_ATOL.  The
# fp16 output alone rounds by up to 2^-11 relative; the measured worst is that rounding.
ATTENTION_REL, ATTENTION_ATOL = 6e-4, 1e-5
# the same kernel on hard inputs (tests/test_attention_hard_gpu.py: a key-0 sink at scores in the hundreds, or each
# row's last key dominant) against float64 with the output rounded to fp16 (tests/attention_ref.py), as (worst prompt
# rel-L2, worst prompt max-abs / max): measured 1.6e-5 / 5.2e-4 on an H100 80GB HBM3 (700 W power limit), the
# max-abs part one fp16 ulp of the output
ATTENTION_HARD = (3e-5, 1.1e-3)
# one block on the declared-rounding oracle's input stream: worst row rel-L2 (measured 4.5e-4, block 0)
BLOCK = 1e-3
# normalised text features: worst row ||t - t_oracle||_2 (measured 7.9e-4; the float64 emulation of the same rounding
# against the exact tower predicts 7.3e-4)
FEATURES = 1.6e-3
# zero-shot logits exp(logit_scale) t.i with logit_scale = ln 100: 100 x FEATURES, plus the head's fp32 dot products
LOGITS = 0.2
