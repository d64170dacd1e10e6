"""Cost of CLIP's zero-shot --show_pred on one GPU: encoding the 400 default prompts ("a photo of {name}" over the
Kinetics-400 classes) with the text tower at each released geometry (512 / 8, 640 / 10, 768 / 12; synthetic weights),
and the per-frame head (row L2 normalisation + classifier head over 400 prompts) at 1000 frames of 512 / 768.  Times
are CUDA events around back-to-back calls from Python, host work (the EOT scan, the token copy) included.  Prints the
card name and power limit read in the same run.

The prompts are tokenized with $VF_CLIP_BPE if it is set, else with a vocabulary trained on the prompts
(tests/clip_text_vocab.py); the row count L the tower runs on is printed with the times.

    python scripts/clip_text_time.py
"""
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def events_ms(fn, reps):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    from video_features_b200 import clip_tokenizer as ct
    from video_features_b200 import synthetic_weights
    from video_features_b200.class_head import ClassHead
    from video_features_b200.clip_text_engine import ClipTextEngine, l2_normalize_rows
    print(f"card: {card()}", flush=True)
    bpe = os.environ.get("VF_CLIP_BPE")
    if not bpe:
        from clip_text_vocab import standard_vocab
        bpe = standard_vocab(os.path.join(tempfile.mkdtemp(), ct.BPE_NAME))
    tok = ct.SimpleTokenizer(bpe)
    tokens = tok.tokenize(ct.default_prompts())
    L = int(tokens.argmax(1).max()) + 1
    print(f"400 prompts, vocabulary {tok.vocab_size}, L = {L} rows per prompt (of 77)", flush=True)
    for width, embed in ((512, 512), (640, 640), (768, 768)):
        sd = synthetic_weights.clip_text_state_dict(0, width, embed, tok.vocab_size)
        t0 = time.perf_counter()
        eng = ClipTextEngine(sd, 0)
        torch.cuda.synchronize()
        create = time.perf_counter() - t0
        ms = events_ms(lambda: eng.encode(tokens), 50)
        # what the length cut saves: every prompt padded to the full context (EOT moved to row 76)
        full = np.zeros_like(tokens)
        full[:, :76] = np.where(tokens[:, :76] == tok.eot, 0, tokens[:, :76])
        full[:, 76] = tok.eot
        ms77 = events_ms(lambda: eng.encode(full), 20)
        print(f"text {width}/{width // 64}: encode 400 prompts {ms:.3f} ms (at L = 77: {ms77:.3f} ms); "
              f"create (weight upload) {create * 1e3:.0f} ms", flush=True)
        eng.close()
    g = torch.Generator().manual_seed(0)
    for E in (512, 768):
        text = torch.randn(400, E, generator=g)
        head = ClassHead(100 * text / text.norm(dim=1, keepdim=True), torch.zeros(400), 0)
        x = torch.randn(1000, E, generator=g).cuda()
        ms = events_ms(lambda: head.forward(l2_normalize_rows(x), 5), 200)
        print(f"head {E}: 1000 frames x 400 prompts, normalise + head {ms:.3f} ms ({ms * 1e3 / 1000:.2f} us/frame)",
              flush=True)


if __name__ == "__main__":
    main()
