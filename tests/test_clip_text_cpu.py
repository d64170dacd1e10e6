"""CLIP zero-shot `--show_pred` without a GPU: the BPE tokenizer against HF ``CLIPTokenizer`` on the same vocabulary,
the text-tower oracle against HF ``CLIPTextModelWithProjection``, and the CLI's flag, refusals and early errors."""
import json
import os

import numpy as np
import pytest
import torch

import main
from clip_text_vocab import standard_vocab, write_hf_files
from oracle import clip_text
from video_features_b200 import clip_tokenizer as ct
from video_features_b200 import synthetic_weights

ODD = ["Hello   World!! it's 2024, they'll   GO... don't #tags $99.5", "A  B\tc\nD  ", "l'ESPRIT 3rd-party (x+y)=z",
       "WE'VE I'M you'd", "!!!???...", "0123456789", "the dog's ball", "  leading and trailing  ", "CamelCase Words"]


@pytest.fixture(scope="module")
def bpe(tmp_path_factory):
    return standard_vocab(str(tmp_path_factory.mktemp("bpe") / ct.BPE_NAME))


@pytest.fixture(scope="module")
def hf_tokenizer(bpe, tmp_path_factory):
    from transformers import CLIPTokenizer
    vocab_file, merges_file = write_hf_files(bpe, str(tmp_path_factory.mktemp("hf")))
    with open(vocab_file, encoding="utf-8") as f:
        vocab = json.load(f)
    with open(merges_file, encoding="utf-8") as f:
        merges = [tuple(ln.split()) for ln in f.read().split("\n")[1:] if ln]
    return CLIPTokenizer(vocab=vocab, merges=merges)


def test_vocabulary_layout(bpe):
    tok = ct.SimpleTokenizer(bpe)
    enc = list(ct.bytes_to_unicode().values())
    assert len(set(enc)) == 256
    assert [tok.encoder[c] for c in enc] == list(range(256))
    assert [tok.encoder[c + "</w>"] for c in enc] == list(range(256, 512))
    assert tok.sot == tok.vocab_size - 2 and tok.eot == tok.vocab_size - 1
    assert tok.vocab_size == 512 + len(tok.bpe_ranks) + 2 and len(tok.bpe_ranks) == 400


@pytest.mark.parametrize("which", ["prompts", "odd"])
def test_ids_equal_hf(bpe, hf_tokenizer, which):
    tok = ct.SimpleTokenizer(bpe)
    texts = ct.default_prompts() if which == "prompts" else ODD
    assert len(texts) == (400 if which == "prompts" else len(ODD))
    for t in texts:
        assert [tok.sot] + tok.encode(t) + [tok.eot] == hf_tokenizer(t)["input_ids"], t


def test_html_is_unescaped_twice(bpe):
    tok = ct.SimpleTokenizer(bpe)
    assert tok.encode("rock &amp; roll") == tok.encode("rock & roll")
    assert tok.encode("rock &amp;amp; roll") == tok.encode("rock & roll")
    assert tok.encode("&lt;b&gt;") == tok.encode("<b>")


def test_tokenize_pads_and_refuses_long_prompts(bpe):
    tok = ct.SimpleTokenizer(bpe)
    rows = tok.tokenize(["a photo of dancing", "x"])
    assert rows.shape == (2, 77) and rows.dtype == np.int32
    n = len(tok.encode("a photo of dancing")) + 2
    assert rows[0, 0] == tok.sot and rows[0, n - 1] == tok.eot and not rows[0, n:].any()
    assert list(rows[1, :3]) == [tok.sot, tok.encode("x")[0], tok.eot]
    assert tok.tokenize(["7 " * 75]).shape == (1, 77)                 # 75 digits + SOT + EOT fit exactly
    with pytest.raises(RuntimeError, match="too long for context length 77"):
        tok.tokenize(["7 " * 76])


def test_bpe_lookup_order(tmp_path, monkeypatch, bpe):
    monkeypatch.setenv("VF_CLIP_BPE", bpe)
    assert ct.find_bpe() == bpe
    monkeypatch.setenv("VF_CLIP_BPE", str(tmp_path / "nope.txt.gz"))
    monkeypatch.setenv("HOME", str(tmp_path))
    cands = ct.bpe_candidates()
    assert cands[0] == str(tmp_path / "nope.txt.gz")
    assert cands[1].endswith(os.path.join("extract", "checkpoints", ct.BPE_NAME))
    assert cands[2] == os.path.join(str(tmp_path), ".cache", "clip", ct.BPE_NAME)


# ---------------------------------------------------------------- oracle against HF


@pytest.mark.parametrize("width,embed", [(512, 1024), (768, 768)])
def test_oracle_equals_hf_text_model(bpe, width, embed):
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    tok = ct.SimpleTokenizer(bpe)
    sd = synthetic_weights.clip_text_state_dict(3, width, embed, tok.vocab_size)
    cfg = clip_text.config(sd)
    assert (cfg["width"], cfg["heads"], cfg["layers"], cfg["context"], cfg["embed"]) == (width, width // 64, 12, 77, embed)
    hf_cfg = CLIPTextConfig(vocab_size=tok.vocab_size, hidden_size=width, intermediate_size=4 * width,
                            projection_dim=embed, num_hidden_layers=12, num_attention_heads=width // 64,
                            max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5,
                            eos_token_id=2, attn_implementation="eager")
    model = CLIPTextModelWithProjection(hf_cfg).eval()
    missing, unexpected = model.load_state_dict(clip_text.to_hf_state_dict(sd), strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    tokens = tok.tokenize(ct.default_prompts()[:24] + ODD[:4])
    ours = clip_text.encode_text(sd, tokens)
    with torch.no_grad():
        ref = model(input_ids=torch.from_numpy(tokens).long()).text_embeds
    rel = ((ours - ref).norm(dim=1) / ref.norm(dim=1)).max().item()
    assert rel < 1e-5, rel
    # the pooled row is the argmax id's, and the declared-rounding float64 tower agrees to fp16 accuracy
    assert (clip_text.eot_positions(tokens) == torch.from_numpy((tokens == tok.eot).argmax(1))).all()
    d = clip_text.encode_text_declared(sd, tokens, rounding=clip_text.Rounding(act=False))
    ref64 = ours.double() / ours.double().norm(dim=1, keepdim=True)
    assert (d - ref64).abs().max().item() < 1e-5


def test_length_cut_is_exact(bpe):
    """Rows after the last EOT never reach an EOT row: the float64 tower on L rows equals it on all 77."""
    tok = ct.SimpleTokenizer(bpe)
    sd = synthetic_weights.clip_text_state_dict(1, 512, 512, tok.vocab_size)
    tokens = tok.tokenize(ct.default_prompts()[:6])
    cut = clip_text.encode_text_declared(sd, tokens, rounding=clip_text.Rounding(act=False))
    full = clip_text.encode_text(sd, tokens, dtype=torch.float64)
    full = full / full.norm(dim=1, keepdim=True)
    assert (cut - full).abs().max().item() < 1e-12


# ---------------------------------------------------------------- CLI


def _args(tmp_path, ft, *extra):
    a = str(tmp_path / "a.mp4")
    open(a, "wb").close()
    return main.make_parser().parse_args(["--feature_type", ft, "--video_paths", a,
                                          "--output_path", str(tmp_path / "out"), "--device_ids", "0", *extra])


def test_pred_texts_parse(tmp_path):
    args = _args(tmp_path, "CLIP-ViT-B/32", "--show_pred", "--pred_texts", "a dog", "a cat playing", "snow")
    assert args.pred_texts == ["a dog", "a cat playing", "snow"]
    main.sanity_check(args)
    assert _args(tmp_path, "CLIP-ViT-B/32").pred_texts is None
    helps = {a.dest: a.help for a in main.make_parser()._actions}
    assert "CLIP" in helps["show_pred"] and "pred_texts" in helps["show_pred"]


def test_pred_texts_needs_show_pred(tmp_path):
    with pytest.raises(AssertionError, match="only takes effect with --show_pred"):
        main.sanity_check(_args(tmp_path, "CLIP-ViT-B/32", "--pred_texts", "a dog"))


@pytest.mark.parametrize("ft", ["resnet50", "i3d", "s3d"])
def test_pred_texts_refused_outside_clip(tmp_path, ft):
    with pytest.raises(AssertionError, match="do not apply to " + ft):
        main.sanity_check(_args(tmp_path, ft, "--show_pred", "--pred_texts", "a dog"))


def _no_video_opened(monkeypatch):
    from video_features_b200.extract import extract_clip

    def boom(*a, **k):
        raise AssertionError("a video was opened")
    monkeypatch.setattr(extract_clip, "extract_frames", boom)
    monkeypatch.setattr(extract_clip, "FrameStream", boom)


def test_missing_vocabulary_is_refused_first(tmp_path, monkeypatch):
    from video_features_b200.extract.extract_clip import ExtractCLIP
    _no_video_opened(monkeypatch)
    monkeypatch.setenv("VF_CLIP_BPE", str(tmp_path / "missing.txt.gz"))
    monkeypatch.setenv("HOME", str(tmp_path))
    monkeypatch.setattr(ct, "bpe_candidates", lambda: [str(tmp_path / "missing.txt.gz"),
                                                       str(tmp_path / ".cache" / "clip" / ct.BPE_NAME)])
    monkeypatch.setenv("VF_CLIP_SYNTHETIC", "0")
    with pytest.raises(FileNotFoundError, match="bpe_simple_vocab_16e6.txt.gz") as e:
        ExtractCLIP(_args(tmp_path, "CLIP-ViT-B/32", "--show_pred"))
    assert "missing.txt.gz" in str(e.value)
    ExtractCLIP(_args(tmp_path, "CLIP-ViT-B/32"))                      # without --show_pred nothing is looked up


def test_vocabulary_size_mismatch_is_refused_first(tmp_path, monkeypatch, bpe):
    from video_features_b200.extract.extract_clip import ExtractCLIP
    _no_video_opened(monkeypatch)
    monkeypatch.setenv("VF_CLIP_BPE", bpe)
    monkeypatch.delenv("VF_CLIP_SYNTHETIC", raising=False)
    sd = synthetic_weights.clip_text_state_dict(0, 512, 512, vocab_size=1000, layers=1)
    path = str(tmp_path / "ViT-B-32.pt")
    torch.save({"clip." + k: v for k, v in sd.items()} | {"clip.visual.proj": torch.zeros(1)}, path)
    monkeypatch.setenv("VF_CLIP_CKPT", path)
    with pytest.raises(ValueError, match=f"has {ct.SimpleTokenizer(bpe).vocab_size} entries but .* 1000 rows"):
        ExtractCLIP(_args(tmp_path, "CLIP-ViT-B/32", "--show_pred"))


def test_long_prompt_is_refused_first(tmp_path, monkeypatch, bpe):
    from video_features_b200.extract.extract_clip import ExtractCLIP
    _no_video_opened(monkeypatch)
    monkeypatch.setenv("VF_CLIP_BPE", bpe)
    monkeypatch.setenv("VF_CLIP_SYNTHETIC", "0")
    with pytest.raises(RuntimeError, match="too long"):
        ExtractCLIP(_args(tmp_path, "CLIP-ViT-B/32", "--show_pred", "--pred_texts", "ok", "9 " * 80))
