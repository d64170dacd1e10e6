"""Generates tests/golden/*.npz by running the REFERENCE's own python (imported from /root/reference, never
copied) and the third-party libraries it relies on (Pillow) in the build container.  /root/reference does not
exist on the GPU box, so tests read only the committed fixtures.

    python scripts/make_golden.py            # needs /root/reference
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import stand_in_state_dict  # noqa: E402


def install_mmcv_shim():
    """mmcv is un-vendored and absent: the reference only uses VideoReader(.fps,.frame_cnt,.get_frame) and imread.
    The shim decodes with cv2 exactly as mmcv does (seek with CAP_PROP_POS_FRAMES, frames are BGR), or -- for
    paths of the form 'synthetic:<frame_cnt>:<fps>' -- fabricates a video whose frame i is the integer i."""
    import cv2

    class VideoReader:
        def __init__(self, path):
            self._synthetic = str(path).startswith("synthetic:")
            if self._synthetic:
                _, cnt, fps = str(path).split(":")
                self.frame_cnt, self.fps = int(cnt), float(fps)
            else:
                self._cap = cv2.VideoCapture(str(path))
                self.fps = self._cap.get(cv2.CAP_PROP_FPS)
                self.frame_cnt = int(self._cap.get(cv2.CAP_PROP_FRAME_COUNT))

        def get_frame(self, i):
            if self._synthetic:
                return int(i)
            self._cap.set(cv2.CAP_PROP_POS_FRAMES, int(i))
            ok, frame = self._cap.read()
            return frame if ok else None

    m = types.ModuleType("mmcv")
    m.VideoReader = VideoReader
    m.imread = lambda p, flag="color": cv2.imread(p, cv2.IMREAD_GRAYSCALE if flag == "grayscale" else cv2.IMREAD_COLOR)
    sys.modules["mmcv"] = m


def main():
    assert os.path.isdir(REF), "needs the reference checkout"
    os.makedirs(OUT, exist_ok=True)
    install_mmcv_shim()
    sys.path.insert(0, REF)
    cwd = os.getcwd()
    os.chdir(REF)
    try:
        from utils.utils import extract_frames          # the reference's sampler, unmodified
        # ---- 1. sampler indices over a grid of (frame_cnt, fps, method)
        cases, flat, offs = [], [], [0]
        for cnt in (3, 4, 10, 65, 100, 355, 420, 1000, 2997, 18000):
            for fps in (19.62, 23.976, 25.0, 29.97, 30.0, 60.0):
                for method in ("uni_1", "uni_2", "uni_12", "uni_64", "fix_1", "fix_2", "fix_5"):
                    frames, fps_out, ts = extract_frames(f"synthetic:{cnt}:{fps}", method)
                    cases.append((cnt, fps, method))
                    flat.extend(int(f) for f in frames)
                    offs.append(len(flat))
        np.savez_compressed(os.path.join(OUT, "sampler_indices.npz"),
                            frame_cnt=np.array([c[0] for c in cases], np.int64),
                            fps=np.array([c[1] for c in cases], np.float64),
                            method=np.array([c[2] for c in cases]),
                            flat=np.array(flat, np.int64), offsets=np.array(offs, np.int64))
        print("sampler cases:", len(cases))

        # ---- 2. BASELINE config 1: uni_12 on the sample video through the reference sampler (real decode)
        frames, fps, ts = extract_frames(os.path.join(REF, "sample", "v_GGSY1Qvo990.mp4"), "uni_12")
        frames = np.stack(frames)                        # (12,240,320,3) uint8 BGR
        import cv2
        cap = cv2.VideoCapture(os.path.join(REF, "sample", "v_GGSY1Qvo990.mp4"))
        cnt = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
        idx = np.linspace(1, cnt - 2, 12).astype(int)
        # the reference transform on two of them: Image.fromarray (no BGR swap) -> torchvision Resize/CenterCrop
        from PIL import Image
        import torchvision.transforms as T
        tf = T.Compose([T.Resize(224, interpolation=T.InterpolationMode.BICUBIC), T.CenterCrop(224)])
        keep = [0, 7]
        cropped = np.stack([np.asarray(tf(Image.fromarray(frames[i]))) for i in keep])
        np.savez_compressed(os.path.join(OUT, "config1_sample_video.npz"), indices=idx, fps=np.float64(fps),
                            frame_cnt=np.int64(cnt), timestamps_ms=np.array(ts, np.float64),
                            frames=frames[keep], kept=np.array(keep), resized_cropped=cropped,
                            frame_checksums=np.array([int(f.astype(np.uint64).sum()) for f in frames], np.uint64))
        print("config1: indices", idx.tolist(), "fps", fps)

        # ---- 3. I3D host resize chain (ToPILImage -> ResizeImproved(256) bilinear) from the reference transforms
        from models.i3d.transforms.transforms import ResizeImproved, PILToTensor, TensorCenterCrop
        import torch
        import torchvision
        rng = np.random.default_rng(5)
        src = [frames[0], rng.integers(0, 256, (135, 240, 3), dtype=np.uint8),
               rng.integers(0, 256, (150, 128, 3), dtype=np.uint8)]
        outs = []
        for s in src:
            t = torch.from_numpy(s).permute(2, 0, 1)
            r = PILToTensor()(ResizeImproved(256)(torchvision.transforms.ToPILImage()(t)))
            outs.append(r.permute(1, 2, 0).numpy())
        np.savez_compressed(os.path.join(OUT, "i3d_resize.npz"),
                            **{f"src{i}": s for i, s in enumerate(src)}, **{f"out{i}": o for i, o in enumerate(outs)})
        print("i3d resize:", [o.shape for o in outs])
    finally:
        os.chdir(cwd)

    # ---- 4. Pillow itself (third-party; the CLIP transform's Resize) on random images, incl. an up-scale
    from PIL import Image
    rng = np.random.default_rng(0)
    d = {}
    for n, (h, w, oh, ow, f) in enumerate([(240, 320, 224, 298, Image.BICUBIC), (90, 120, 56, 74, Image.BICUBIC),
                                           (100, 60, 373, 224, Image.BICUBIC), (120, 160, 128, 170, Image.BILINEAR),
                                           (135, 240, 128, 227, Image.BILINEAR), (64, 48, 31, 17, Image.BICUBIC)]):
        im = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        d[f"in{n}"] = im
        d[f"out{n}"] = np.asarray(Image.fromarray(im).resize((ow, oh), f))
        d[f"filter{n}"] = np.int64(f)
    import PIL
    d["pillow_version"] = np.array(PIL.__version__)
    np.savez_compressed(os.path.join(OUT, "pillow_resize.npz"), **d)

    # ---- 5. CLIP tower: oracle restatement vs HF transformers (independent implementation), seeded
    import torch
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    from oracle import clip_tower
    sd = clip_tower.synthetic_state_dict(0)
    hf = CLIPVisionModelWithProjection(CLIPVisionConfig()).eval()
    missing = hf.load_state_dict(clip_tower.to_hf_state_dict(sd), strict=False)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(4, 3, 224, 224, generator=g)
    with torch.no_grad():
        y_hf = hf(pixel_values=x).image_embeds
    y_or = clip_tower.encode_image(sd, x)
    print("oracle vs HF rel:", float((y_or - y_hf).norm() / y_hf.norm()), "missing:", missing.missing_keys)
    np.savez_compressed(os.path.join(OUT, "clip_tower_seed0.npz"), x_seed=np.int64(11), y_hf=y_hf.numpy(),
                        y_oracle=y_or.numpy())




def i3d_golden():
    """Reference I3D module + the seeded stand-ins of its checkpoints (oracle/stand_in.py) vs the restated oracle, seeded
    inputs; stores only the outputs."""
    import torch
    sys.path.insert(0, REF)
    cwd = os.getcwd()
    os.chdir(REF)
    try:
        from models.i3d.i3d_src.i3d_net import I3D
        from oracle import i3d_net
        d = {}
        for mod, cin in (("rgb", 3), ("flow", 2)):
            sd = stand_in_state_dict(f"i3d_{mod}.pt")
            net = I3D(num_classes=400, modality=mod).eval()
            net.load_state_dict(sd)
            for T in (16, 11):
                x = torch.rand(1, cin, T, 224, 224, generator=torch.Generator().manual_seed(100 + T)) * 2 - 1
                with torch.no_grad():
                    y_ref = net(x, features=True)
                y_or = i3d_net.forward_features(sd, x)
                rel = float((y_or - y_ref).norm() / y_ref.norm())
                print(f"i3d {mod} T={T}: oracle vs reference rel {rel:.2e}")
                assert rel < 1e-5
                d[f"{mod}_T{T}"] = y_ref.numpy()
        # synthetic-weight outputs, so the oracle is also pinned where the checkpoints are not available
        for mod, cin in (("rgb", 3), ("flow", 2)):
            sd = i3d_net.synthetic_state_dict(mod, 0)
            net = I3D(num_classes=400, modality=mod).eval()
            net.load_state_dict(sd, strict=False)
            x = torch.rand(1, cin, 12, 224, 224, generator=torch.Generator().manual_seed(7)) * 2 - 1
            with torch.no_grad():
                y_ref = net(x, features=True)
            y_or = i3d_net.forward_features(sd, x)
            print(f"i3d {mod} synthetic: rel {float((y_or - y_ref).norm() / y_ref.norm()):.2e}")
            d[f"{mod}_synth_T12"] = y_ref.numpy()
        np.savez_compressed(os.path.join(OUT, "i3d_outputs.npz"), **d)
    finally:
        os.chdir(cwd)


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "i3d":
    i3d_golden()
    raft_golden()


if __name__ == "__main__" and len(sys.argv) == 1:
    main()
    i3d_golden()
    raft_golden()


def raft_golden():
    """Reference RAFT module + the seeded stand-in of raft-sintel.pth (oracle/stand_in.py) vs the restated oracle on
    synthetic moving frames."""
    import torch
    sys.path.insert(0, REF)
    cwd = os.getcwd()
    os.chdir(REF)
    try:
        from models.raft.raft_src.raft import RAFT, InputPadder
        from oracle import raft_net
        sd = stand_in_state_dict("raft-sintel.pth")
        net = torch.nn.DataParallel(RAFT(), device_ids=None)
        net.load_state_dict(sd)
        net = net.module.eval()
        d = {}
        for (h, w, n) in ((128, 160, 3), (270, 480, 2)):
            fr = raft_net.synthetic_frames(n, h, w, seed=h)
            padder = InputPadder(fr.shape)
            x = padder.pad(fr)
            assert torch.equal(x, raft_net.pad(fr))
            with torch.no_grad():
                y_ref = net(x[:-1], x[1:], iters=20)
            y_or = raft_net.forward(sd, x[:-1], x[1:], 20)
            rel = float((y_or - y_ref).norm() / y_ref.norm())
            print(f"raft {h}x{w}: oracle vs reference rel {rel:.2e}; mean |flow| {float(y_ref.abs().mean()):.3f}")
            assert rel < 1e-4
            full = padder.unpad(y_ref).numpy().astype(np.float32)
            d[f"flow_{h}x{w}"] = full if h < 200 else full[:, :, ::3, ::3]      # keep the fixture small
        np.savez_compressed(os.path.join(OUT, "raft_outputs.npz"), **d)
    finally:
        os.chdir(cwd)


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "raft":
    raft_golden()


def raft_one_pixel_level_golden():
    """The reference RAFT module (stand-in weights, 2 iterations) at padded sizes whose 4th pyramid level is one pixel
    tall (96x128: 12x16 /8 map, level 3 is 1x2) or one pixel in both axes (64x120: 8x15, level 3 is 1x1).  Its
    bilinear_sampler divides by H - 1 = 0 there: the fixture records the flow it returns (NaN)."""
    import torch
    sys.path.insert(0, REF)
    cwd = os.getcwd()
    os.chdir(REF)
    try:
        from models.raft.raft_src.raft import RAFT
        from oracle import raft_net
        sd = stand_in_state_dict("raft-sintel.pth")
        net = torch.nn.DataParallel(RAFT(), device_ids=None)
        net.load_state_dict(sd)
        net = net.module.eval()
        d = {}
        for (h, w) in ((96, 128), (64, 120)):
            fr = raft_net.synthetic_frames(2, h, w, seed=h)
            with torch.no_grad():
                y_ref = net(fr[:-1], fr[1:], iters=2)
            print(f"raft {h}x{w}: {int(torch.isnan(y_ref).sum())} of {y_ref.numel()} flow values NaN")
            d[f"flow_{h}x{w}"] = y_ref.numpy().astype(np.float32)
        np.savez_compressed(os.path.join(OUT, "raft_one_pixel_level.npz"), **d)
    finally:
        os.chdir(cwd)


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "raft_1px":
    raft_one_pixel_level_golden()


def resnet_golden():
    """The reference's own ExtractResNet.extract on the sample video, with torchvision's resnet constructors patched to
    return the calibrated stand-in (oracle/resnet_net.py); stores fps, timestamps, a sha1 per frame of the transform
    output, and the feature rows of every 16th frame plus the last, for resnet18 and resnet50."""
    import argparse
    import torch
    from oracle import resnet_net
    install_mmcv_shim()
    sys.path.insert(0, REF)
    cwd = os.getcwd()
    os.chdir(REF)
    try:
        from models.resnet import extract_resnet
        video = os.path.join(REF, "sample", "v_GGSY1Qvo990.mp4")
        d = {}
        for depth in (18, 50):
            name = f"resnet{depth}"
            tv = extract_resnet.models

            sd = resnet_net.stand_in_state_dict(depth)       # built before the constructor is patched
            orig = getattr(tv, name)

            def patched(pretrained=False, _sd=sd, _orig=orig):
                net = _orig(weights=None)
                net.load_state_dict(_sd)
                return net
            args = argparse.Namespace(feature_type=name, video_paths=[video], file_with_video_paths=None, batch_size=16,
                                      extraction_fps=None, show_pred=False, keep_tmp_files=False, on_extraction="print",
                                      tmp_path="./tmp", output_path="./output", video_dir=None,
                                      flow_paths=None, flow_dir=None)
            ex = extract_resnet.ExtractResNet(args)
            hashes = []
            tf = ex.transforms

            def hashing(img, _tf=tf, _h=hashes):
                t = _tf(img)
                _h.append(resnet_net.tensor_hash(t))
                return t
            ex.transforms = hashing
            setattr(tv, name, patched)
            model = getattr(tv, name)(pretrained=True).eval()
            model.fc = torch.nn.Identity()
            out = ex.extract(torch.device("cpu"), model, None, video)
            setattr(tv, name, orig)
            feats = out[name]
            n = feats.shape[0]
            rows = np.array(sorted(set(range(0, n, 16)) | {n - 1}), np.int64)
            d[name] = feats[rows]
            d["rows"], d["fps"], d["timestamps_ms"] = rows, out["fps"], out["timestamps_ms"]
            d["transform_sha1"] = np.array(hashes)
            print(f"{name}: {n} frames, fps {out['fps']}, kept rows {len(rows)}")
        np.savez_compressed(os.path.join(OUT, "resnet_outputs.npz"), **d)
    finally:
        os.chdir(cwd)


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "resnet":
    resnet_golden()


def r21d_golden():
    """The reference's own R(2+1)D pieces on the sample video, with the calibrated stand-in (oracle/r21d_net.py):
    frames decoded with OpenCV and swapped BGR->RGB (the reference's torchvision.io.read_video needs PyAV), the
    reference's rgb_transforms Compose, its form_slices, and torchvision r2plus1d_18 with fc = Identity.  Stores the
    sha1 of every transformed stack and all feature rows (355 frames -> 22 stacks of 16)."""
    import cv2
    import torch
    import torchvision
    from torchvision.transforms import Compose
    from oracle import r21d_net
    install_mmcv_shim()
    sys.path.insert(0, REF)
    import models.r21d.transforms.rgb_transforms as T
    from utils.utils import form_slices
    cap = cv2.VideoCapture(os.path.join(REF, "sample", "v_GGSY1Qvo990.mp4"))
    frames = []
    while True:
        ok, bgr = cap.read()
        if not ok:
            break
        frames.append(bgr[:, :, ::-1].copy())
    rgb = torch.from_numpy(np.stack(frames))                                 # (T, H, W, 3), read_video's layout
    tf = Compose([T.ToFloatTensorInZeroOne(), T.Resize((128, 171)),
                  T.Normalize(mean=[0.43216, 0.394666, 0.37645], std=[0.22803, 0.22145, 0.216989]),
                  T.CenterCrop((112, 112))])                                 # extract_r21d.py's Compose
    x = tf(rgb).unsqueeze(0)
    net = torchvision.models.video.r2plus1d_18(weights=None)
    net.load_state_dict(r21d_net.stand_in_state_dict())
    net.fc = torch.nn.Identity()
    net.eval()
    feats, hashes = [], []
    with torch.no_grad():
        for s, e in form_slices(x.size(2), 16, 16):
            hashes.append(r21d_net.tensor_hash(x[0, :, s:e]))
            feats.extend(net(x[:, :, s:e]).tolist())
    feats = np.array(feats)
    print(f"r21d: {len(frames)} frames -> {feats.shape}")
    np.savez_compressed(os.path.join(OUT, "r21d_outputs.npz"), r21d_rgb=feats, transform_sha1=np.array(hashes),
                        n_frames=np.array(len(frames)))


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "r21d":
    r21d_golden()


def vggish_golden():
    """The reference's own VGGish pieces (models/vggish_torch/vggish_src) on a seeded ~7 s 16 kHz mono clip
    (oracle/vggish_net.py synthetic_audio): vggish_input.waveform_to_examples of samples / 32768.0 (what
    wavfile_to_examples feeds it) and VGG.forward on the calibrated stand-in (postprocess=False).  resampy and soundfile
    need not be installed: they are stubbed in sys.modules, and neither is called at 16 kHz.  Stores the int16 samples, the
    fp32 examples and the features."""
    import torch
    from oracle import vggish_net
    for name in ("resampy", "soundfile"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.path.insert(0, os.path.join(REF, "models", "vggish_torch"))
    from vggish_src import vggish, vggish_input
    samples = vggish_net.synthetic_audio(7.0, 16000, 1, seed=7)
    ex = vggish_input.waveform_to_examples(samples / 32768.0, 16000)          # (n, 1, 96, 64) fp32
    net = vggish.VGG(vggish.make_layers())
    net.load_state_dict(vggish_net.stand_in_state_dict())
    net.eval()
    with torch.no_grad():
        feats = net(ex).numpy()
    ex = ex.detach().numpy()[:, 0]
    print(f"vggish: {samples.shape[0]} samples -> examples {ex.shape}, features {feats.shape}")
    np.savez_compressed(os.path.join(OUT, "vggish_outputs.npz"), samples=samples, sample_rate=np.array(16000),
                        examples=ex, vggish_torch=feats)


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "vggish":
    vggish_golden()


def show_pred_golden():
    """--show_pred fixtures: (1) the reference's own printer (utils/utils.py show_predictions_on_dataset) on seeded
    logits for both datasets, its stdout captured; (2) both label maps, as data; (3) the reference I3D module's
    (softmax, logits) = model(x, features=False) on the stand-in weights (oracle/stand_in.py) for the rgb and flow
    streams at T = 64 and 16; (4) with the reference's real i3d_rgb.pt, the logits of the first five 64-frame rgb stacks
    of sample/v_GGSY1Qvo990.mp4, decoded (cv2, BGR kept) and transformed with the reference's own transforms."""
    import contextlib
    import io
    import torch
    import torchvision
    install_mmcv_shim()
    sys.path.insert(0, REF)
    cwd = os.getcwd()
    os.chdir(REF)
    try:
        from utils.utils import show_predictions_on_dataset
        from models.i3d.i3d_src.i3d_net import I3D
        from models.i3d.transforms.transforms import (PermuteAndUnsqueeze, PILToTensor, ResizeImproved, ScaleTo1_1,
                                                      TensorCenterCrop, ToFloat)
        from oracle import class_heads
        d = {}
        # (1) + (2)
        for ds, n_cls, fname in (("kinetics", 400, "K400_label_map.txt"), ("imagenet", 1000, "IN_label_map.txt")):
            g = torch.Generator().manual_seed(31 if ds == "kinetics" else 32)
            logits = torch.randn(6, n_cls, generator=g) * 3.0
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                show_predictions_on_dataset(logits, ds)
            d[f"{ds}_logits"] = logits.numpy()
            d[f"{ds}_text"] = np.array(buf.getvalue())
            d[f"{ds}_labels"] = np.array([x.strip() for x in open(os.path.join(REF, "utils", fname))])
        # (3)
        for mod, cin in (("rgb", 3), ("flow", 2)):
            sd = stand_in_state_dict(f"i3d_{mod}.pt")
            net = I3D(num_classes=400, modality=mod).eval()
            net.load_state_dict(sd)
            for T in (64, 16):
                x = torch.rand(1, cin, T, 224, 224, generator=torch.Generator().manual_seed(200 + T)) * 2 - 1
                with torch.no_grad():
                    smax, logits = net(x, features=False)
                osm, olg = class_heads.i3d_forward_logits(sd, x)
                rel = float((olg - logits).norm() / logits.norm())
                print(f"i3d {mod} T={T} features=False: oracle vs reference logits rel {rel:.2e}")
                assert rel < 1e-5
                d[f"{mod}_T{T}_softmax"], d[f"{mod}_T{T}_logits"] = smax.numpy(), logits.numpy()
        # (4)
        real = os.path.join(REF, "models", "i3d", "checkpoints", "i3d_rgb.pt")
        import cv2
        cap = cv2.VideoCapture(os.path.join(REF, "sample", "v_GGSY1Qvo990.mp4"))
        frames = []
        while True:
            ok, f = cap.read()
            if not ok:
                break
            frames.append(f)
        resize = torchvision.transforms.Compose([torchvision.transforms.ToPILImage(), ResizeImproved(256), PILToTensor(),
                                                 ToFloat()])
        tf = torchvision.transforms.Compose([TensorCenterCrop(224), ScaleTo1_1(), PermuteAndUnsqueeze()])
        net = I3D(num_classes=400, modality="rgb").eval()
        net.load_state_dict(torch.load(real, map_location="cpu"))
        sm, lg = [], []
        for s in range(5):                      # stacks of 65 frames, step 64; rgb_stack[:-1]
            stack = torch.stack([resize(f) for f in frames[64 * s:64 * s + 64]])
            with torch.no_grad():
                a, b = net(tf(stack), features=False)
            sm.append(a.numpy())
            lg.append(b.numpy())
        d["real_rgb_softmax"], d["real_rgb_logits"] = np.concatenate(sm), np.concatenate(lg)
        print("real i3d_rgb top-1:", d["real_rgb_logits"].argmax(1).tolist())
        np.savez_compressed(os.path.join(OUT, "show_pred.npz"), **d)
    finally:
        os.chdir(cwd)


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "show_pred":
    show_pred_golden()
