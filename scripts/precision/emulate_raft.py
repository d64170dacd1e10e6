"""CPU emulation behind DESIGN.md §2 (RAFT): how much of the flow error on block-compressed frames comes from rounding
which operand to fp16.  Runs the oracle (fp32 torch, CPU) on 6 decoded frames of a synthetic 128x160 mp4 and perturbs
one operand group at a time.  Needs oracle/_ref/checkpoints/raft-sintel.pth (oracle/fetch_ref.py) and cv2.

Measured in the build container (rel-L2 / max-abs relative to max |flow|, 20 iterations):
    fp32, 16 threads vs 1 thread (summation order only)          2.6e-05 / 2.8e-04
    fp32 vs fp64 oracle                                          2.5e-05 / 2.2e-04     (smooth synthetic frames: 2.4e-06)
    fp16 weights only (all groups)                               6.2e-04 / 4.6e-03
    fp16 weights: fnet / cnet / motion enc. / gru / flow head    3.4e-04 / 2.5e-04 / 5.3e-04 / 4.6e-04 / 6.5e-04   (mask head 4e-06)
    fp16 activations, fp32 weights: cnet inner layers            4.4e-04 / 6.3e-03
                                    motion-encoder intermediates 1.0e-03 / 1.2e-02
                                    flow-head hidden layer       3.7e-04 / 3.7e-03
                                    motion slice of the GRU input 2.0e-04 / 1.8e-03
    every conv input fp16 (weights fp32)                         7.6e-03
The errors do not add (the iteration is chaotic at this level): any single fp16 operand costs 2e-4 .. 1e-3 and a
max-abs outlier above the 1e-3 bar, hence split-fp16 pairs for every operand in the engine."""
import os, sys
import cv2, numpy as np, torch, torch.nn.functional as F
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import raft_net as R


def compressed_frames(path="/tmp/_raft_emul.mp4"):
    fr = R.synthetic_frames(6, 128, 160, seed=11, shift=(0.8, 0.5)).permute(0, 2, 3, 1).numpy().astype(np.uint8)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"mp4v"), 25.0, (160, 128))
    for f in fr:
        vw.write(f)
    vw.release()
    cap, out = cv2.VideoCapture(path), []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        out.append(cv2.cvtColor(f, cv2.COLOR_BGR2RGB))
    return torch.from_numpy(np.stack(out)).permute(0, 3, 1, 2).float()


def main():
    torch.set_num_threads(os.cpu_count() or 1)
    sd = torch.load(os.path.join(ROOT, "oracle", "_ref", "checkpoints", "raft-sintel.pth"), map_location="cpu")
    x = compressed_frames()
    ref = R.forward(sd, x[:-1], x[1:], 20)
    err = lambda y: (float((y - ref).norm() / ref.norm()), float((y - ref).abs().max() / ref.abs().max()))
    orig = R._conv

    def run(round_input=lambda name: False, w16=lambda name: False, gru_motion=False):
        def conv(sd_, name, xx, stride=1, padding=0):
            w = sd_[name + ".weight"]
            if w16(name):
                w = w.half().float()
            if round_input(name):
                xx = xx.half().float()
            if gru_motion and ".gru." in name:
                xx = xx.clone(); xx[:, 256:382] = xx[:, 256:382].half().float()
            return F.conv2d(xx, w, sd_[name + ".bias"], stride=stride, padding=padding)
        R._conv = conv
        try:
            return err(R.forward(sd, x[:-1], x[1:], 20))
        finally:
            R._conv = orig

    print("fp16 weights, all:", run(w16=lambda n: True))
    for g in ("fnet", "cnet", "update_block.encoder", ".gru.", "flow_head", ".mask."):
        print(f"fp16 weights, {g}:", run(w16=lambda n, g=g: g in n))
    print("fp16 inputs: cnet inner:", run(lambda n: n.startswith("cnet") and n != "cnet.conv1"))
    print("fp16 inputs: motion-encoder intermediates:", run(lambda n: n.endswith(("convc2", "convf2", "encoder.conv"))))
    print("fp16 inputs: flow_head.conv2:", run(lambda n: n.endswith("flow_head.conv2")))
    print("fp16 inputs: motion slice of the GRU input:", run(gru_motion=True))
    print("fp16 inputs: every conv:", run(lambda n: True))


if __name__ == "__main__":
    main()
