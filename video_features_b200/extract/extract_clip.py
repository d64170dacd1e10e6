"""``ExtractCLIP`` -- drop-in for the reference's models/CLIP/extract_clip.py on the H100 engine.

Same constructor, attributes, ``forward(indices)`` / ``extract(...)`` signatures, dict keys and file naming.  What
changes underneath: ``clip.load`` is replaced by a ``ClipEngine`` (device weights + workspace), and ``preprocess`` +
``model.encode_image`` by ONE call into libvfeat.so that takes the decoder's raw uint8 frames and runs the
Pillow-exact bicubic resize, centre crop, normalisation and the ViT-B/32 tower on the GPU.

A list of videos does not go through the engine one 12-frame video at a time (600 token rows would fill 3 of the
GEMM's 74 tile slots): ``forward`` decodes ahead on a thread pool, packs the frames of consecutive videos of equal
geometry into a pinned staging buffer (three buffers: one being filled by the pool, two with engine calls in flight) and makes
one engine call per ``VF_CLIP_BATCH_FRAMES`` (default 1000: four tower chunks of <= 250 frames, whose 49 x 12 GEMM tiles
fill 8 waves of the 74 CTA pairs; 1024 would spill a ninth) frames; the features are cut back per video and handed to
the sink exactly as the reference does, per-video error behaviour included.

Differences a user can observe, all deliberate:
  * features are float32 on the GPU as well (the reference's GPU path returns float16 because ``clip.load`` keeps the
    model in half precision on CUDA; its ``--cpu`` path returns float32);
  * a CPU device is refused (no CPU fallback);
  * weights come from a local checkpoint (``$VF_CLIP_CKPT`` or ``~/.cache/clip/ViT-B-32.pt``), never the network.
"""
from __future__ import annotations

import os
import pathlib
import threading
import time
import traceback
from concurrent.futures import ThreadPoolExecutor
from typing import Dict, List, Optional

import numpy as np
import torch
from tqdm import tqdm

from .. import synthetic_weights
from ..clip_engine import ClipEngine
from ..utils import (AsyncSink, FrameStream, action_on_extraction, already_extracted, extract_frames,
                     form_list_from_user_input)

_CKPT_NAMES = {'CLIP-ViT-B/32': 'ViT-B-32.pt', 'CLIP-ViT-B/16': 'ViT-B-16.pt', 'CLIP4CLIP-ViT-B-32': 'CLIP4CLIP-ViT-B-32.pth'}


def read_clip_checkpoint(path: str) -> Dict[str, torch.Tensor]:
    """A checkpoint in one of the forms ``clip.load`` accepts (third-party openai/CLIP ``clip/clip.py``): a TorchScript
    archive (what it downloads) or a pickled state dict, possibly nested under 'state_dict' and possibly with the
    ``clip.`` prefix CLIP4Clip checkpoints carry.  Returns openai's flat ``visual.*`` keys."""
    try:
        sd = torch.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:
        sd = torch.load(path, map_location="cpu")
        sd = sd.get("state_dict", sd)
    if not any(k.startswith("visual.") for k in sd) and any(k.startswith("clip.visual.") for k in sd):
        sd = {k[5:]: v for k, v in sd.items() if k.startswith("clip.")}
    return dict(sd)


def load_clip_state_dict(feature_type: str) -> Dict[str, torch.Tensor]:
    """``$VF_CLIP_CKPT``, then ``<this dir>/checkpoints/<name>`` (where the reference keeps CLIP4CLIP's file,
    extract_clip.py:56), then ``~/.cache/clip/<name>`` (where ``clip.load`` caches its download).
    ``VF_CLIP_SYNTHETIC=<seed>[:outliers]`` selects seeded synthetic weights instead (benchmarks without the file)."""
    if os.environ.get("VF_CLIP_SYNTHETIC") is not None:
        seed, outliers = synthetic_weights.parse_env(os.environ["VF_CLIP_SYNTHETIC"])
        return synthetic_weights.clip_vit_b32_state_dict(seed, outliers, patch=16 if feature_type.endswith('/16') else 32)
    name = _CKPT_NAMES[feature_type]
    cands = [os.environ.get("VF_CLIP_CKPT"), os.path.join(pathlib.Path(__file__).parent, 'checkpoints', name),
             os.path.expanduser(os.path.join("~/.cache/clip", name))]
    for p in cands:
        if p and os.path.exists(p):
            return read_clip_checkpoint(p)
    if feature_type == 'CLIP4CLIP-ViT-B-32':
        raise ValueError(cands[1])                 # extract_clip.py:57-58
    raise FileNotFoundError(f"CLIP checkpoint {name} not found (looked at {[c for c in cands if c]}); "
                            "there is no network access -- set VF_CLIP_CKPT")


class _Batch:
    """Videos of one geometry sharing one pinned staging buffer and one engine call."""

    def __init__(self, hw, slot, limit):
        self.hw = hw
        self.slot = slot
        self.limit = limit                # frames this call may hold
        self.items: List[list] = []       # [list position, video, stream, first row, future -> frames written]
        self.rows = 0


class _ListStream:
    """A fully decoded video (what a one-step `frame_source` returns) behind the two-step stream interface."""

    def __init__(self, frames, fps, stamps):
        frames = [f for f in frames if f is not None]
        if not frames:
            raise RuntimeError("no frames decoded")
        self._frames = frames
        self.count = len(frames)
        hw = tuple(frames[0].shape[:2])
        self.hw = hw if all(tuple(f.shape[:2]) == hw for f in frames) else None
        self.fps, self.timestamps_ms = fps, stamps

    def read_into(self, dst) -> int:
        for i, f in enumerate(self._frames):
            np.copyto(dst[i], f)
        return self.count

    def frames(self):
        return self._frames


class ExtractCLIP(torch.nn.Module):

    def __init__(self, args, external_call=False):
        super().__init__()
        for name in ('feature_type', 'extraction_fps', 'extract_method', 'on_extraction'):
            setattr(self, name, getattr(args, name))
        self.path_list = form_list_from_user_input(args)
        self.external_call = external_call
        if not external_call:
            # --output_direct writes <output_path>/<stem>.npy; otherwise a per-feature sub-folder (which cannot exist for
            # 'CLIP-ViT-B/32': the '/' in the key -- reference quirk, SURVEY 8 quirk 4)
            self.output_direct = args.output_direct
            self.output_path = args.output_path if self.output_direct is True else os.path.join(args.output_path, self.feature_type)
        self.progress = tqdm(total=len(self.path_list))
        self._engines: Dict[int, ClipEngine] = {}
        # engine-side knobs (not in the reference): where frames come from, and how many go into one engine call
        self.frame_source = extract_frames                  # (path, method) -> (frames, fps, timestamps_ms)
        # two-step source used by the list path: stream = frame_stream(path, method) knows .count / .hw / .fps /
        # .timestamps_ms, and stream.read_into(dst) decodes straight into the pinned staging rows (no extra copy).
        # None: wrap `frame_source` (tests and callers that replaced it).
        self.frame_stream = FrameStream
        self.batch_frames = int(os.environ.get("VF_CLIP_BATCH_FRAMES", "1000"))
        # the first engine call of a list is one tower chunk: the GPU starts after ~250 decoded frames instead of 1000
        self.first_batch_frames = int(os.environ.get("VF_CLIP_FIRST_BATCH_FRAMES", "250"))
        self.decode_workers = int(os.environ.get("VF_DECODE_WORKERS", str(min(8, os.cpu_count() or 1))))
        self.keep_features = False        # dispatch sets it when the features are all-gathered as well as saved
        # with keep_features: (first list position, rows of consecutive delivered videos still on the GPU), one per engine call
        self.device_chunks: List[tuple] = []
        # seconds the stages of the last batched forward spent waiting on each other (diagnostics: which side is the limiter)
        self.stage_wait = {"engine_for_decode": 0.0, "engine_enqueue": 0.0, "host_for_slot": 0.0, "deliver_for_gpu": 0.0}

    def _engine(self, device: torch.device) -> ClipEngine:
        if device.type != 'cuda':
            raise RuntimeError("the H100 engine has no CPU path: pass indices on a CUDA device "
                               "(the reference's --cpu flow is timed by bench.py --impl reference)")
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._engines:
            if self.feature_type not in _CKPT_NAMES:
                # the reference's clip.load would also take the ResNet towers (extract_clip.py:46-64); the ViT-B
                # towers (patch 32: north_star; patch 16) are the ones built here
                raise NotImplementedError(self.feature_type)
            self._engines[idx] = ClipEngine(load_clip_state_dict(self.feature_type), device=idx)
        return self._engines[idx]

    # ------------------------------------------------------------------ forward
    def forward(self, indices: torch.LongTensor):
        """indices {torch.LongTensor} -- indices to self.path_list; the device is taken from ``indices.device``."""
        device = indices.device
        model = self._engine(device)          # one engine per device, kept across calls
        ids = indices.tolist() if hasattr(indices, 'tolist') else [int(i) for i in indices]   # ONE device read, not one per index
        # opt-in extras beyond the reference (SURVEY 8(f) rank 2): VF_ASYNC_SINK=1 saves from a writer thread,
        # VF_RESUME=1 skips videos whose output files already exist
        saving = not self.external_call
        sink = AsyncSink() if saving and os.environ.get("VF_ASYNC_SINK") == "1" else None
        resume = saving and os.environ.get("VF_RESUME") == "1"
        todo = []
        for pos, idx in enumerate(ids):
            video = self.path_list[idx]
            if resume and already_extracted([self.feature_type], video, self.output_path, self.on_extraction,
                                            self.output_direct):
                self.progress.update()
                continue
            todo.append((pos, video))
        collected: Dict[int, dict] = {}
        self.device_chunks = []
        try:
            if len(todo) > 1 and self.batch_frames > 0:
                self._forward_batched(device, model, todo, collected, sink)
            else:
                for pos, video in todo:
                    try:                            # per-video catch-print-continue (extract_clip.py:71-84)
                        self._deliver(self.extract(device, model, None, video), pos, video, collected, sink)
                    except KeyboardInterrupt:
                        raise
                    except Exception as err:
                        self._report(err, video)
                    self.progress.update()
        finally:
            if sink is not None:
                sink.close()
        return [collected[p] for p in sorted(collected)]

    def _report(self, err, video):
        print(err)
        print(f'Extraction failed at: {video} with error (↑). Continuing extraction')
        traceback.print_exception(type(err), err, err.__traceback__)

    def _deliver(self, feats: dict, pos: int, video, collected: dict, sink: Optional[AsyncSink]):
        if self.external_call or self.keep_features:
            collected[pos] = feats
        if self.external_call:
            return
        if sink is not None:
            sink.submit(feats, video, self.output_path, self.on_extraction, self.output_direct)
        else:
            action_on_extraction(feats, video, self.output_path, self.on_extraction, self.output_direct)

    def _decode(self, video):
        frames, fps, stamps = self.frame_source(str(video), self.extract_method)
        frames = [f for f in frames if f is not None]
        if not frames:
            raise RuntimeError(f"no frames decoded from {video}")
        return frames, fps, stamps

    def _open(self, video):
        if self.frame_stream is not None and self.frame_source is extract_frames:
            st = self.frame_stream(str(video), self.extract_method)
            if st.count <= 0:
                raise RuntimeError(f"no frames decoded from {video}")
            return st
        return _ListStream(*self.frame_source(str(video), self.extract_method))

    def _open_block(self, videos):
        """Open a block of videos on one pool thread: [stream or the exception]."""
        out = []
        for v in videos:
            try:
                out.append(self._open(v))
            except KeyboardInterrupt:
                raise
            except Exception as err:
                out.append(err)
        return out

    def _forward_batched(self, device, model: ClipEngine, todo, collected, sink):
        """Stages, each on its own thread(s), so the GPU never waits for Python:
             pool: open videos (blocks of 8)  ->  this thread: rows of a pinned staging slot are assigned in list order
             ->  pool: every stream decodes INTO its rows  ->  engine thread: ONE asynchronous engine call per
             <= batch_frames rows (enqueued while the previous one still runs: its first H2D copy overlaps that tower)
             ->  delivery thread: waits for the call, per-video slices, sink."""
        workers = max(1, self.decode_workers)
        pool = ThreadPoolExecutor(workers, thread_name_prefix="vf-decode")
        gpu = ThreadPoolExecutor(1, thread_name_prefix="vf-engine")           # engine calls are serialised: one handle
        out = ThreadPoolExecutor(1, thread_name_prefix="vf-deliver")
        n_slots = 3
        pinned: List[Optional[torch.Tensor]] = [None] * n_slots
        pinned_np: List[Optional[np.ndarray]] = [None] * n_slots
        feats_out: List[Optional[torch.Tensor]] = [None] * n_slots            # pinned (batch_frames, 512) landing buffers
        busy = [None] * n_slots                                               # engine future still reading slot k
        delivered = []
        state = {"slot": 0, "batches": 0}
        lock = threading.Lock()
        waits = self.stage_wait = dict.fromkeys(self.stage_wait, 0.0)

        def deliver_one(pos, video, feats, fps, stamps):
            try:
                with lock:
                    self._deliver({self.feature_type: feats, 'fps': np.array(fps), 'timestamps_ms': np.array(stamps)},
                                  pos, video, collected, sink)
                ok = True
            except Exception as err:
                self._report(err, video)
                ok = False
            self.progress.update()
            return ok

        def deliver(batch: _Batch, feats, counts, dev=None):
            good = []                                                         # (row0, k) of the videos that were delivered
            for (pos, video, st, row0, _), k in zip(batch.items, counts):
                if isinstance(k, Exception):
                    self._report(k, video)
                    self.progress.update()
                elif k <= 0:
                    self._report(RuntimeError(f"no frames decoded from {video}"), video)
                    self.progress.update()
                elif deliver_one(pos, video, feats[row0:row0 + k].copy(), st.fps, st.timestamps_ms):
                    good.append((row0, k))
            if dev is not None and good:
                # the same rows, still on the GPU, for a gather: the call's tensor as it is when every video made it
                rows = dev[:batch.rows] if sum(k for _, k in good) == batch.rows else torch.cat([dev[a:a + k] for a, k in good])
                with lock:
                    self.device_chunks.append((batch.items[0][0], rows))

        def batch_failed(batch: _Batch, counts, view):
            # the batched call failed: find the culprit by running its videos one at a time (engine thread only)
            for (pos, video, st, row0, _), k in zip(batch.items, counts):
                try:
                    if isinstance(k, Exception):
                        raise k
                    f = model.encode_frames_u8_host(view[row0:row0 + k]).numpy()
                    deliver_one(pos, video, f, st.fps, st.timestamps_ms)
                except Exception as err:
                    self._report(err, video)
                    self.progress.update()

        def finish(batch: _Batch, ticket, feats, counts, dev):
            try:
                t0 = time.perf_counter()
                model.wait(ticket)                                            # features are in the pinned landing buffer
                waits["deliver_for_gpu"] += time.perf_counter() - t0
            except Exception as err:                                          # a device fault: every video of the call is lost
                for (pos, video, st, row0, _) in batch.items:
                    self._report(err, video)
                    self.progress.update()
                return
            deliver(batch, feats.numpy(), counts, dev)

        def run_batch(batch: _Batch):
            counts = []
            t0 = time.perf_counter()
            for it in batch.items:                                            # the decodes into this slot are complete
                fut, i = it[4]
                counts.append(fut.result()[i])
            t1 = time.perf_counter()
            waits["engine_for_decode"] += t1 - t0
            h, w = batch.hw
            view = pinned[batch.slot][:batch.rows * h * w * 3].view(batch.rows, h, w, 3)
            feats = feats_out[batch.slot][:batch.rows]
            try:
                ticket, dev = model.encode_frames_u8_host_async(view, feats, out_dev=self.keep_features)
            except Exception:
                batch_failed(batch, counts, view)
                return None
            waits["engine_enqueue"] += time.perf_counter() - t1
            done = out.submit(finish, batch, ticket, feats, counts, dev)           # waiting, slicing and the sink run beside the
            delivered.append(done)                                            # next call's enqueue
            return done

        def wait_slot(k):
            if busy[k] is not None:
                t0 = time.perf_counter()
                done = busy[k].result()                                       # enqueued ...
                if done is not None:
                    done.result()                                             # ... and finished with the slot's buffers
                busy[k] = None
                waits["host_for_slot"] += time.perf_counter() - t0

        def new_batch(hw):
            k = state["slot"]
            state["slot"] = (k + 1) % n_slots
            wait_slot(k)                                                      # the engine has finished with this buffer
            need = self.batch_frames * hw[0] * hw[1] * 3
            if pinned[k] is None or pinned[k].numel() < need:
                pinned[k] = torch.empty(need, dtype=torch.uint8)
                if torch.cuda.is_available():                                 # (host-logic tests run without a device)
                    pinned[k] = pinned[k].pin_memory()
                pinned_np[k] = pinned[k].numpy()
            if feats_out[k] is None:
                feats_out[k] = torch.empty((self.batch_frames, 512), dtype=torch.float32)
                if torch.cuda.is_available():
                    feats_out[k] = feats_out[k].pin_memory()
            first = state["batches"] == 0 and 0 < self.first_batch_frames < self.batch_frames
            state["batches"] += 1
            return _Batch(hw, k, self.first_batch_frames if first else self.batch_frames)

        pending: List[tuple] = []                                             # (batch item, its staging rows) not yet submitted

        def read_many(jobs):
            out_counts = []
            for item, dst in jobs:
                try:
                    out_counts.append(item[2].read_into(dst))
                except Exception as err:
                    out_counts.append(err)
            return out_counts

        def submit_reads():
            if pending:
                jobs = list(pending)
                pending.clear()
                fut = pool.submit(read_many, jobs)
                for i, (item, _) in enumerate(jobs):
                    item[4] = (fut, i)

        def seal(batch: _Batch):
            submit_reads()
            if batch.items:
                busy[batch.slot] = gpu.submit(run_batch, batch)

        try:
            block = 8                                                         # videos per open task
            blocks = [todo[i:i + block] for i in range(0, len(todo), block)]
            window = 4 * workers                                              # open blocks in flight, bounds host memory
            futs = {}
            nxt = 0
            batch: Optional[_Batch] = None
            for bi, blk in enumerate(blocks):
                while nxt < len(blocks) and nxt < bi + window:
                    futs[nxt] = pool.submit(self._open_block, [v for _, v in blocks[nxt]])
                    nxt += 1
                for (pos, video), st in zip(blk, futs.pop(bi).result()):
                    if isinstance(st, Exception):
                        self._report(st, video)
                        self.progress.update()
                        continue
                    if st.hw is None or st.count > self.batch_frames:         # mixed geometry / longer than a batch: own call
                        if batch is not None:
                            seal(batch)
                            batch = None
                        for k in range(n_slots):
                            wait_slot(k)
                        gpu.submit(self._run_lone, model, pos, video, st, collected, sink, lock).result()
                        continue
                    if batch is not None and (batch.hw != st.hw or batch.rows + st.count > max(batch.limit, st.count)):
                        seal(batch)
                        batch = None
                    if batch is None:
                        batch = new_batch(st.hw)
                    h, w = st.hw
                    dst = pinned_np[batch.slot][batch.rows * h * w * 3:(batch.rows + st.count) * h * w * 3]
                    item = [pos, video, st, batch.rows, None]
                    batch.items.append(item)
                    batch.rows += st.count
                    pending.append((item, dst.reshape(st.count, h, w, 3)))
                    if len(pending) >= block:
                        submit_reads()
                submit_reads()                                                # one pool task per block of videos
            if batch is not None:
                seal(batch)
            for k in range(n_slots):
                wait_slot(k)
            for d in delivered:
                d.result()
        finally:
            gpu.shutdown(wait=True)
            out.shutdown(wait=True)
            pool.shutdown(wait=True)

    def _run_lone(self, model, pos, video, st, collected, sink, lock):
        """A video that cannot share a staging buffer (frames of different sizes -- never seen from a real decoder -- or
        more frames than a batch holds): its own engine call(s), like the reference's per-video loop."""
        try:
            if st.hw is None:
                f = np.concatenate([model.encode_frames_u8_host(torch.from_numpy(np.ascontiguousarray(x))[None]).numpy()
                                    for x in st.frames()])
            else:
                buf = np.empty((st.count, st.hw[0], st.hw[1], 3), np.uint8)
                k = st.read_into(buf)
                if k <= 0:
                    raise RuntimeError(f"no frames decoded from {video}")
                f = model.encode_frames_u8_host(torch.from_numpy(buf[:k])).numpy()
            with lock:
                self._deliver({self.feature_type: f, 'fps': np.array(st.fps), 'timestamps_ms': np.array(st.timestamps_ms)},
                              pos, video, collected, sink)
        except Exception as err:
            self._report(err, video)
        self.progress.update()

    # ------------------------------------------------------------------ extract (one video)
    def extract(self, device: torch.device, model: ClipEngine, preprocess_func=None, video_path=None):
        """-> {feature_type: (T,512) float32, 'fps': (), 'timestamps_ms': (T,)}.  ``preprocess_func`` is accepted for
        signature compatibility; the transform is fused into the engine call."""
        decoded, fps, stamps = self._decode(video_path)
        batch = torch.from_numpy(np.stack(decoded))         # (T,H,W,3) uint8, decoder channel order untouched
        feats = model.encode_frames_u8_host(batch)          # H2D + transform + tower + D2H
        return {self.feature_type: feats.numpy(), 'fps': np.array(fps), 'timestamps_ms': np.array(stamps)}
