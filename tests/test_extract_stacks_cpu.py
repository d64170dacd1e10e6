"""base.stack_calls: how the stack extractors (R(2+1)D, S3D, Swin3D, MViT) group decoded frames into engine calls,
driven with plain objects in place of frames.  CPU only."""
import weakref

import pytest

from video_features_b200.extract.base import stack_calls
from video_features_b200.utils import form_slices


class _Frame:
    __slots__ = ("i", "__weakref__")

    def __init__(self, i):
        self.i = i


def _steps(T):
    """A step below T (where there is one), T, and one above T."""
    return [s for s in (T // 2, T, T + 3) if s >= 1]


@pytest.mark.parametrize("per_call", [1, 4, 8])
@pytest.mark.parametrize("T", [1, 8, 13, 16, 32, 64])
def test_stack_calls_cover_form_slices_within_the_staging_bound(T, per_call):
    for n_frames in sorted({0, 1, T - 1, T, T + 1, 355}):
        for step in _steps(T):
            bound = min(per_call * T, (per_call - 1) * step + T)      # the pinned slot's frame capacity
            alive, peak = weakref.WeakSet(), [0]

            def source():
                for i in range(n_frames):
                    fr = _Frame(i)
                    alive.add(fr)
                    yield fr
                    peak[0] = max(peak[0], len(alive))         # frames the consumer did not let go of
                peak[0] = max(peak[0], len(alive))

            stacks, sizes = [], []
            for first, frames, starts in stack_calls(source(), T, step, per_call):
                idx = [f.i for f in frames]
                del frames
                assert idx == sorted(set(idx)) and len(idx) <= bound
                assert first == len(stacks)
                sizes.append(len(starts))
                stacks += [idx[s:s + T] for s in starts]
            where = f"n_frames {n_frames}, T {T}, step {step}, per_call {per_call}"
            assert stacks == [list(range(s, e)) for s, e in form_slices(n_frames, T, step)], where
            assert all(k == per_call for k in sizes[:-1]) and all(1 <= k <= per_call for k in sizes[-1:]), where
            assert peak[0] <= bound, where
