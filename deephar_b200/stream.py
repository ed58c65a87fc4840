"""Streamed clip inference: one new frame per video stream in, an action decision per stream out, for every frame.

`Model.predict` / `forward_device` on a clip model run all T frames of a clip through the network.  Called once per
new frame on a sliding window, T - 1 of those frames were already computed for the previous window.  Everything up to
the action head is per-frame (the 'frame'-kind tensors of graph.py; `TimeDistributed` in the reference), and the only
crossings from frames to clips are `frames_to_clip` views, so a ClipStream runs the model's plan in two stages
(compiler.split_stages):

  frame stage   the per-frame network on the S new frames (one per stream)
  window        dh_clip_window_f32: each crossing tensor joins a per-stream ring of its last T frames, and the clip
                stage's (S, T, ...) input is rewritten from that ring in time order
  clip stage    the action head on the S windows

The same kernels as `predict`, with the same weights and settings; the per-frame network runs once per frame instead
of T times.  The three steps are captured as one CUDA graph on the second push (Model.use_cuda_graph) and replayed
after that: the ring position is a device-side counter the window launch advances itself.

    s = ClipStream(model, n_streams=S)      # a clip Model, or a split_model view of one
    out = s.push(frames)                    # float32 CUDA (S, H, W, 3), one new frame per stream
    out.clip_outputs[k][s]                  # output k for the clip of the last T frames pushed to stream s
    out.frame_outputs[k][s]                 # frame output k (e.g. the poses) of the frame just pushed
    out.ready[s]                            # stream s has had >= T frames since its last reset
    s.reset([2])                            # stream 2 starts a new video
"""
import ctypes as C

import numpy as np

from . import _ffi
from .compiler import split_stages
from .model import _graphed, _item_dims, _OutputSubset


class StreamOutputs(object):
    """What one push returns.  Device tensors are views into the stream's buffers, valid until the next push."""
    __slots__ = ('frame_outputs', 'clip_outputs', 'ready')

    def __init__(self, frame_outputs, clip_outputs, ready):
        self.frame_outputs, self.clip_outputs, self.ready = frame_outputs, clip_outputs, ready


class ClipStream(object):
    """S video streams advancing one frame per `push` through a clip model (spnet.build with T > 1,
    action.build_merge_model) or a split_model view of one, which then computes only the view's outputs.

    For a ready stream, clip_outputs[k][s] equals the model's output k on the clip made of the last T frames pushed to s,
    in push order; rows of streams that are not ready are NaN.  frame_outputs[k][s] is the model's frame output k for
    the frame just pushed (row T-1 of that clip); it depends on that frame alone, so it is valid for every stream.
    The stream owns activation buffers and rings but no weights: it uses the model's device weights, its `precision`
    and `use_tensor_cores` settings at construction, and its `use_cuda_graph` setting at each push.
    Output shapes have one leading axis of S, trimmed as Keras shapes are here: (S, nj, dim) poses, (S, n_act) action
    probabilities."""

    def __init__(self, model, n_streams):
        if isinstance(model, _OutputSubset):
            full, outputs = model.full, [model.full.graph.outputs[i] for i in model.indices]
        else:
            full, outputs = model, list(model.graph.outputs)
        T = full.graph.frames_per_clip
        if T == 1:
            raise ValueError('model %r takes single frames (frames_per_clip == 1): there is no clip to stream' % full.name)
        S = int(n_streams)
        if S != n_streams or S < 1:
            raise ValueError('n_streams must be a positive integer, got %r' % (n_streams,))
        torch = full._torch()
        self.model, self.n_streams, self.frames_per_clip = full, S, T
        self.stages = stages = split_stages(full.graph, outputs)
        self.frame_output_tensors = [t for t in outputs if t.kind == 'frame']
        self.clip_output_tensors = [t for t in outputs if t.kind == 'clip']
        self._frame = full._bind_plan(stages.frame, S)
        self._clip = full._bind_plan(stages.clip, S * T)
        self._weights = full._dev                   # set_weights replaces it: the bound pointers would be stale
        self._rings, entries = [], []
        for t in stages.boundary:
            ring = torch.zeros(S * T * t.shape[0] * t.shape[1] * t.shape[2], dtype=torch.float32, device='cuda')
            self._rings.append(ring)
            entries.append(_ffi.dh_clip_window(self._frame.view(t), self._clip.view(t), ring.data_ptr()))
        table = (_ffi.dh_clip_window * len(entries))(*entries)
        self._table = torch.from_numpy(np.frombuffer(bytearray(table), np.uint8).copy()).cuda()
        self._counter = torch.zeros(2, dtype=torch.int32, device='cuda')
        self._window = (_ffi.lib().dh_clip_window_f32, full._ctx.handle, C.c_void_p(self._table.data_ptr()),
                        len(entries), S, T, C.c_void_p(self._counter.data_ptr()))
        self._count = np.zeros(S, np.int64)         # frames since the last reset, per stream
        self._graph, self._uses = None, 0

    # ---- public --------------------------------------------------------------------------------------------------
    def reset(self, ids=None):
        """Start new videos on streams `ids` (all if None): they are not ready until T more frames are pushed."""
        if ids is None:
            self._count[:] = 0
        else:
            self._count[np.asarray(ids, np.int64)] = 0

    @property
    def ready(self):
        return self._count >= self.frames_per_clip

    def push(self, frames):
        """frames: float32 CUDA tensor (S, H, W, 3), one new frame per stream (what FramePipeline returns and
        forward_device takes).  Advances every stream by one frame.  -> StreamOutputs."""
        m, S = self.model, self.n_streams
        torch = m._torch()
        if m._dev is not self._weights:
            raise RuntimeError('the model\'s weights were replaced after this ClipStream was built: build a new one')
        t_in = m.graph.inputs[0]
        if tuple(frames.shape) != (S,) + tuple(t_in.shape):
            raise ValueError('frames have shape %s, expected %s (one frame per stream)'
                             % (tuple(frames.shape), (S,) + tuple(t_in.shape)))
        s = self.stages.frame.storage[t_in.id]
        self._frame.slots[s.buf.phys].copy_(frames.reshape(-1), non_blocking=True)
        self._graph, self._uses = _graphed(m.use_cuda_graph, self._graph, self._uses, self._issue)
        self._count += 1
        ready = self.ready
        frame_outs = [self._frame.tensor(t).reshape((S,) + _item_dims(t)) for t in self.frame_output_tensors]
        clip_outs = [self._clip.tensor(t).reshape((S,) + _item_dims(t)) for t in self.clip_output_tensors]
        if not ready.all():
            idx = torch.from_numpy(np.flatnonzero(~ready)).to(clip_outs[0].device) if clip_outs else None
            for o in clip_outs:
                o.index_fill_(0, idx, float('nan'))
        return StreamOutputs(frame_outs, clip_outs, ready.copy())

    def export(self, path):
        """Write this stream -- both stages as bound, the boundary table, the weights, the outputs -- to one file that
        the C ABI runs with no Python in the process (dh_stream_load / dh_stream_push, include/deephar_b200.h).  The
        rings, ring position and counts are not recorded: a loaded stream starts with no stream ready.  Neither this
        stream's state nor the model's bound batch sizes change."""
        from . import export
        export.write_stream(self, str(path))

    def launches_per_push(self):
        """Kernel launches one push issues: frame stage + window + clip stage."""
        return self._frame.kernels + 1 + self._clip.kernels

    # ---- engine --------------------------------------------------------------------------------------------------
    def _issue(self, stream_ptr):
        self._frame.issue(stream_ptr)
        rc = self._window[0](*self._window[1:], stream_ptr)
        if rc != 0:
            _ffi.check(rc, 'dh_clip_window_f32')
        self._clip.issue(stream_ptr)
