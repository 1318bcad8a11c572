"""Device-resident stream buffer with the reference ring buffer's framing semantics.

``RingBuffer.data_indexed(end_index, length)`` returns the ``length`` samples that END at
``end_index`` (friture/ringbuffer.py:87-99) and the widgets advance ``old_index`` by the hop per
column (friture/spectrogram.py:131-159, friture/spectrum.py:125-155, friture/delay_estimator.py:
104-126).  ``StreamFramer`` keeps, for many channels at once, exactly the samples those frames can
still need -- the last ``frame_len`` samples before ``old_index`` (zeros before the stream starts,
like the reference's zero-initialised buffer, ringbuffer.py:36) plus everything newer -- in one
contiguous tensor, so a tick's frames are ``x[:, f*hop : f*hop + frame_len]`` of the returned view
and can be handed to the batched kernels without copies.  With ``history`` it keeps that many
samples before ``old_index`` instead, so that ``set_geometry`` can lengthen the frame in mid-stream
up to ``history`` and still frame what the reference's ring buffer would (friture/spectrogram.py:
setfftsize changes the frame length and keeps ``old_index``).  Works on any torch device (CUDA in the
product, CPU in the host-logic tests).
"""
from __future__ import annotations

from math import floor


class StreamFramer:
    def __init__(self, n_channels, frame_len, hop, device, capacity=None, pre_increment=False, history=None):
        import torch
        self.n_channels = int(n_channels)
        self.frame_len = int(frame_len)
        self.hop = int(hop)
        # samples kept before old_index: the longest frame set_geometry may switch to
        self.history = int(history) if history is not None else self.frame_len
        if self.history < self.frame_len:
            raise ValueError("history must be >= frame_len")
        # spectrum / spectrogram use the frame ending at old_index, then advance (post-increment);
        # the delay estimator advances first (delay_estimator.py:122-126)
        self.pre_increment = bool(pre_increment)
        self.capacity = max(int(capacity or (4 * self.history + 64 * self.hop)), self.history)
        self.buf = torch.zeros((self.n_channels, self.capacity), dtype=torch.float32, device=device)
        self.offset = 0                 # total samples pushed (RingBuffer.offset)
        self.old_index = 0              # the widget's old_index
        self._base = -self.history      # stream index of buf[:, 0]
        self._fill = self.history       # valid samples in buf (starts with history zeros)

    def push(self, chunk):
        """Append chunk [C, n] (friture/ringbuffer.py:39-61)."""
        n = chunk.shape[1]
        if chunk.shape[0] != self.n_channels:
            raise ValueError("expected %d channels" % self.n_channels)
        if self._fill + n > self.capacity:
            self._compact(n)
        self.buf[:, self._fill:self._fill + n] = chunk
        self._fill += n
        self.offset += n

    def _compact(self, incoming):
        import torch
        keep_from = self.old_index - self.history - self._base       # oldest sample still needed
        keep = self._fill - keep_from
        if keep + incoming > self.capacity:
            new_cap = max(2 * self.capacity, keep + incoming)
            nb = torch.zeros((self.n_channels, new_cap), dtype=self.buf.dtype, device=self.buf.device)
            nb[:, :keep] = self.buf[:, keep_from:self._fill]
            self.buf = nb
            self.capacity = new_cap
        else:
            self.buf[:, :keep] = self.buf[:, keep_from:self._fill].clone()
        self._base += keep_from
        self._fill = keep

    def set_geometry(self, frame_len, hop):
        """New frame length and hop from the next ``take`` on; ``old_index`` and the samples pushed
        so far are kept, so the next frame is the new ``frame_len`` samples ending where the old
        framing stopped.  frame_len may not exceed ``history``."""
        frame_len, hop = int(frame_len), int(hop)
        if frame_len > self.history:
            raise ValueError("frame_len %d exceeds the %d samples of history kept" % (frame_len, self.history))
        if frame_len < 1 or hop < 1:
            raise ValueError("frame_len and hop must be >= 1")
        self.frame_len, self.hop = frame_len, hop

    def realizable(self):
        """Frames the widget would compute now: floor(available / hop) (spectrogram.py:135-145)."""
        available = self.offset - self.old_index
        return int(floor(available / self.hop)) if available > 0 else 0

    def take(self):
        """(view, n_frames): frame f of this tick is view[:, f*hop : f*hop + frame_len]; advances
        old_index by n_frames * hop.  n_frames may be 0 (view is then None)."""
        r = self.realizable()
        if r == 0:
            return None, 0
        first_end = self.old_index + (self.hop if self.pre_increment else 0)
        start = first_end - self.frame_len - self._base
        stop = start + self.frame_len + (r - 1) * self.hop
        self.old_index += r * self.hop
        return self.buf[:, start:stop], r
