"""TEST INFRASTRUCTURE ONLY — CPU restatement of the reference's final mix, `combine_audio` (src/main.py:229-233):

    main   = AudioSegment.from_wav(ai_vocals_mixed) - 4 + main_gain
    backup = AudioSegment.from_wav(backup_vocals)   - 6 + backup_gain
    inst   = AudioSegment.from_wav(instrumental)    - 7 + inst_gain
    main.overlay(backup).overlay(inst).export(path, format=...)

`pydub==0.25.1` (requirements.txt:12) is a third-party dependency that is absent from the reference repository.
Its sample arithmetic is CPython's `audioop` C module, which IS in this image (Python 3.12 stdlib) and is called here
directly, so every sample operation (`mul`, `ratecv`, `tostereo`, `add`) is the reference's own code: PINNED.  The glue around
it is restated from pydub's published source (audio_segment.py: `apply_gain`, `_sync`, `set_channels`, `set_frame_rate`,
`__getitem__`, `overlay`): PARITY OF THE GLUE UNPINNED (restated, not executed):

  seg - x            -> apply_gain(-x) = audioop.mul(data, width, 10 ** (-x / 20));  seg + x -> apply_gain(x)   (two muls)
  overlay(other)     -> seg1, seg2 = _sync(self, other): both to max(channels), max(frame_rate), max(sample_width):
                          set_channels (mono -> stereo: audioop.tostereo(data, width, 1, 1)), then
                          set_frame_rate (audioop.ratecv(data, width, channels, rate, new_rate, None)), then width
                        output = seg1[:0] + add(seg1[0:][:len2], seg2[:len1]) + rest of seg1[0:]
                        where the MILLISECOND slice seg1[0:] keeps int(len_ms * rate / 1000) frames, len_ms =
                        round(1000 * frames / rate) — a few frames are dropped, or up to 2 ms of silence appended
  export(wav)        -> the int16 frames as they are

Inputs/outputs are int16 arrays as `scipy.io.wavfile.read` returns them ([n] mono or [n, channels])."""
from __future__ import annotations

import warnings
from typing import Tuple

import numpy as np

with warnings.catch_warnings():
    warnings.simplefilter("ignore", DeprecationWarning)
    import audioop                                     # CPython's Modules/audioop.c — what pydub calls

WIDTH = 2


def db_to_float(db: float) -> float:
    """pydub.utils.db_to_float(db, using_amplitude=True)."""
    return 10 ** (float(db) / 20)


class Segment:
    """The part of pydub.AudioSegment the mix uses: raw int16 bytes + channels + frame rate."""

    def __init__(self, data: bytes, channels: int, frame_rate: int):
        self.data, self.channels, self.frame_rate = data, int(channels), int(frame_rate)

    @classmethod
    def from_array(cls, x: np.ndarray, frame_rate: int) -> "Segment":
        x = np.ascontiguousarray(x, dtype=np.int16)
        return cls(x.tobytes(), 1 if x.ndim == 1 else x.shape[1], frame_rate)

    def to_array(self) -> np.ndarray:
        a = np.frombuffer(self.data, dtype=np.int16)
        return a.copy() if self.channels == 1 else a.reshape(-1, self.channels).copy()

    @property
    def frame_width(self) -> int:
        return self.channels * WIDTH

    def frame_count(self, ms=None) -> float:
        if ms is not None:
            return ms * (self.frame_rate / 1000.0)
        return float(len(self.data) // self.frame_width)

    def __len__(self) -> int:                       # milliseconds
        return round(1000 * (self.frame_count() / self.frame_rate))

    def _spawn(self, data: bytes) -> "Segment":
        return Segment(data, self.channels, self.frame_rate)

    def apply_gain(self, db: float) -> "Segment":
        return self._spawn(audioop.mul(self.data, WIDTH, db_to_float(float(db))))

    def set_channels(self, channels: int) -> "Segment":
        if channels == self.channels:
            return self
        if channels == 2 and self.channels == 1:
            return Segment(audioop.tostereo(self.data, WIDTH, 1, 1), 2, self.frame_rate)
        raise NotImplementedError("the mix only ever widens mono to stereo")

    def set_frame_rate(self, frame_rate: int) -> "Segment":
        if frame_rate == self.frame_rate:
            return self
        if self.data:
            conv, _ = audioop.ratecv(self.data, WIDTH, self.channels, self.frame_rate, frame_rate, None)
        else:
            conv = self.data
        return Segment(conv, self.channels, frame_rate)

    def ms_slice(self, start_ms: int, end_ms=None) -> "Segment":
        """AudioSegment.__getitem__(slice) in milliseconds, with the missing-frame silence fill."""
        end_ms = len(self) if end_ms is None else end_ms
        start_ms, end_ms = min(start_ms, len(self)), min(end_ms, len(self))
        start = int(self.frame_count(ms=start_ms)) * self.frame_width
        end = int(self.frame_count(ms=end_ms)) * self.frame_width
        data = self.data[start:end]
        missing = (end - start - len(data)) // self.frame_width
        if missing:
            if missing > self.frame_count(ms=2):
                raise ValueError("TooManyMissingFrames")
            data += audioop.mul(data[:self.frame_width], WIDTH, 0) * missing
        return self._spawn(data)

    def overlay(self, other: "Segment") -> "Segment":
        """AudioSegment.overlay(seg, position=0, loop=False, times=None, gain_during_overlay=None)."""
        channels = max(self.channels, other.channels)
        rate = max(self.frame_rate, other.frame_rate)
        seg1 = self.set_channels(channels).set_frame_rate(rate)
        seg2 = other.set_channels(channels).set_frame_rate(rate)
        out = seg1.ms_slice(0, 0).data
        d1, d2 = seg1.ms_slice(0).data, seg2.data
        if len(d2) >= len(d1):
            d2 = d2[:len(d1)]
        out += audioop.add(d1[:len(d2)], d2, WIDTH)
        out += d1[len(d2):]
        return seg1._spawn(out)


def combine_audio(main: np.ndarray, sr_main: int, backup: np.ndarray, sr_backup: int, inst: np.ndarray, sr_inst: int,
                  main_gain: float = 0, backup_gain: float = 0, inst_gain: float = 0) -> Tuple[np.ndarray, int]:
    """main.py:229-233 up to the encoder: the int16 frames `export` hands to the WAV / mp3 writer, and their rate."""
    m = Segment.from_array(main, sr_main).apply_gain(-4).apply_gain(main_gain)
    b = Segment.from_array(backup, sr_backup).apply_gain(-6).apply_gain(backup_gain)
    i = Segment.from_array(inst, sr_inst).apply_gain(-7).apply_gain(inst_gain)
    out = m.overlay(b).overlay(i)
    return out.to_array(), out.frame_rate
