"""The streaming Griffin-Lim workspace restated (csrc/vocoder_stream.cu, GlLayout): the FFT tables, then one slot per stream, each a 256-byte
header {committed, admitted, frames, carry} followed by the overlap-add ring c, the estimate ring x and the magnitude ring S, every region
256-aligned.  Rings, in the kernel's conventions:
  c[z mod N]               committed overlap-add at sample z of the untrimmed signal
  x[(j mod A) N + n]       windowed estimate w x_j of frame j of the look-ahead set, A = lookahead + 1
  S[(j mod A) K + k]       magnitude of frame j, K = N/2 + 1
Readers and writers work on a host copy of the workspace bytes (numpy uint8), one slot at a time."""
from dataclasses import dataclass

import numpy as np

MAX_LOOKAHEAD = 7                 # B200TTS_GL_STREAM_MAX_LOOKAHEAD
MAX_A = MAX_LOOKAHEAD + 1         # GL_MAX_A: the FFT buffers hold this many frames whatever the look-ahead
MAX_SLOTS = 64
MAX_SMEM = 227 * 1024             # sm_90 opt-in dynamic shared memory per block
HEADER = 256


def _up(x, a=256):
    return -(-x // a) * a


def plan_ok(N):
    """make_plan: even N <= 2048 whose half has no prime factor above 31."""
    if N < 2 or N > 2048 or N % 2:
        return False
    m = N // 2
    for q in (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31):
        while m % q == 0:
            m //= q
    return m == 1


@dataclass(frozen=True)
class GlLayout:
    N: int
    lookahead: int
    slots: int = 1

    @property
    def M(self):
        return self.N // 2

    @property
    def K(self):
        return self.N // 2 + 1

    @property
    def A(self):
        return self.lookahead + 1

    @property
    def twM(self):
        return 0

    @property
    def twN(self):
        return _up(8 * self.M)

    @property
    def window(self):
        return _up(self.twN + 8 * self.K)

    @property
    def slots_at(self):
        return _up(self.window + 4 * self.N)

    c = HEADER

    @property
    def x(self):
        return _up(self.c + 4 * self.N)

    @property
    def S(self):
        return _up(self.x + 4 * self.A * self.N)

    @property
    def slot_bytes(self):
        return _up(self.S + 4 * self.A * self.K)

    @property
    def bytes(self):
        return self.slots_at + self.slots * self.slot_bytes

    @property
    def smem(self):
        """Dynamic shared memory of gl_stream_run_kernel: FFT tables and 2 GL_MAX_A frame buffers (fft_smem_bytes), then c, x and S."""
        M = self.M
        fft = (M + (M + 1) + 2 * MAX_A * (M + 1)) * 8 + 4 * self.N
        return _up(fft, 16) + 4 * (self.N + self.A * self.N + self.A * self.K)

    def slot_base(self, slot):
        return self.slots_at + slot * self.slot_bytes


def accepted(N, hop, win, lookahead):
    """gl_stream_validate's shape conditions (iters, slots and preemphasis aside)."""
    return (plan_ok(N) and 1 <= win <= N and 1 <= hop <= win and 0 <= lookahead <= MAX_LOOKAHEAD and (lookahead >= 1 or 2 * hop <= N)
            and GlLayout(N, lookahead).smem <= MAX_SMEM)


def max_frames(N, hop):
    """The longest stream gl_stream_run accepts: hop * frames + 2 N < 2^31."""
    return (2 ** 31 - 1 - 2 * N) // hop


@dataclass
class Slot:
    committed: int
    admitted: int
    frames: int
    carry: np.float32
    c: np.ndarray       # [N]
    x: np.ndarray       # [A, N]
    S: np.ndarray       # [A, K]


def _f32(buf, off, n):
    return buf[off:off + 4 * n].view(np.float32)


def read_slot(buf, lay, slot):
    """Slot `slot` of the workspace bytes `buf` (numpy uint8, a copy) -> Slot of float32 arrays (copies)."""
    b = lay.slot_base(slot)
    hdr = buf[b:b + 16].view(np.int32)
    carry = buf[b + 12:b + 16].view(np.float32)[0]
    return Slot(int(hdr[0]), int(hdr[1]), int(hdr[2]), np.float32(carry), _f32(buf, b + lay.c, lay.N).copy(),
                _f32(buf, b + lay.x, lay.A * lay.N).reshape(lay.A, lay.N).copy(), _f32(buf, b + lay.S, lay.A * lay.K).reshape(lay.A, lay.K).copy())


def write_slot(buf, lay, slot, st):
    """Writes Slot `st` (cast to float32) into slot `slot` of `buf` in place; the rest of the header's 256 bytes is left as it is."""
    b = lay.slot_base(slot)
    buf[b:b + 12].view(np.int32)[:] = (st.committed, st.admitted, st.frames)
    buf[b + 12:b + 16].view(np.float32)[0] = np.float32(st.carry)
    _f32(buf, b + lay.c, lay.N)[:] = np.asarray(st.c, np.float32)
    _f32(buf, b + lay.x, lay.A * lay.N)[:] = np.asarray(st.x, np.float32).reshape(-1)
    _f32(buf, b + lay.S, lay.A * lay.K)[:] = np.asarray(st.S, np.float32).reshape(-1)


def read_tables(buf, lay):
    """(W_M [M] complex64, W_N [K] complex64, window [N] float32) as the reset wrote them."""
    twM = buf[lay.twM:lay.twM + 8 * lay.M].view(np.complex64).copy()
    twN = buf[lay.twN:lay.twN + 8 * lay.K].view(np.complex64).copy()
    return twM, twN, _f32(buf, lay.window, lay.N).copy()


def empty_slot(lay):
    return Slot(0, 0, 0, np.float32(0), np.zeros(lay.N, np.float32), np.zeros((lay.A, lay.N), np.float32), np.zeros((lay.A, lay.K), np.float32))
