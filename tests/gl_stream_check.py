"""One call of streaming Griffin-Lim (b200tts_gl_stream_run, csrc/vocoder_stream.cu) recomputed in fp64 from the slot state before it, with
an error bound for every element of the slot after it and of the samples it releases (DESIGN "Griffin-Lim vocoder", "Streaming").

one_call(before, new_S, row, shape, window) follows the kernel's loop: admit the frames up to m + k one at a time, run `iters` Jacobi passes
over the look-ahead set, commit frame m into the overlap-add ring, release and de-emphasise, for every ready frame; the rings keep the
kernel's ring conventions (tests/gl_stream_slot.py), so every ring entry, stale ones included, has an expected value.  `window` is the
kernel's own fp32 window table (or the fp64 window of the specification): its rounding is then no part of the bound.

Bounds, unit roundoff u = 2^-24, gamma(n) = n u / (1 - n u):
  * fill  p_j = (c + sum_q w x_q) / e: the sum of nt terms in fp32 is off by gamma(nt) sum |terms| plus the bounds of the terms; the
    one-sided envelope e is an fmaf chain of te terms, relative error gamma(te); one division and the window multiply add one rounding each.
    Where the fp64 e is exactly 0 the kernel writes an exact 0 (every window value there is 0).
  * projection  x_j = w irfft(S_j X / |X|), X = rfft(w p_j): the mixed-radix transform's error is bounded element by element from the
    plan's radices, not from log2 N.  Every output of a radix-R stage is a chain of 2R fmaf per real component with rounded twiddles, so
    along every path of the transform the product of the rounding factors is within gamma(sum_s (2 R_s + 1)) of 1; summed over the paths,
    whose twiddle components are at most 1 in magnitude and branch into real and imaginary parts at each of the S stages,
    |dX_k| <= sqrt(2) gamma(sum_s (2 R_s + 1)) 2^(S/2) sum |inputs|.  The even/odd split of the real transform adds 6 roundings of
    |Z_k| + |Z_{M-k}|.  The fill's bound enters linearly (|rfft(d)_k| <= ||d||_1).  The phase error of bin k is min(2, 2 |dX_k| / |X_k|),
    2 where X_k = 0 unless X_k is exactly 0 in both (then the phase is exactly 1).  The inverse: the exact sensitivity of irfft to
    dY plus the same path bound over the half-length inverse; then the 1/N scale and the window multiply.
  * chaining: an admitted frame's bound enters the next fill linearly; passes compound.
  * commit c += x_m is one fp32 add; release v / wss with wss an fmaf chain over frames 0..lf; de-emphasis y = fmaf(a, carry, v) by the
    recursion D_q = (D_v + |a| D_{q-1} + u |y_q|) / (1 - u).
Exact: the header counters, the S ring, every ring entry the call does not write, and the released entries of c (0).  exact_checks()
adds the bit-exact commit c_after = fl(c_before + x_m) from the kernel's own x_m and the few-ulp release fl(v / wss).

emulate_call() is the same call in fp32 in the kernel's order (fmaf chains, fp32 sums in ascending frame order, single-precision FFTs);
its `fault` argument plants one of FAULTS, for the tests that show each one fails its bound or an exact check."""
from dataclasses import dataclass, field

import numpy as np
import scipy.fft
import scipy.signal

from gl_stream_slot import Slot

U = 2.0 ** -24
TINY = float(np.finfo(np.float32).tiny)
INT_MAX = 2 ** 31 - 1
SQ2 = np.sqrt(2.0)

FAULTS = ('release_envelope_lf_plus_1', 'envelope_cut_at_F', 'commit_index_off_by_one_at_wrap', 'released_not_zeroed', 'gauss_seidel',
          'admission_includes_own_frame', 'phase_0_where_X_0', 'window_lpad_off_by_one', 'carry_reset_per_call', 'tail_release_frames_F_minus_2')


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U / (1 - n * U)


def fft_plan(lib, N):
    """The radices b200tts_vocoder_fft_plan reports for N (the plan of the half-length complex transform)."""
    import ctypes
    r = (ctypes.c_int * 12)()
    k = lib.b200tts_vocoder_fft_plan(N, r, 12)
    assert k > 0, N
    return tuple(r[:k])


@dataclass(frozen=True)
class Shape:
    N: int
    hop: int
    win: int
    lookahead: int
    iters: int
    a: float                      # de-emphasis coefficient, as the kernel receives it (fp32)
    radices: tuple

    @property
    def A(self):
        return self.lookahead + 1

    @property
    def M(self):
        return self.N // 2

    @property
    def K(self):
        return self.N // 2 + 1

    @property
    def fft_path_bound(self):
        """G: per real output component, the rounding of one half-length complex transform is at most G times the sum of |components|
        of its input."""
        return float(gamma(sum(2 * r + 1 for r in self.radices)) * 2.0 ** (len(self.radices) / 2))


@dataclass
class Expected:
    after: Slot                    # fp64 values in the kernel's ring layout
    cb: np.ndarray                 # bounds of after.c
    xb: np.ndarray                 # bounds of after.x
    carry_b: float
    out: np.ndarray                # released samples (after de-emphasis)
    out_b: np.ndarray
    x_stage: list                  # per ring frame: None (untouched), 'projection', 'chained' or 'admission'
    processed: list = field(default_factory=list)      # the frames the call commits


def _fmaf_sq(v, s):
    """fmaf(v, v, s) in fp32: the product is exact in fp64, then one rounding (two near a tie: an emulation only)."""
    return (v.astype(np.float64) * v + s).astype(np.float32)


class _Call:
    """The kernel's loop over one call, in fp64 with bounds (f32=False) or as the fp32 emulation (f32=True)."""

    def __init__(self, before, new_S, row, sh, window, f32=False, fault=None):
        self.sh, self.f32, self.fault = sh, f32, fault
        dt = np.float32 if f32 else np.float64
        self.dt = dt
        w = np.asarray(window, np.float64)
        if fault == 'window_lpad_off_by_one':
            w = np.roll(w, 1)
        self.w = w.astype(dt)
        self.c = before.c.astype(dt).copy()
        self.x = before.x.astype(dt).copy()
        self.S = before.S.astype(np.float32).copy()
        self.cb = np.zeros(sh.N)
        self.xb = np.zeros((sh.A, sh.N))
        self.x_stage = [None] * sh.A
        self.new_S = None if new_S is None else np.asarray(new_S, np.float32)
        self.F, self.ended = int(row[0]), bool(row[1])
        self.before = before

    # one-sided (last = INT_MAX) or partial window sum-square at the samples z, in ascending frame order; its number of terms
    def envelope(self, z, last):
        N, H = self.sh.N, self.sh.hop
        i0 = np.where(z - N + 1 <= 0, 0, (z - N + 1 + H - 1) // H)
        i1 = np.minimum(z // H, last)
        nt = np.maximum(i1 - i0 + 1, 0)
        s = np.zeros(len(z), self.dt)
        for t in range(int(nt.max()) if len(z) else 0):
            i = i0 + t
            ok = i <= i1
            d = np.where(ok, z - i * H, 0)
            v = self.w[d]
            if self.f32:
                s = np.where(ok, _fmaf_sq(v, s), s)
            else:
                s = np.where(ok, s + v * v, s)
        return s, nt

    def fill(self, j, m, upto):
        sh = self.sh
        N, H, A = sh.N, sh.hop, sh.A
        z = j * H + np.arange(N, dtype=np.int64)
        live = z < m * H + N
        ci = z % N
        acc = np.where(live, self.c[ci], 0).astype(self.dt)
        absum = np.abs(acc).astype(np.float64)
        accb = np.where(live, self.cb[ci], 0)
        nt = np.ones(N)
        for q in range(m, upto):
            d = z - q * H
            ok = (d >= 0) & (d < N)
            dd = np.where(ok, d, 0)
            xv = np.where(ok, self.x[q % A, dd], 0).astype(self.dt)
            acc = (acc + xv).astype(self.dt)
            if not self.f32:
                absum += np.abs(xv)
                accb += np.where(ok, self.xb[q % A, dd], 0)
                nt += ok
        last = self.F - 1 if self.fault == 'envelope_cut_at_F' else INT_MAX
        e, te = self.envelope(z, last)
        nz = e != 0
        p = np.where(nz, acc / np.where(nz, e, 1), 0).astype(self.dt)
        wp = (self.w * p).astype(self.dt)
        if self.f32:
            return wp, None
        ge = gamma(te)
        ds = gamma(nt) * (absum + accb) + accb
        ee = np.where(nz, e, 1)
        q = (ds + np.abs(acc) * ge) / (ee * (1 - ge))
        pb = q + U * (np.abs(p) + q)
        wpb = np.where(nz, self.w * pb + U * self.w * (np.abs(p) + pb), 0)
        return wp, wpb

    def project(self, j, wp, wpb):
        sh = self.sh
        N, M, A = sh.N, sh.M, sh.A
        Sj = self.S[j % A].astype(np.float64)
        if self.f32:
            X = scipy.fft.rfft(wp.astype(np.float32))
            mag = np.hypot(X.real, X.imag).astype(np.float32)
            zero = mag == 0
            one = 0 if self.fault == 'phase_0_where_X_0' else 1
            ph = np.where(zero, one, X / np.where(zero, 1, mag)).astype(np.complex64)
            Y = (self.S[j % A] * ph).astype(np.complex64)
            Y[0] = Y[0].real
            Y[M] = Y[M].real
            y = scipy.fft.irfft(Y, n=N).astype(np.float32)
            return (y * np.float32(1.0)).astype(np.float32) * self.w, None
        X = scipy.fft.rfft(wp)
        l1 = np.abs(wp).sum() + wpb.sum()
        G = sh.fft_path_bound
        Xb = (2 * SQ2 * G + 12 * U) * l1 + wpb.sum()
        mag = np.abs(X)
        pos = mag > 0
        ph = np.where(pos, X / np.where(pos, mag, 1), 1)
        phb = np.where(pos, np.minimum(2.0, 2 * Xb / np.where(pos, mag, 1)) + 8 * U, 2.0 if Xb > 0 else 0.0)
        Y = Sj * ph
        Yb = Sj * phb + 2 * U * Sj
        y = scipy.fft.irfft(Y, n=N)
        sens = (Yb[0] + Yb[M] + 2 * Yb[1:M].sum()) / N
        Yl1 = (np.abs(Y) + Yb).sum()
        yb = sens + (4 * SQ2 * G + 24 * U) * Yl1 / N
        x = self.w * y
        xb = self.w * yb + 3.01 * U * self.w * (np.abs(y) + yb)
        return x, xb

    def _set_x(self, j, x, xb, stage):
        A = self.sh.A
        self.x[j % A] = x
        if xb is not None:
            self.xb[j % A] = xb
        self.x_stage[j % A] = stage

    def run(self):
        sh, b = self.sh, self.before
        N, H, A, I = sh.N, sh.hop, sh.A, sh.iters
        F, ended, fr = self.F, self.ended, b.frames
        m, adm = b.committed, b.admitted
        carry = np.float64(0 if self.fault == 'carry_reset_per_call' else b.carry)
        carry_b = 0.0
        a = float(np.float32(sh.a))
        rel = max(0, m * H - N // 2)
        outs, outbs, processed = [], [], []
        admitted_here = False
        while True:
            process = m < F and (m + A - 1 < F or ended)
            tail = not process and ended and m == F and rel < H * (F - 1)
            if not process and not tail:
                break
            lf = m if process else F - 1
            base = lf * H
            if process:
                processed.append(m)
                last = min(m + A - 1, F - 1)
                it = 0
                while adm <= last or it < I:
                    admit = adm <= last
                    if admit and adm >= fr:
                        self.S[adm % A] = self.new_S[adm - fr]
                    if admit:
                        upto = adm + 1 if self.fault == 'admission_includes_own_frame' else adm
                        wp, wpb = self.fill(adm, m, upto)
                        self._set_x(adm, *self.project(adm, wp, wpb), 'admission')
                        admitted_here = True
                        adm += 1
                    else:
                        stage = 'chained' if admitted_here else 'projection'
                        if self.fault == 'gauss_seidel':
                            for j in range(m, adm):
                                self._set_x(j, *self.project(j, *self.fill(j, m, adm)), stage)
                        else:
                            filled = [(j, *self.fill(j, m, adm)) for j in range(m, adm)]
                            for j, wp, wpb in filled:
                                self._set_x(j, *self.project(j, wp, wpb), stage)
                        it += 1
                idx = (base + np.arange(N)) % N
                if self.fault == 'commit_index_off_by_one_at_wrap':
                    idx = np.where(base % N + np.arange(N) >= N, (idx + 1) % N, idx)
                xm = self.x[m % A]
                s = (self.c[idx] + xm).astype(self.dt)
                if not self.f32:
                    self.cb[idx] = self.cb[idx] + self.xb[m % A] + U * (np.abs(s) + self.cb[idx] + self.xb[m % A])
                self.c[idx] = s
            final = ended and lf == F - 1
            rel_end = H * (F - 1) if final else max(0, base + H - N // 2)
            if rel_end > rel:
                z = np.arange(rel, rel_end, dtype=np.int64) + N // 2
                v = self.c[z % N]
                lfe = lf
                if self.fault == 'release_envelope_lf_plus_1':
                    lfe = lf + 1
                if self.fault == 'tail_release_frames_F_minus_2' and not process:
                    lfe = F - 2
                wss, te = self.envelope(z, lfe)
                big = wss > TINY
                o = np.where(big, v / np.where(big, wss, 1), v).astype(self.dt)
                if self.f32:
                    y = np.empty(len(o), np.float32)
                    cr = np.float32(carry)
                    for qq in range(len(o)):
                        val = o[qq]
                        if a != 0:
                            val = np.float32(np.float64(a) * np.float64(cr) + np.float64(val))
                        cr = val
                        y[qq] = val
                    carry = cr
                    outs.append(y)
                else:
                    vb = self.cb[z % N]
                    ge = gamma(te)
                    ww = np.where(big, wss, 1)
                    qd = (vb + np.abs(v) * ge) / (ww * (1 - ge))
                    ob = np.where(big, qd + U * (np.abs(o) + qd), vb)
                    if a != 0:
                        y = scipy.signal.lfilter([1.0], [1.0, -a], o, zi=[a * carry])[0]
                        D = np.empty(len(o))
                        d = carry_b
                        for qq in range(len(o)):
                            d = (ob[qq] + abs(a) * d + U * abs(y[qq])) / (1 - U)
                            D[qq] = d
                        carry, carry_b = y[-1], D[-1]
                    else:
                        y, D = o, ob
                        carry, carry_b = o[-1], ob[-1]
                    outs.append(y)
                    outbs.append(D)
            if process and not final and self.fault != 'released_not_zeroed':
                idz = (base + np.arange(H)) % N
                self.c[idz] = 0
                self.cb[idz] = 0
            rel = max(rel, rel_end)
            if process:
                m += 1
        for j in range(max(adm, fr), F):
            self.S[j % A] = self.new_S[j - fr]
        cat = lambda xs, dt: np.concatenate(xs) if xs else np.zeros(0, dt)   # noqa: E731
        after = Slot(m, adm, F, carry if self.f32 else float(carry), self.c, self.x, self.S)
        if self.f32:
            after.carry = np.float32(carry)
            return after, cat(outs, np.float32)
        return Expected(after, self.cb, self.xb, float(carry_b), cat(outs, np.float64), cat(outbs, np.float64), self.x_stage, processed)


def one_call(before, new_S, row, shape, window):
    """Slot state `before` (Slot), the new frames' magnitudes new_S [F - frames, K] (or None), row = (F, ended) -> Expected in fp64."""
    return _Call(before, new_S, row, shape, window).run()


def emulate_call(before, new_S, row, shape, window, fault=None):
    """The same call in fp32 in the kernel's order -> (Slot after, released samples); `fault` one of FAULTS or None."""
    assert fault is None or fault in FAULTS, fault
    return _Call(before, new_S, row, shape, window, f32=True, fault=fault).run()


def _ratio(got, ref, bound):
    """|got - ref| / bound per element; inf where got is not finite, the bound is not finite, or the bound is 0 and they differ."""
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    with np.errstate(divide='ignore', invalid='ignore'):
        r = np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err == 0, 0.0, np.inf))
    r = np.where(np.isfinite(got) & np.isfinite(bound), r, np.inf)
    return r


def compare(exp, got_after, got_out, a0=True):
    """The kernel's slot after the call and released samples against Expected -> {stage: worst err / bound} (inf: an exact part differs,
    or a value or bound is not finite).  Stages: header, S ring, c ring (commit), x ring by how it was last written (projection, chained,
    admission), the released samples (release, or deemphasis when the call de-emphasises)."""
    e = exp.after
    worst = {}

    def put(name, r):
        r = np.asarray(r, np.float64)
        if r.size:
            worst[name] = max(worst.get(name, 0.0), float(r.max()))

    put('header', [0.0 if (got_after.committed, got_after.admitted, got_after.frames) == (e.committed, e.admitted, e.frames) else np.inf])
    put('S ring', [0.0 if np.array_equal(got_after.S, e.S) else np.inf])
    put('commit', _ratio(got_after.c, e.c, exp.cb))
    for f, stage in enumerate(exp.x_stage):
        put(stage or 'untouched', _ratio(got_after.x[f], e.x[f], exp.xb[f]))
    rel = 'release' if a0 else 'deemphasis'
    if len(got_out) != len(exp.out):
        put(rel, [np.inf])
    else:
        put(rel, _ratio(got_out, exp.out, exp.out_b))
    put(rel, _ratio([got_after.carry], np.array([e.carry], np.float64), np.array([exp.carry_b])))
    return worst


def exact_checks(before, got_after, got_out, row, shape, window, exp):
    """Bit-level checks from the kernel's own values, for a call that processes at most one frame (so its x_m is still in the ring):
    c_after = fl(c_before + x_m) where the frame was committed and 0 where it was released, every other c entry unchanged; with a = 0 each
    released sample within 2 ulp of fl(v / wss) from the committed fp32 value v.  -> list of failures."""
    sh = shape
    N, H, A = sh.N, sh.hop, sh.A
    F, ended = row
    a0 = float(np.float32(sh.a)) == 0.0
    fails = []

    def release_ulps(v, z, lf, got):
        wss, _ = _Call(before, None, row, sh, window, f32=True).envelope(z, lf)
        big = wss > TINY
        o = np.where(big, v / np.where(big, wss, 1), v).astype(np.float32)
        ulps = np.abs(got.view(np.int32).astype(np.int64) - o.view(np.int32).astype(np.int64))
        if ulps.max() > 2:
            fails.append(('release ulps', int(ulps.max())))

    # the final release leaves c as it is: its samples divide the kernel's own c after the call, whatever else the call did
    if a0 and ended and exp.processed and exp.processed[-1] == F - 1:
        r0 = max(0, (F - 1) * H - N // 2)
        n = H * (F - 1) - r0
        if 0 < n <= len(got_out):
            z = np.arange(r0, H * (F - 1), dtype=np.int64) + N // 2
            release_ulps(got_after.c[z % N], z, F - 1, got_out[len(got_out) - n:])
    if len(exp.processed) > 1:
        return fails
    c_mid = before.c.astype(np.float32).copy()
    zeroed = np.zeros(N, bool)
    if exp.processed:
        m = exp.processed[0]
        idx = (m * H + np.arange(N)) % N
        c_mid[idx] = (c_mid[idx] + got_after.x[m % A]).astype(np.float32)
        final = row[1] and m == row[0] - 1
        if not final:
            zeroed[(m * H + np.arange(H)) % N] = True
    want = np.where(zeroed, np.float32(0), c_mid)
    if not np.array_equal(got_after.c.view(np.uint32), want.view(np.uint32)):
        fails.append(('commit bits', int((got_after.c.view(np.uint32) != want.view(np.uint32)).sum())))
    if a0 and len(got_out):
        lf = exp.processed[0] if exp.processed else F - 1
        m0 = exp.processed[0] if exp.processed else before.committed
        rel = max(0, m0 * H - N // 2)
        z = np.arange(rel, rel + len(got_out), dtype=np.int64) + N // 2
        release_ulps(c_mid[z % N], z, lf, got_out)
    return fails


def deemphasis_ratio(v_a0, carry_before, a, got):
    """The kernel's de-emphasised samples against fp64 lfilter of its own a = 0 output from the same state: y_q = fmaf(a, y_{q-1}, v_q) is
    within D_q = (|a| D_{q-1} + u |y_q|) / (1 - u) of it -> worst ratio."""
    a = float(np.float32(a))
    v = np.asarray(v_a0, np.float64)
    if not len(v):
        return 0.0
    y = scipy.signal.lfilter([1.0], [1.0, -a], v, zi=[a * float(carry_before)])[0]
    D = np.empty(len(v))
    d = 0.0
    for q in range(len(v)):
        d = (abs(a) * d + U * abs(y[q])) / (1 - U)
        D[q] = d
    return float(_ratio(got, y, D).max())


def crafted_state(shape, window, m, kind, rng, admit=False):
    """A slot state that is one call away from a single step -> (before, new_S, row).  admit=False: committed m, admitted = frames =
    m + k + 1, not ended; with iters = 1 the call runs exactly one Jacobi pass over the A = k + 1 frames of the look-ahead set, with no
    admission, then commits frame m and releases.  admit=True: one frame short, delivered in the call, so it admits frame m + k first.
    kind: 'noise' (white rings, each frame at its own scale in 10^[-3, 3]), 'zero' (c and the live estimates exactly 0: every X is exactly
    0), 'tone' (estimates of a windowed cosine at an exact bin: most bins near 0) or 'tiny' (noise at 1e-30).  Stale ring frames hold large
    noise: a call that reads them is wrong."""
    N, H, A, K, k = shape.N, shape.hop, shape.A, shape.K, shape.lookahead
    w = np.asarray(window, np.float64)
    F = m + k + 1
    adm = F - 1 if admit else F
    scale = 1e-30 if kind == 'tiny' else 1.0
    c = np.zeros(N)
    if m >= 1 and kind in ('noise', 'tiny'):
        z = np.arange(m * H, (m - 1) * H + N)
        c[z % N] = scale * rng.standard_normal(len(z)) * 10 ** rng.uniform(-1, 1)
    x = 1e3 * rng.standard_normal((A, N))                               # stale
    for j in range(m, adm):
        if kind == 'zero':
            x[j % A] = 0
        elif kind == 'tone':
            x[j % A] = w * np.cos(2 * np.pi * (3 + j % 5) * np.arange(N) / N) * (0.5 + j % 3)
        else:
            x[j % A] = scale * w * rng.standard_normal(N) * 10 ** rng.uniform(-3, 3)
    S = rng.uniform(0, 1, (A, K)) * 10 ** rng.uniform(-2, 2, (A, 1))
    S[:, rng.integers(0, K, max(1, K // 16))] = 0
    before = Slot(m, adm, adm, np.float32(rng.standard_normal()), c.astype(np.float32), x.astype(np.float32), S.astype(np.float32))
    new_S = (rng.uniform(0, 1, (1, K)) * 10).astype(np.float32) if admit else None
    return before, new_S, (F, False)
