"""Helpers of the long-stream tests: a group fed past 2^31 and 2^32 input samples, checked on windows.

A client's output depends on its last history samples and the current block, not on the absolute stream
position.  Take a client attached at position A whose window phase repeats every p input samples (its
period: D for an integer client, M for a rational L/M one, D1 * D2 or D1 * M2 for a cascade, D1 times the
member's period in sub-band samples for a sub-band member, and a multiple of 2 * D1 for a bank channel, the
period of its twiddle offset r0).  At exact stimuli and centre 0 (the oscillator stays at 1 + 0i) its outputs
in every block after a block boundary B with (B - A) = 0 (mod p) equal those of a fresh client attached at B
and fed the same blocks, from the first block whose windows all start at or after B.  So the float64
reference of a fresh client, fed a few blocks, checks a client that has run for 2^32 samples.

* N: one block length that every period used divides.
* Pump: feeds a group XLG_INPUT_DEVICE blocks cut from a few device buffers filled once, in a seeded order,
  with XLG_SLOTS tickets in flight, and reads outputs only of the blocks it is told to watch.
* window_start: the boundary B for a checked range.

numpy only; the pump takes the torch module and the group from its caller.
"""
import numpy as np

# 2^10 * 3^3 * 5 * 7: divisible by every period the tests use (8, 21, 42, 60, 128, 160, 640, 945, 1280, and
# 32 * 16 and 32 * 40 for sub-band members); 2^31 is reached after 2220 blocks, 2^32 after 4439
N = 2 ** 10 * 3 ** 3 * 5 * 7
SLOTS = 4  # XLG_SLOTS


def window_start(starts, c0, attach, period, hist):
    """The index b of the latest block boundary at or before block c0 with (starts[b] - attach) = 0 (mod
    period) and starts[c0] - starts[b] >= hist (hist: how many input samples before a window's end the client
    reads, stages before it included), or the attach block itself.  starts[i] is the stream position of block
    i; attach is a position in starts.  A fresh client fed blocks b, b+1, ... then produces the outputs of
    blocks c0, c0+1, ... of the client attached at `attach`."""
    a = starts.index(attach)
    for b in range(c0, a - 1, -1):
        if b == a or ((starts[b] - attach) % period == 0 and starts[c0] - starts[b] >= hist):
            return b
    raise AssertionError("no boundary")  # unreachable: b == a ends the loop


class Pump:
    """Feeds group g blocks of raw `fmt` elements from device buffers (a torch CUDA tensor of the stacked host
    buffers `bufs`), XLG_INPUT_DEVICE, SLOTS tickets in flight.

    feed(k, off, n) submits n complex samples of buffer k from sample off on; the block's host copy is
    blocks[i] and its stream position starts[i].  Blocks whose index is in `watch` are handed, once waited
    for, to read(ticket, index), which must copy their outputs before the ticket is recycled."""

    def __init__(self, torch, pkg, g, fmt, bufs, seed, flags=0, read=None):
        self.pkg, self.g, self.fmt, self.flags = pkg, g, fmt, flags | pkg.XLG_INPUT_DEVICE
        self.code = pkg.FMT[fmt]
        self.host = np.stack(bufs)
        self.dev = torch.from_numpy(self.host.view(np.uint8).reshape(len(bufs), -1).copy()).cuda()
        torch.cuda.current_stream().synchronize()
        self.item = self.host.itemsize * 2  # bytes per complex sample
        self.rng = np.random.default_rng(seed)
        self.read = read
        self.watch = set()
        self.pending = []  # (ticket, block index)
        self.blocks, self.starts = [], [0]

    def feed(self, k=None, off=0, n=None):
        """Submit one block (buffer k, or a seeded choice); returns its index."""
        k = int(self.rng.integers(0, len(self.host))) if k is None else k
        n = self.host.shape[1] // 2 - off if n is None else n
        ptr = self.dev.data_ptr() + k * self.dev.stride(0) + off * self.item
        t = self.g.submit_ptr(self.code, ptr, 2 * n, self.flags)  # (raw elements: two per complex sample)
        i = len(self.blocks)
        self.blocks.append(self.host[k, 2 * off:2 * (off + n)])
        self.starts.append(self.starts[-1] + n)
        self.pending.append((t, i))
        if len(self.pending) >= SLOTS:
            self._retire()
        return i

    def pair(self, a):
        """A ragged pair: the first a and the other N - a samples of one buffer, as two blocks.  Returns the
        index of the first."""
        k = int(self.rng.integers(0, len(self.host)))
        i = self.feed(k, 0, a)
        self.feed(k, a, N - a)
        return i

    def _retire(self):
        t, i = self.pending.pop(0)
        self.g.wait(t)
        if i in self.watch and self.read is not None:
            self.read(t, i)

    def drain(self):
        while self.pending:
            self._retire()

    def run_to(self, pos):
        """Full blocks until the next block would start past pos."""
        while self.starts[-1] + N <= pos:
            self.feed()

    @property
    def S(self):
        return self.starts[-1]


# ---------------------------------------------------------------------------
# fresh references, one per kernel family (centre 0, exact stimuli)
# ---------------------------------------------------------------------------
# A client spec is a tuple:
#   ("int", D, taps)                    an integer client (ref_f64)
#   ("q15", D, taps)                    an integer client on the Q15 path (ref_q15)
#   ("rat", L, M, taps)                 a rational client (ref_rational_f64)
#   ("casc", d1, taps1, l2, d2, taps2)  a cascade (f64_composition; l2 = 1 for an integer one)
#   ("sub", d1, taps1, l2, d2, taps2)   a member at offset 0 of a centre-0 sub-band (f64_rows + f64_member)
#   ("bank", d1, taps1, k, d2, taps2)   a member at offset 0 of channel k of a bank (bank_member_model)
def period(spec):
    """Input samples after which the spec's window phase repeats."""
    kind = spec[0]
    if kind in ("int", "q15"):
        return spec[1]
    if kind == "rat":
        return spec[2]
    if kind in ("casc", "sub"):
        return spec[1] * spec[4]
    d1, d2 = spec[1], spec[4]
    return int(np.lcm(2 * d1, d1 * d2))


def history(spec):
    """An upper bound of the input samples a window reads before its end, through every stage."""
    kind = spec[0]
    if kind in ("int", "q15"):
        return len(spec[2])
    if kind == "rat":
        return len(spec[3]) // spec[1] + 2
    d1, t1, t2 = spec[1], len(spec[2]), len(spec[5])
    return t1 + d1 * (t2 + 2)


def fresh_refs(specs, fmt, fs, blocks, mat=0):
    """Outputs per block of fresh clients `specs` attached before blocks[0] (bank channels materialised before
    blocks[mat]).  Integer clients of one shape share one matrix product."""
    from bank_exact import bank_member_model
    from cascade_rational import f64_composition
    from exact import ref_f64_many, ref_q15, to_complex
    from rational import ref_rational_f64
    from subband_exact import f64_member, f64_rows

    out = [None] * len(specs)
    shapes = {}
    for i, s in enumerate(specs):
        if s[0] == "int":
            shapes.setdefault((s[1], len(s[2])), []).append(i)
    for (D, _), idx in shapes.items():
        for i, y in zip(idx, ref_f64_many([specs[i][2] for i in idx], D, fmt, blocks)):
            out[i] = y
    xs = None
    for i, s in enumerate(specs):
        kind = s[0]
        if kind == "q15":
            out[i] = ref_q15(s[2], s[1], fmt, blocks)
        elif kind == "rat":
            out[i] = ref_rational_f64(s[3], s[1], s[2], fmt, blocks)
        elif kind == "casc":
            y = f64_composition(s[1], s[2], s[3], s[4], s[5], fs, [to_complex(fmt, b) for b in blocks])
            out[i] = [v.astype(np.complex64) for v in y]
        elif kind == "sub":
            out[i] = f64_member(f64_rows(s[1], s[2], fs, fmt, blocks), s[3], s[4], s[5], fs // s[1])
        elif kind == "bank":
            if xs is None:
                xs = np.concatenate([to_complex(fmt, b) for b in blocks]).astype(np.complex64)
            sizes = [np.asarray(b).size // 2 for b in blocks]
            out[i] = bank_member_model(s[2], s[1], s[3], xs, 0, sizes, [(1, s[4], s[5], 0)], fs, mat=mat)[0]
    return out
