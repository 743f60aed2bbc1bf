"""Which conversion kernel the batch group runs for a block: a mirror of launch_convert's rule
(sdr-server_b200/csrc/xlating_group.cu), so that a test can prove its schedule reaches each of them.

The Q15 path always runs convert_q15_kernel.  The float path runs the vectorised kernel, which loads two
complex samples at a time, when the block has an even number n of complex samples, starts at an even stream
position S and its raw pointer is aligned to two samples (4 bytes for cu8 and cs8, 8 for cs16); otherwise
the scalar kernel.  Host blocks are read from the group's own staging buffer, which is aligned, so only a
device block's own address counts.  numpy-free, no GPU."""

SAMPLE_BYTES = {"cu8": 2, "cs8": 2, "cs16": 4}
VEC, SCALAR, Q15 = "vec", "scalar", "q15"


def conv_kind(fmt, q15, n, S, ptr=None):
    """The kernel that converts n complex samples at stream position S (on the block's path) read from ptr
    (None: the group's aligned staging buffer)."""
    if q15:
        return Q15
    pair = 2 * SAMPLE_BYTES[fmt]
    aligned = ptr is None or ptr % pair == 0
    return VEC if n % 2 == 0 and S % 2 == 0 and aligned else SCALAR


def device_offsets(fmt, offsets=(0, 2, 4, 8)):
    """The byte offsets of `offsets` at which a device block of fmt is aligned to one complex sample (the
    others are refused)."""
    return [o for o in offsets if o % SAMPLE_BYTES[fmt] == 0]
