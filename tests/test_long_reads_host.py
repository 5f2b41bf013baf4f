"""Long reads through the device engine's state machine on the host (tests/parity_fuzz.run_case: bt2g_xengine_align_host over the C
oracle's entry-point table) against the unmodified reference program: fuzz configurations with their reads made 300, 424 and 512
bases long, and -X raised to 2000-8000 on paired ones.  This pins the state machine's long-read policy without a GPU: the reseed of
each end-to-end backtrace after the reference's u8 matrix gives way to the i16 one (minimum scores below -254, reads of 424 bases
and more), the gap limits of long reads and the room their op strings take.

The configurations are drawn by parity_fuzz.draw_case and overridden here, so that the draws of existing seeds keep their cases."""
import os

import pytest

import parity_fuzz

# (seed, case, read length, -X or None): unpaired end-to-end (.bt2 and .bt2l), unpaired local, paired end-to-end and local
CASES = [
    (11, 10, 512, None),        # --fast
    (11, 28, 424, None),        # --sensitive -L 25 -M 20
    (100, 24, 300, None),       # .bt2l --sensitive -R 1 --np 1 --rfg 8,1, Ns
    (11, 17, 300, None),        # --sensitive-local, Ns
    (11, 20, 300, 2000),        # paired --very-sensitive --dovetail --no-overlap --rdg 5,1
    (100, 0, 424, 8000),        # paired --very-sensitive -L 32 -R 0 -M 1
    (11, 31, 300, 4000),        # paired --fast-local
]


def _long(seed, k, read_len, maxfrag):
    c = parity_fuzz.draw_case(seed, k)
    c["read_len"] = read_len
    if maxfrag is not None:
        c["kw"]["pe"].maxfrag = maxfrag
        flags = c["flags"]
        if "-X" in flags:
            flags[flags.index("-X") + 1] = str(maxfrag)
        else:
            flags += ["-X", str(maxfrag)]
    return c


@pytest.mark.skipif(not os.path.exists(parity_fuzz.REF), reason="oracle/_ref is not built")
@pytest.mark.parametrize("seed,k,read_len,maxfrag", CASES)
def test_long_read_configurations_identical_to_reference(seed, k, read_len, maxfrag, tmp_path):
    c = _long(seed, k, read_len, maxfrag)
    assert c["paired"] == (maxfrag is not None)
    n, bad, first, st, desc = parity_fuzz.run_case(c, str(tmp_path), n_unpaired=120, n_pairs=60)
    assert n > 0 and bad == 0, (desc, first)
