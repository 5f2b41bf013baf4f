"""GPU: fixed cases of tests/parity_fuzz.py on the device engine itself (bt2g_xengine_align / _align_k over the CUDA kernels, at the
engine's own op-row width): random genome / reads / preset and option sets, every SAM record identical to the unmodified reference
program's (oracle/_ref).  Together the cases take every scoring option (--mp, --np, --rdg, --rfg, --ma, --score-min, --n-ceil),
local and end-to-end, paired and unpaired, a .bt2l index, -M, -k and -a, the dense SA and a 12-mer seed table beside -L 10."""
import os

import pytest

import parity_fuzz

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900),
              pytest.mark.skipif(not os.path.exists(parity_fuzz.REF), reason="oracle/_ref is not built")]

CASES = [
    # 101/13: --local --ma 3 --rdg 3,1: op strings longer than read length + 64 (the host build of the fuzz needs wider rows; the
    # device engine sizes its own from the scoring)
    (101, [13]),
    # 7/6: 250 bp, --rdg 3,1 --mp 6,1, -L 10 beside the seed table; 7/34: -L 10, --ma 1, paired -M 3; 7/88: paired local -a (dense SA);
    # 7/138: .bt2l paired --mp --np --score-min --no-mixed; 7/170: paired local --ff -M; 7/293: -k with --n-ceil and --score-min
    (7, [6, 34, 88, 138, 170, 293]),
    # 21/1: .bt2l paired --nofw --ff -M 20 with the dense SA; 21/4: paired --nofw --no-mixed --no-discordant: the seed wave searched
    # both strands whatever --nofw / --norc said
    (21, [1, 4]),
]
SEEN = set()


@pytest.fixture(scope="module", autouse=True)
def _cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


@pytest.mark.parametrize("seed,cases", CASES, ids=[f"seed{s}" for s, _ in CASES])
def test_device_engine_identical_to_reference(seed, cases, tmp_path):
    for k in cases:
        c = parity_fuzz.draw_case(seed, k)
        n, bad, first, st, desc = parity_fuzz.run_case(c, str(tmp_path), device=True)
        print(f"case {seed}/{k}: {desc}: {n} records; {st[1]} of {st[0]} units finished by the coroutine engine")
        assert bad == 0, (k, desc, first)
        SEEN.update(c["flags"])
        SEEN.update(f for f, on in (("local", c["local"]), ("end-to-end", not c["local"]), ("paired", c["paired"]), ("unpaired", not c["paired"]),
                                    (".bt2l", c["large"]), ("dense-SA", c["dense_sa"]), ("seed-table", c["seed_table"])) if on)


def test_zz_every_option_ran():
    """the end of the file: the cases above took every scoring option and reporting mode"""
    want = {"--mp", "--np", "--rdg", "--rfg", "--ma", "--score-min", "--n-ceil", "-M", "-k", "-a", "-L", "local", "end-to-end", "paired",
            "unpaired", ".bt2l", "dense-SA", "seed-table"}
    assert want <= SEEN, sorted(want - SEEN)
