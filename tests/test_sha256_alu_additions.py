"""CPU: the SHA-256 TMR kernels add the round constants K_t off the ALU pipe (DESIGN.md §5.0).

The segmented kernel is bound by ALU-pipe issue.  ptxas lowers `K_t + W_t` to VIADD, which issues beside the ALU pipe
(a VIADD + SHF stream runs at 0.97 warp instructions per clock, one pipe alone at 0.5), or to IADD3, which issues on it.
It picks between them by its own pipe balance, so a ptxas upgrade or a source change could move the additions onto the
ALU pipe without changing a result; the SASS of the embedded cubin is held here."""
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import sha_pipe_rates as spr  # noqa: E402
from mock_run import CUBIN  # noqa: E402

K = {0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
     0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
     0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
     0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
     0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
     0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
     0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
     0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2}

# per kernel: IADD3 against a K_t immediate at most, IADD3 in all at most (16 of them are the byte-wise vote).
# The injecting kernel's fault-round branches copy rounds, and ptxas puts 2 of its copies' K_t additions on IADD3.
BOUND = {"xmr_sha256_b64_seg_nc3_inj0": (0, 28), "xmr_sha256_b64_seg_nc3_inj1": (2, 75)}


def _k_immediates(fun):
    """opcode -> how many of its instructions carry a K_t immediate (SASS prints some as negative hex)"""
    out = {}
    for _, op, line in spr.sass_ops(CUBIN, fun):
        for m in re.finditer(r"(-?)0x([0-9a-f]+)\b", line.split(";")[0]):
            v = int(m.group(2), 16)
            if ((-v) & 0xFFFFFFFF if m.group(1) else v) in K:
                out[op] = out.get(op, 0) + 1
                break
    return out


@pytest.mark.parametrize("fun", sorted(BOUND))
def test_round_constants_are_added_off_the_alu_pipe(built_lib, fun):
    k_iadd3_max, iadd3_max = BOUND[fun]
    by_op = _k_immediates(fun)
    on_alu = sum(n for op, n in by_op.items() if spr.pipe_of(op) == "alu")
    assert on_alu <= k_iadd3_max, (fun, by_op)
    # block 1 adds each of the 64 K_t to a message word (block 2's K_t + W_t fold into immediates of other additions)
    assert by_op.get("VIADD", 0) >= 64, (fun, by_op)
    assert spr.histogram(spr.sass_ops(CUBIN, fun)).get("IADD3", 0) <= iadd3_max


def test_round_additions_read_the_one_from_a_uniform_register(built_lib):
    """add_imad's 1 sits in a uniform register, so each of the ~850 round and schedule IMADs reads two registers, not three.
    Held in a per-thread register (as when the padding block's IMADs share it), the kernel ran 9% slower."""
    fun = "xmr_sha256_b64_seg_nc3_inj0"
    mult = [re.split(r",\s*", line.split(op, 1)[1].split(";")[0])[2].strip()
            for _, op, line in spr.sass_ops(CUBIN, fun) if op == "IMAD"]
    on_ur = sum(1 for b in mult if b.startswith("UR"))
    assert on_ur >= 800, (on_ur, len(mult))


def test_viadd_counts_on_the_pipe_measured_for_it():
    assert spr.pipe_of("VIADD") == "other"
    assert spr.pipe_of_measured("VIADD", "imad") == "imad" and spr.pipe_of_measured("VIADD", "alu") == "alu"
    assert spr.pipe_of_measured("IADD3", "imad") == "alu" and spr.pipe_of_measured("IMAD.IADD", "alu") == "imad"
    rates = lambda all_: {"viadd_shf_1_1": {"warp_inst_per_clk_per_smsp": {"all": all_}}}
    assert spr.viadd_pipe(rates(0.970)) == "imad" and spr.viadd_pipe(rates(0.50)) == "alu"
