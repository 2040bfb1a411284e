"""CPU: the emitter's printf-free "%.2f" (round-half-even on the exact binary value) against libc on 40M+ floats."""
import subprocess

import cases


def test_put_f2_matches_printf():
    p = subprocess.run([cases.check_program("fmt_check")], capture_output=True, text=True)
    assert p.returncode == 0, p.stdout[-2000:]
    assert "0 mismatches" in p.stdout
