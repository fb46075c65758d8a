"""tests/test_gpu_g2_hash.py at reduced sizes on the CPU simulators of the library (the five-limb one for
a, a1, e, f, d159 and g149, the eight-limb one for the five wide type D sets), against the compiled
reference: the bit-exactness check of G2 hashing and decompression that needs no GPU."""
from tests import live_reference as L
from tests.test_live_reference_inputs import _run_gpu_file, _sim

FILE = "test_gpu_g2_hash.py"


def test_g2_hash_file_on_the_simulator(tmp_path):
    so = _sim(tmp_path, "make_host_sim.py")
    sel = " or ".join("%s_set" % s for s in ("a", "a1", "e", "f", "d159", "g149")) + " or reference_basis"
    _run_gpu_file(so, sel, 36, FILE)


def test_g2_hash_file_on_the_eight_limb_simulator(tmp_path):
    so = _sim(tmp_path, "make_host_sim_d_wide.py")
    _run_gpu_file(so, " or ".join("%s_set" % s for s in L.WIDE_D), 38, FILE)
