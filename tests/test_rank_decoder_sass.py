"""-m "not gpu": the rank decoder's counting epilogue (renet_decoder_rank and renet_decoder_rank_multi, EPI 6 of the packed
wgmma GEMM) is one instantiation and adds its counts with integer atomics only: no float RED / ATOM in its SASS, read from
the built library."""
import re

from test_deterministic_sass import FLOAT_ATOMIC, _matching, sass  # noqa: F401  (sass is a fixture)


def test_rank_epilogue_has_integer_atomics_only(sass):  # noqa: F811
    found = _matching(sass, r'umma_gemm_packed_kernel<\(bool\)0, \(int\)6>')
    assert len(found) == 1, sorted(found)
    for name, body in found.items():
        hits = [ln.strip() for ln in body.split('\n') if FLOAT_ATOMIC.search(ln)]
        assert not hits, '%s: %s' % (name, hits[:3])
        assert re.search(r'\b(RED|REDG|ATOM|ATOMG)\.E\.ADD', body), name            # the integer count adds are there
