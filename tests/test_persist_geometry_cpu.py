"""The plan of the persistent decoder loops against what their launchers take, and every loop geometry the plan produces against the
step-checked representatives of persist_geometry.py (host-only queries, no GPU).

The enumeration covers every decoder width D that is a multiple of 64 up to 2048, memory dims 256, 288, 292, 384 and 512, batches on
both sides of the 16-, 32- and 64-utterance limits, and text lengths L = 16k and 16k + 1 (both sides of every 16-position tile step of
the shared-memory carve-up) until the forward loops refuse, in evaluation and in training."""
import ctypes

import pytest

import persist_geometry as G

NUM_SMS = 132
WIDTHS = range(64, 2049, 64)
MEMORY_DIMS = (256, 288, 292, 384, 512)
BATCHES = (1, 2, 16, 17, 31, 32, 33, 60, 64)


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as entry
    entry.build()
    from multilingual_text_to_speech_b200 import _lib
    return _lib.load()


@pytest.fixture(scope='module')
def plan(lib):
    """{(B, L, M, D, training): (path bits, geometry query)} of every enumerated shape that runs at least one persistent loop"""
    out = {}
    for training in (0, 1):
        for D in WIDTHS:
            for M in MEMORY_DIMS:
                for B in BATCHES:
                    k = 0
                    while True:
                        forward = False
                        for L in ((16 * k, 16 * k + 1) if k else (1,)):
                            s = G.shape(B, L, 16, M, D, training)
                            bits = lib.b200tts_decoder_path(ctypes.byref(s)) & (G.ALL if training else 0b11)
                            if bits:
                                out[(B, L, M, D, training)] = (bits, G.query(s, lib))
                            forward |= bool(bits & 1)
                        k += 1
                        if k > 1 and not forward:
                            break
    return out


def test_every_accepted_shape_is_launchable(plan):
    """The forward loops launch D / 16 row blocks x ceil(B / 32) batch halves of CTAs, all co-resident, and their attention needs one CTA
    pair per utterance; the attention reverse loop needs the same of its grid."""
    bad = []
    for (B, L, M, D, training), (bits, g) in plan.items():
        if bits & 1:
            grid = D // 16 * -(-B // 32)
            if not (grid <= NUM_SMS and grid % 2 == 0 and grid // 2 >= B):
                bad.append(('forward', B, L, M, D, training, grid))
            assert (g['grid'], g['NBH']) == (grid, -(-B // 32)), (B, L, M, D, g)
        if bits & 16 and not (g['bwd_grid'] <= NUM_SMS and g['bwd_grid'] // 2 >= B):
            bad.append(('attention reverse', B, L, M, D, training, g['bwd_grid']))
    assert not bad, (len(bad), bad[:20])


def test_every_geometry_has_a_step_checked_representative(plan):
    """A plan change that produces a new loop geometry fails here until persist_geometry.REPRESENTATIVES step-checks it (reported with
    the enumerated shape of its largest text length)."""
    seen = {}
    for (B, L, M, D, training), (bits, g) in plan.items():
        k = G.key(g, training)
        assert G.passes(g, training) == bits, (B, L, M, D, training)
        if k not in seen or L > seen[k][1]:
            seen[k] = (B, L, M, D, training)
    listed = set(G.REPRESENTATIVES.values())
    missing = {k: v for k, v in seen.items() if k not in listed}
    assert not missing, missing
    assert len(listed) == len(G.REPRESENTATIVES), 'two representatives of one key'
    assert set(seen) == listed, ('representatives of keys the plan no longer produces', listed - set(seen))


def test_representatives_have_their_keys(lib):
    for (B, L, T, M, D, training), key in G.REPRESENTATIVES.items():
        assert G.key_of(B, L, M, D, training, lib) == key, (B, L, T, M, D, training)
        assert 12 <= T <= 24
    B, L, T, M, D, training = G.ALIGNMENT_SIZED
    assert G.key_of(B, L, M, D, training, lib) in G.REPRESENTATIVES.values()


def test_shapes_past_the_limits_leave_the_forward_loops(lib):
    for (B, L, T, M, D, training), bits in G.PAST_LIMITS.items():
        g = G.query(G.shape(B, L, T, M, D, training), lib)
        assert G.passes(g, training) == bits, (B, L, M, D, training, bin(g['path']))
    # and the shapes one step inside those limits run the forward loops
    for B, L, M, D, training in ((16, 1152, 288, 1024, 0), (16, 100, 288, 512, 0), (16, 100, 288, 512, 1), (32, 464, 288, 1024, 1)):
        assert G.query(G.shape(B, L, 12, M, D, training), lib)['path'] & 1, (B, L, M, D, training)


def test_geometry_query_answers_for_the_step_shape(lib):
    """like every decoder query: T frames at R frames per step is the shape of ceil(T / R) steps; a rejected shape writes nothing"""
    s = G.shape(16, 300, 100, 288, 1024, 1)
    s.R = 3
    a = G.query(s, lib)
    assert a == G.query(G.shape(16, 300, 34, 288, 1024, 1), lib)
    assert a['path'] == lib.b200tts_decoder_path(ctypes.byref(s))
    out = (ctypes.c_int * len(G.FIELDS))(*([-7] * len(G.FIELDS)))
    assert lib.b200tts_debug_decoder_geometry(ctypes.byref(G.shape(0, 300, 12, 288, 1024, 1)), out, len(G.FIELDS)) == 0
    assert list(out) == [-7] * len(G.FIELDS)
    assert lib.b200tts_debug_decoder_geometry(ctypes.byref(G.shape(16, 300, 12, 288, 1024, 1)), out, 3) == 3
    assert list(out)[3:] == [-7] * (len(G.FIELDS) - 3)
