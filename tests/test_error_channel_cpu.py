"""CPU: libuhc_b200.so keeps one error text per thread.  Whichever module refuses a call, every uhc_*_last_error() reader returns the same
text, naming the entry point that failed, and a later failure never reports an earlier one's text.  Every call below is refused by its
argument checks before it touches a device."""
import ctypes as C

import pytest

READERS = ("uhc_last_error", "uhc_nn_last_error", "uhc_tc_last_error", "uhc_ppo_last_error", "uhc_rollout_last_error", "uhc_eval_last_error",
           "uhc_track_last_error", "uhc_render_last_error", "uhc_export_last_error")


@pytest.fixture(scope="module")
def lib():
    from uhc_b200 import build
    L = C.CDLL(build.build())
    for f in READERS:
        getattr(L, f).restype = C.c_char_p
    return L


def _texts(L):
    return [getattr(L, f)() for f in READERS]


# (entry point, call) -- each returns -2 from its argument checks
def _refused_calls(L):
    p = C.c_void_p(64)                       # a non-null pointer none of the checks below reads
    buf = (C.c_char * 4096)()                # zeroed stand-in for a policy / output struct, not read either
    n = (C.c_int * 1)(1)
    return [
        ("uhc_engine_create", lambda: L.uhc_engine_create(None, None, C.c_int(8), C.c_int(0), C.c_int(32), None)),
        ("uhc_mcp_combine", lambda: L.uhc_mcp_combine(p, p, None, p, C.c_int(8), C.c_int(4), C.c_int(0), None)),
        ("uhc_linear_forward_tc", lambda: L.uhc_linear_forward_tc(p, p, None, None, p, C.c_int(8), C.c_int(8), C.c_int(3), C.c_int(0), C.c_int(0), None)),
        ("uhc_ppo_trainer_create", lambda: L.uhc_ppo_trainer_create(None, None, C.c_long(8), C.c_int(8), C.c_int(0), None)),
        ("uhc_rollout", lambda: L.uhc_rollout(None, C.c_int(1), C.c_int(0), buf, p, p, C.c_float(5.0), C.c_int(1), C.c_ulonglong(0), C.c_float(1.0), buf,
                                              C.c_int(1), None)),
        ("uhc_eval_run_groups", lambda: L.uhc_eval_run_groups(None, C.c_int(1), n, n, buf, None, C.c_float(5.0), C.c_int(1), C.c_int(32), p, buf, None,
                                                              None)),
        ("uhc_track_begin", lambda: L.uhc_track_begin(None, C.c_int(8), C.c_int(0), C.c_int(72), None, None)),
        ("uhc_qpos_to_smpl", lambda: L.uhc_qpos_to_smpl(None, p, C.c_int(32), C.c_long(1), C.c_long(76), None, p, p, None)),
        ("uhc_render_init", lambda: L.uhc_render_init(None, None)),
    ]


def test_every_reader_returns_the_failing_calls_text(lib):
    for who, call in _refused_calls(lib):
        assert call() == -2, who
        texts = _texts(lib)
        assert len(set(texts)) == 1, (who, texts)
        assert texts[0].startswith(who.encode() + b": "), (who, texts[0])


def test_a_tensor_core_failure_after_an_nn_failure_reports_its_own_text(lib):
    from uhc_b200 import nn
    calls = dict(_refused_calls(lib))
    assert calls["uhc_mcp_combine"]() == -2
    rc = calls["uhc_linear_forward_tc"]()
    assert rc == -2
    with pytest.raises(RuntimeError) as e:
        nn._chk(rc)
    assert str(e.value).startswith("uhc_nn: uhc_linear_forward_tc: ") and "uhc_mcp_combine" not in str(e.value)
