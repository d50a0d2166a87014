"""Every w2l_trainer_* entry point that takes a trainer refuses a NULL one with W2L_ERR_INVALID_ARGUMENT and names itself
in w2l_last_error() (num_params, param_layout and time_stride return -1, describe ""), as a closed Python Trainer passes
exactly that NULL.  The arena calls check `which` (and get_flat `what`) before they read the trainer.  The sweep is driven
from the header's prototypes, so an entry point added later is covered too.  Both checks run in a child process, so
that a call that dereferences its handle cannot take the test session down.  Nothing here reaches a GPU."""
import ctypes
import json
import os
import subprocess
import sys

INVALID = 1
NOT_A_HANDLE = {"w2l_trainer_create", "w2l_trainer_create_seq2seq", "w2l_trainer_load"}
VALUE_CALLS = {"w2l_trainer_num_params": -1, "w2l_trainer_param_layout": -1, "w2l_trainer_time_stride": -1, "w2l_trainer_describe": ""}


def sweep():
    """{name: [result, last error]} of every trainer entry point called with a NULL trainer; each name is printed before
    its call, so a crash shows which call it was"""
    from wav2letter_b200 import capi

    plausible = {ctypes.c_int: 1, ctypes.c_longlong: 1, ctypes.c_ulonglong: 1, ctypes.c_size_t: 1, ctypes.c_float: 1.0,
                 ctypes.c_double: 1.0}
    out = {}
    for name, (_, argtypes) in sorted(capi.PROTOTYPES.items()):
        if not name.startswith("w2l_trainer_") or name in NOT_A_HANDLE:
            continue
        print("calling", name, flush=True)
        assert capi.lib.w2l_set_precision(-1) == INVALID  # an unrelated error text, so each call must set its own
        r = getattr(capi.lib, name)(None, *(plausible.get(t) for t in argtypes[1:]))
        out[name] = [r.decode() if isinstance(r, bytes) else r, capi.lib.w2l_last_error().decode()]
    return out


def arena_checks():
    """{call: [result, last error]} of the arena calls on a fake trainer handle with an out-of-range `which` or `what`:
    the handle is never dereferenced when the check runs first"""
    from wav2letter_b200 import capi

    lib, fake = capi.lib, ctypes.c_void_p(256)
    calls = {"num_params which=3": lambda: lib.w2l_trainer_num_params(fake, 3),
             "num_params which=-1": lambda: lib.w2l_trainer_num_params(fake, -1),
             "param_layout which=3": lambda: lib.w2l_trainer_param_layout(fake, 3, 0, None, None),
             "get_flat which=3": lambda: lib.w2l_trainer_get_flat(fake, None, 3, 0, None),
             "get_flat what=2": lambda: lib.w2l_trainer_get_flat(fake, None, 0, 2, None),
             "set_flat which=3": lambda: lib.w2l_trainer_set_flat(fake, None, 3, None)}
    out = {}
    for label, call in calls.items():
        print("calling", label, flush=True)
        out[label] = [call(), lib.w2l_last_error().decode()]
    return out


def child(what: str):
    r = subprocess.run([sys.executable, "-s", __file__, what], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout.splitlines()[-1])


def test_null_trainer_is_refused_by_every_entry_point():
    results = child("sweep")
    assert "w2l_trainer_step" in results and "w2l_trainer_evaluate" in results and "w2l_trainer_destroy" in results
    for name, (got, err) in results.items():
        if name == "w2l_trainer_destroy":  # void, and NULL is a no-op
            assert got is None, name
            continue
        assert got == VALUE_CALLS.get(name, INVALID), (name, got, err)
        assert name[len("w2l_"):] in err and "null handle" in err, (name, err)


def test_arena_calls_check_which_and_what_before_the_trainer():
    for label, (got, err) in child("arena").items():
        call, arg = label.split()
        assert got == (-1 if call in ("num_params", "param_layout") else INVALID), (label, got, err)
        assert err.startswith(f"trainer_{call}: {arg.split('=')[0]} must be"), (label, err)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    print(json.dumps({"sweep": sweep, "arena": arena_checks}[sys.argv[1]]()))
