"""Set-up shared by the scripts that run the adapters' host logic on the stand-in library tests/fake_lib.FakeLib (the
runners of tests/test_host_double.py and the gloo workers).  Each script is a process of its own: a stand-in installed
in the pytest process would be handed CUDA device pointers by any GPU test that ran after it, and whether the adapter
subclasses the reference's AbstractBackend is fixed when tensornetwork_b200 is first imported."""
import importlib.util
import itertools
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)
OK = "HOST STAND-IN OK"          # the last line every runner prints


def install(reference=False):
  """Loads the reference when `reference` is True (when it is present, for None), BEFORE tensornetwork_b200, so that the
  adapters subclass its AbstractBackend and register in its factory; then installs a fresh FakeLib and points the
  backend at host memory.  Returns (the reference's `tensornetwork` module or None, the FakeLib)."""
  from baseline import refenv
  tn = refenv.load() if reference else refenv.try_load() if reference is None else None
  import fake_lib
  from tensornetwork_b200 import _lib, backend
  lib = fake_lib.FakeLib()
  _lib.set_lib(lib)
  backend._CONFIG["device"] = "cpu"
  return tn, lib


def raises(exc, f, *args, match=None):
  """f(*args) must raise `exc`, with `match` in its message when given; returns the exception"""
  try:
    f(*args)
  except exc as e:
    assert match is None or match in str(e), str(e)
    return e
  raise AssertionError("no {} raised".format(exc.__name__))


def run_gpu_tests(filename, tn, lib):
  """Calls every test_* function of tests/<filename> with `tn` and each combination of the values of its parametrize
  marks, and prints "<name> ok" once all its calls passed.  Returns [(name, parameters, the entry points the call
  reached, counted)]."""
  spec = importlib.util.spec_from_file_location(filename[:-3], os.path.join(ROOT, "tests", filename))
  module = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(module)
  record = []
  for name, test in vars(module).items():
    if not name.startswith("test_"):
      continue
    grid = [[{m.args[0]: v} for v in m.args[1]] for m in getattr(test, "pytestmark", []) if m.name == "parametrize"]
    for combo in itertools.product(*grid):
      params = {k: v for p in combo for k, v in p.items()}
      before = lib.calls.copy()
      test(tn, **params)
      record.append((name, params, lib.calls - before))
    print(name, "ok")
  return record


def done(lib):
  """The runner's last step: no entry point of the stand-in raised (an exception the product caught would hide one)."""
  assert not lib.raised, lib.raised
  print(OK)
