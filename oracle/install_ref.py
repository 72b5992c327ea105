"""Recipe for oracle/_ref: the unmodified upstream TensorNetwork package that the reference-caller tests and the
reference arm of bench.py import (through baseline/refenv.py).

The upstream package is pure Python, so "building" it is copying its `tensornetwork/` package directory, unmodified,
into oracle/_ref.  oracle/_ref is git-ignored: no upstream source enters the repository.  The upstream checkout is
read from $TENSORNETWORK_SRC (default /root/reference); where there is none, an existing oracle/_ref is kept.
"""
import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "_ref")


def source():
  return os.environ.get("TENSORNETWORK_SRC", "/root/reference")


def installed():
  return os.path.isdir(os.path.join(TARGET, "tensornetwork", "backends"))


def install():
  """Returns the directory to put on sys.path, or None when neither an install nor an upstream checkout exists."""
  if installed():
    return TARGET
  src = os.path.join(source(), "tensornetwork")
  if not os.path.isdir(os.path.join(src, "backends")):
    return None
  shutil.rmtree(TARGET, ignore_errors=True)
  shutil.copytree(src, os.path.join(TARGET, "tensornetwork"), ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
  return TARGET


if __name__ == "__main__":
  print(install())
