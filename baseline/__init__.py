"""The reference arm: the UNMODIFIED google/TensorNetwork package copied into oracle/_ref by
build() (git-ignored; recipe oracle/install_ref.py) plus the import environment it needs
(baseline/refenv.py)."""
