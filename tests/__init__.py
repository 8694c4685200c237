"""Test suite: `-m \"not gpu\"` runs on CPU (oracle vs goldens, host logic, ABI), `-m gpu` on an H100."""
