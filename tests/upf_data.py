"""The UPF fixtures of tests/golden/upf (stored xz-compressed) as text, as parsed pseudopotentials, or as a plain file."""
import lzma
import os

UPF_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "upf")


def upf_text(name):
    with lzma.open(os.path.join(UPF_DIR, name + ".xz"), "rt") as fh:
        return fh.read()


def product_psp(name):
    from dftk_b200 import parse_upf
    return parse_upf(upf_text(name), identifier=name)


def oracle_psp(name):
    from oracle.psp_upf import PspUpf
    return PspUpf(upf_text(name), description=name)


def upf_file(name, directory):
    """Write the decompressed file into `directory` and return its path."""
    path = os.path.join(str(directory), name)
    with open(path, "w") as fh:
        fh.write(upf_text(name))
    return path
