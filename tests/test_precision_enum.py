"""CPU check that the C header and the Python binding agree on the aae_precision values (no GPU needed)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_precisions():
    src = open(os.path.join(ROOT, "include", "aae_b200.h")).read()
    body = re.search(r"typedef enum \{([^}]*)\} aae_precision;", src).group(1)
    return {k: int(v) for k, v in re.findall(r"(AAE_PREC_\w+)\s*=\s*(\d+)", body)}


def test_header_and_binding_agree_on_the_precisions():
    from augmentedautoencoder_b200 import _lib
    prec = header_precisions()
    assert prec == {"AAE_PREC_FP32_SIMT": 0, "AAE_PREC_TC_SPLIT": 1, "AAE_PREC_TC_FP16": 2}
    assert (_lib.PREC_FP32_SIMT, _lib.PREC_TC_SPLIT, _lib.PREC_TC_FP16) == (0, 1, 2)
