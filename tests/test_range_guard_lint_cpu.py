"""Source check of the range guard of include/aae_b200.h (aae_encoder_range_status) over csrc/*.cu and *.cuh (no GPU needed; the
device half is tests/test_gpu_o_range_guard.py).

The tensor-core path stores fp32 values as fp16 operand planes at static scales (activations 16 x, weights 256 x).  A value past
the fp16 range becomes inf there and NaN after the next product, and NaN vanishes in a ReLU and in an fmaxf-based amax: the model
then computes garbage with status 0.  So every device site that turns fp32 into fp16 planes (split_f16, split_f16x2,
__float2half_rn, __floats2half2_rn, tc_store_f16) must either

  * be a tc_store_f16 call that passes a range flag, or sit in a function that checks one against TC_F16_OVERFLOW, or
  * be listed below with the reason its values cannot leave the fp16 range."""
import os
import re

from tests.test_stream_lint_cpu import CSRC, blank_comments_and_strings, functions, split_args

SITES = ("split_f16x2", "split_f16", "__float2half_rn", "__floats2half2_rn", "tc_store_f16")
_SITE = re.compile(r"\b(%s)\s*(?:<[^<>;]*>)?\s*\(" % "|".join(SITES))

# (file, function) -> why its conversions need no range flag
ALLOW = {
    ("tc_common.cuh", "split_f16"): "the split primitive itself: its callers check the range",
    ("tc_common.cuh", "split_f16x2"): "the split primitive itself: its callers check the range",
    ("tc_conv1.cu", "bytes_to_half4"): "the constant 1024 of the exact byte-to-fp16 trick",
    ("tc_match.cu", "tc_match_kernel"): "the query row normalised to unit length, x 64",
    ("tc_match.cu", "pack_codebook_kernel"): "codebook rows of unit length, x 64",
    ("tc_train.cu", "finish_kernel"): "dynamically scaled gradient (tc_dyn_scale puts the tensor's amax in [2^13, 2^14))",
    ("tc_train.cu", "pack_loss_grad_sep_kernel"): "dynamically scaled gradient (tc_dyn_scale puts the tensor's amax in [2^13, 2^14))",
    ("tc_train.cu", "pack_dec_dgrad_sep_kernel"): "the merged weights the guarded forward pack of the same master version checks",
    ("tc_train.cu", "pack_dec_dgrad_kernel"): "the merged weights the guarded forward pack of the same master version checks",
    ("tc_train.cu", "pack_enc_dgrad_kernel"): "the weights the guarded forward pack of the same master version checks",
    ("tc_train.cu", "conv1_im2col_kernel"): "the training crops at 16 x: crops are in [0, 1] by the header's contract",
}


def lint(name, src, allow=ALLOW):
    """(problems, allow-list keys used) of one source file."""
    clean = blank_comments_and_strings(src)
    funcs = functions(clean)
    problems, used = [], set()
    for m in _SITE.finditer(clean):
        fn = next(((f, a, b) for f, _, a, b in funcs if a <= m.start() < b), None)
        if fn is None:                                  # the declaration of a site function, not a conversion
            continue
        f, a, b = fn
        body = clean[a:b]
        if m.group(1) == "tc_store_f16":
            depth, j = 1, m.end()
            while depth:
                depth += {"(": 1, ")": -1}.get(clean[j], 0)
                j += 1
            if any("range_flag" in arg for arg in split_args(clean[m.end():j - 1])):
                continue
        if "range_flag" in body and "TC_F16_OVERFLOW" in body:
            continue
        if (name, f) in allow:
            used.add((name, f))
            continue
        problems.append("%s:%d (in %s): %s writes fp16 planes without a range flag (pass one, check one, or list the function "
                        "with its reason)" % (name, clean.count("\n", 0, m.start()) + 1, f, m.group(1)))
    return problems, used


def test_every_fp16_store_of_the_library_is_guarded_or_listed():
    problems, used, sites = [], set(), 0
    for f in sorted(x for x in os.listdir(CSRC) if x.endswith((".cu", ".cuh"))):
        src = open(os.path.join(CSRC, f)).read()
        sites += len(_SITE.findall(blank_comments_and_strings(src)))
        p, u = lint(f, src)
        problems += p
        used |= u
    assert sites >= 30, sites                            # the reader still finds the conversions
    assert not problems, "\n" + "\n".join(problems)
    assert not [k for k in ALLOW if k not in used], "allow-list entries that no longer match anything"


# the fp32 conv1's split store into conv2's (hi, lo) input, as it was before it checked the range
SNIPPET = r'''
namespace aae {
template <int MODE>
__global__ void igemm_f32_kernel(const IGemmParams p) {
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  if (MODE == GATHER_FWD && p.split_hi != nullptr) {
    __half h[4], l[4];
    for (int j = 0; j < 4; ++j) {
      const float x = v[j] * p.split_scale;
      h[j] = __float2half_rn(x);
      l[j] = __float2half_rn(x - __half2float(h[j]));
    }
  }
}
template <int PLANES>
__global__ void pack_kernel(const float* w, __half* hi, __half* lo, unsigned* range_flag, unsigned range_bit) {
  tc_store_f16<PLANES>(w[0] * 256.f, hi, lo, 0, range_flag, range_bit);
  tc_store_f16<PLANES>(w[1] * 256.f, hi, lo, 1);
}
}  // namespace aae
'''


def test_the_lint_flags_an_unguarded_split_store():
    problems, used = lint("snippet.cu", SNIPPET, allow={})
    text = "\n".join(problems)
    assert len(problems) == 3, text
    assert "snippet.cu:10 (in igemm_f32_kernel): __float2half_rn" in text
    assert "snippet.cu:11 (in igemm_f32_kernel): __float2half_rn" in text
    assert "snippet.cu:18 (in pack_kernel): tc_store_f16" in text
    guarded = SNIPPET.replace("l[j] = __float2half_rn(x - __half2float(h[j]));",
                              "l[j] = __float2half_rn(x - __half2float(h[j]));\n"
                              "      if (p.range_flag != nullptr && !(fabsf(x) < TC_F16_OVERFLOW)) atomicOr(p.range_flag, p.range_bit);")
    assert len(lint("snippet.cu", guarded, allow={})[0]) == 1
