"""Source check of the stream contract of include/aae_b200.h over csrc/*.cu and *.cuh (no GPU needed; the device half is
tests/test_gpu_n_streams.py):

  * every kernel launch names a stream: four launch arguments, the fourth not a spelling of the default stream;
  * the calls that run on the legacy default stream or wait for the whole device (cudaMemset, cudaMemcpy, cudaDeviceSynchronize,
    cudaMalloc, cudaFree) appear only in the functions listed below, each with the reason it may;
  * every extern "C" entry point that takes `void* stream` uses it.

A caller's non-blocking stream (every torch.cuda.Stream is one) is not ordered against the legacy stream, so a launch or fill
that lands there races the caller's work, and no test that runs on the default stream of a fresh process can see it."""
import os
import re

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "augmentedautoencoder_b200", "csrc")

DEFAULT_STREAM_SPELLINGS = {"0", "nullptr", "NULL", "cudaStreamLegacy", "cudaStreamPerThread", "cudaStreamDefault"}
LEGACY_CALLS = ("cudaMemset", "cudaMemcpy", "cudaDeviceSynchronize", "cudaMalloc", "cudaFree")

# (file, function) -> why it may launch on the default stream
LAUNCH_ALLOW = {
    ("tc_match.cu", "tc_codebook_create"): "creator: packs the codebook on the legacy stream and waits for the device before returning",
}

# (file, function) -> why it may call one of LEGACY_CALLS
CALL_ALLOW = {
    ("common.cuh", "creation_fence"): "the device-wide wait every creator ends with",
    ("common.cuh", "DevArray::replace"): "the one cudaMalloc: by creators, and by scratch that appears or grows on first use",
    ("common.cuh", "DevArray::reset"): "the one cudaFree: owners going away or being replaced",
    ("common.cuh", "DevArray::alloc_zeroed"): "zero-filled allocation for creators only (they end in creation_fence)",
    ("capi.cu", "aae_encoder_create"): "creator: zero masters; ends in creation_fence",
    ("capi.cu", "aae_encoder_enable_sigma_head"): "creator: zero head; ends in creation_fence",
    ("capi.cu", "aae_codebook_create"): "creator: uploads the embedding; ends in creation_fence",
    ("capi.cu", "aae_decoder_create"): "creator: zero masters; ends in creation_fence",
    ("capi.cu", "aae_decoder_enable_mask_head"): "creator: zero head; ends in creation_fence",
    ("capi.cu", "fill_slot"): "trainer creation: initial optimizer slots; trainer_create ends in creation_fence",
    ("capi.cu", "make_pg"): "trainer creation: zero gradients; trainer_create ends in creation_fence",
    ("capi.cu", "aae_encoder_activation"): "takes no stream: waits for the device, documented in the header",
    ("tc_match.cu", "tc_codebook_create"): "creator: packs the codebook and waits for the device",
}


# ------------------------------------------------------------------------------------------------ a small C++ reader
def blank_comments_and_strings(src):
    """Comments, string and character literals replaced by spaces (quotes and newlines kept), so offsets and lines survive."""
    out, i, n = [], 0, len(src)
    while i < n:
        c = src[i]
        if src.startswith("//", i):
            j = src.find("\n", i)
            j = n if j < 0 else j
            out.append(" " * (j - i))
            i = j
        elif src.startswith("/*", i):
            j = src.find("*/", i + 2)
            j = n if j < 0 else j + 2
            out.append(re.sub(r"[^\n]", " ", src[i:j]))
            i = j
        elif c in "\"'":
            j = i + 1
            while j < n and src[j] != c:
                j += 2 if src[j] == "\\" else 1
            out.append(c + " " * (j - i - 1) + c)
            i = j + 1
        else:
            out.append(c)
            i += 1
    return "".join(out)


_CONTAINER = re.compile(r'\b(namespace|struct|class|union)\b|extern\s*"\s*"\s*$')
_NAME = re.compile(r"([A-Za-z_~][\w:~]*)\s*$")


def functions(clean):
    """[(name, header, body_start, body_end)] of every function body in blanked source.  Methods defined inside a struct are
    named Struct::method; lambdas and nested blocks belong to the function around them."""
    found, stack, i, n, stmt = [], [], 0, len(clean), 0      # stack of container names ('' for namespace / extern "C")
    while i < n:
        c = clean[i]
        if c in ";}":
            if c == "}" and stack:
                stack.pop()
            stmt = i + 1
        elif c == "{":
            header = re.sub(r"__launch_bounds__\s*\([^)]*\)", " ", clean[stmt:i])
            header = "\n".join(l for l in header.split("\n") if not l.lstrip().startswith("#")).strip()
            paren = header.find("(")
            m = _CONTAINER.search(header if paren < 0 else header[:paren])
            if m and (paren < 0 or m.group(1) is None):
                s = re.search(r"\b(?:struct|class|union)\s+(\w+)", header)
                stack.append(s.group(1) if s else "")
                stmt = i + 1
            else:
                depth, j = 1, i + 1
                while j < n and depth:
                    depth += {"{": 1, "}": -1}.get(clean[j], 0)
                    j += 1
                nm = _NAME.search(header[:paren]) if paren >= 0 else None
                if nm:
                    scope = "::".join(s for s in stack if s)
                    found.append(((scope + "::" if scope else "") + nm.group(1), header, i + 1, j - 1))
                i, stmt = j - 1, j
        i += 1
    return found


def split_args(text):
    """Top-level comma split: (), [], {} and template argument lists (`name<a, b>(`) keep their commas."""
    text = re.sub(r"([\w:]+)<([\w\s:,*&]+)>(?=\s*\()", lambda m: m.group(1) + "<" + m.group(2).replace(",", ";") + ">", text)
    args, depth, cur = [], 0, []
    for c in text:
        depth += c in "([{"
        depth -= c in ")]}"
        if c == "," and depth == 0:
            args.append("".join(cur).strip())
            cur = []
        else:
            cur.append(c)
    args.append("".join(cur).strip())
    return args


def launches(clean):
    """[(offset, [launch arguments])] of every <<<...>>> in blanked source."""
    out, i = [], 0
    while True:
        a = clean.find("<<<", i)
        if a < 0:
            return out
        depth, j = 0, a + 3
        while j < len(clean) and not (depth == 0 and clean.startswith(">>>", j)):
            depth += clean[j] in "(["
            depth -= clean[j] in ")]"
            j += 1
        out.append((a, split_args(clean[a + 3:j])))
        i = j + 3


def lint(name, src, launch_allow=LAUNCH_ALLOW, call_allow=CALL_ALLOW):
    """(problems, allow-list keys used) of one source file."""
    clean = blank_comments_and_strings(src)
    funcs = functions(clean)
    problems, used = [], set()

    def owner(off):
        for fn, _, a, b in funcs:
            if a <= off < b:
                return fn
        return "<file scope>"

    def where(off):
        return "%s:%d (in %s)" % (name, clean.count("\n", 0, off) + 1, owner(off))

    for off, args in launches(clean):
        stream = re.sub(r"\(\s*cudaStream_t\s*\)|\s", "", args[3]) if len(args) == 4 else None
        if stream is None or stream in DEFAULT_STREAM_SPELLINGS or stream == "":
            key = (name, owner(off))
            if key in launch_allow:
                used.add(("launch",) + key)
            else:
                problems.append("%s: kernel launch <<<%s>>> does not name the caller's stream" % (where(off), ", ".join(args)))
    for m in re.finditer(r"\b(%s)\s*\(" % "|".join(LEGACY_CALLS), clean):
        key = (name, owner(m.start()))
        if key in call_allow:
            used.add(("call",) + key)
        else:
            problems.append("%s: %s outside the creators and destroyers (use the *Async form on the caller's stream, or list the "
                            "function with its reason)" % (where(m.start()), m.group(1)))
    for fn, header, a, b in funcs:
        if re.search(r'extern\s*"\s*"', header) and re.search(r"\bvoid\s*\*\s*stream\b", header) and not re.search(r"\bstream\b", clean[a:b]):
            problems.append("%s: takes `void* stream` and never uses it" % where(a))
    return problems, used


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh")))


# ------------------------------------------------------------------------------------------------ the tests
def test_the_library_sources_keep_the_stream_contract():
    problems, used = [], set()
    for f in sources():
        p, u = lint(f, open(os.path.join(CSRC, f)).read())
        problems += p
        used |= u
    assert not problems, "\n" + "\n".join(problems)
    stale = [k for k in LAUNCH_ALLOW if ("launch",) + k not in used] + [k for k in CALL_ALLOW if ("call",) + k not in used]
    assert not stale, "allow-list entries that no longer match anything: %s" % stale


def test_the_reader_sees_every_launch_and_entry_point():
    """Guards the lint itself: if the reader lost track of the sources, the check above would pass vacuously."""
    n_launch, entry = 0, set()
    for f in sources():
        clean = blank_comments_and_strings(open(os.path.join(CSRC, f)).read())
        found = launches(clean)
        assert len(found) == clean.count("<<<")
        n_launch += len(found)
        if f in ("capi.cu", "crops.cu"):
            entry |= {fn for fn, header, _, _ in functions(clean) if re.search(r'extern\s*"\s*"', header)}
    assert n_launch >= 75
    header = open(os.path.join(CSRC, "..", "..", "include", "aae_b200.h")).read()
    declared = set(re.findall(r"AAE_API\s+[\w\s\*]+?\b(aae_\w+)\s*\(", header))
    assert declared and declared <= entry, sorted(declared - entry)


SNIPPET = r'''
namespace aae {
struct Buf {
  float* p = nullptr;
  void release() { cudaFree(p); }
};
template <int K, class P>
__global__ void __launch_bounds__(256) k_kernel(const float* a, float* b) { b[0] = a[0]; }
int launch_ok(const float* a, float* b, cudaStream_t s) {
  k_kernel<2, int><<<dim3(1, std::min<int, int>(2, 3)),
                     256, 0, s>>>(a, b);   // cudaMemset(p, 0, 4) in a comment is not a call
  set_error("cudaMalloc(%zu) failed", 4);
  return 0;
}
int launch_without_stream(const float* a, float* b) {
  k_kernel<2, int><<<1, 256>>>(a, b);
  return 0;
}
int launch_on_zero(const float* a, float* b) {
  with_planes(1, [&](auto P) { k_kernel<2, int><<<1, 256, 0, (cudaStream_t)0>>>(a, b); });
  return 0;
}
int stray_fill(float* p, cudaStream_t s) {
  cudaMemsetAsync(p, 0, 4, s);
  cudaMemset(p, 0, 4);
  return 0;
}
}  // namespace aae
extern "C" int aae_uses(float* p, void* stream) { return aae::stray_fill(p, (cudaStream_t)stream); }
extern "C" int aae_ignores(float* p, void* stream) {
  return aae::stray_fill(p, nullptr);
}
'''


def test_the_lint_flags_what_it_is_for():
    problems, _ = lint("snippet.cu", SNIPPET, launch_allow={}, call_allow={("snippet.cu", "Buf::release"): "destroyer"})
    text = "\n".join(problems)
    assert len(problems) == 4, text
    assert "snippet.cu:16 (in launch_without_stream): kernel launch" in text
    assert "snippet.cu:20 (in launch_on_zero): kernel launch" in text
    assert "snippet.cu:25 (in stray_fill): cudaMemset outside" in text
    assert "(in aae_ignores): takes `void* stream` and never uses it" in text
    # the same snippet without the allow-list entry: the destroyer's cudaFree is reported too
    assert any("Buf::release" in p and "cudaFree" in p for p in lint("snippet.cu", SNIPPET, {}, {})[0])


@pytest.mark.parametrize("text,want", [
    ("grid, 256, 0, s", ["grid", "256", "0", "s"]),
    ("dim3(a, b), std::min<long long>(132 * 16, ceil_div(t, 256)), smem(H, W), s", ["dim3(a, b)", "std::min<long long>(132 * 16, ceil_div(t, 256))", "smem(H, W)", "s"]),
    ("1, 256", ["1", "256"]),
])
def test_launch_argument_split(text, want):
    assert split_args(text) == want
