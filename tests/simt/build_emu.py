"""Build tests/simt/_build/libthb_emu.so: theseus_b200/csrc/{thb_sparse_lane,thb_costs,thb_gram,thb_sparse,thb_lie_ops}.cu compiled for the HOST with g++ on
top of simt_shim.h (one OS thread per CUDA thread).  The sources are used as they are except for three mechanical rewrites done here:
  kernel<<<grid, block, smem, stream>>>(args)  ->  SIMT_LAUNCH(kernel, grid, block, smem, args)
  extern __shared__ T name[];                   ->  T* name = simt_dyn_smem<T>();
  #include "thb_common.cuh"                     ->  #include "simt_shim.h"
Test infrastructure only (like oracle/): nothing in the product imports it."""
import os
import re
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "..", "theseus_b200", "csrc")
SOURCES = ["thb_sparse_lane.cu", "thb_costs.cu", "thb_gram.cu", "thb_sparse.cu", "thb_lie_ops.cu", "thb_front.cu"]     # + the headers they include (thb_lie.cuh)
HEADERS = ["thb_lie.cuh"]
OUT_DIR = os.path.join(HERE, "_build")


def _split_top_level(s: str):
    parts, depth, cur = [], 0, ""
    for ch in s:
        if ch in "([":
            depth += 1
        elif ch in ")]":
            depth -= 1
        if ch == "," and depth == 0:
            parts.append(cur.strip()); cur = ""
        else:
            cur += ch
    parts.append(cur.strip())
    return parts


def _rewrite_launches(text: str) -> str:
    """kernel<targs><<<grid, block, smem, stream>>>(args...)  ->  SIMT_LAUNCH((kernel<targs>), grid, block, smem, args...); the
    argument list may span lines."""
    out, pos = [], 0
    while True:
        i = text.find("<<<", pos)
        if i < 0:
            break
        if text.startswith("<<<...>>>", i):           # prose in a comment
            out.append(text[pos:i + 9]); pos = i + 9
            continue
        k = i                                        # walk back over the kernel expression: name, optional <template args>
        if text[k - 1] == ">":
            depth = 0
            while True:
                k -= 1
                depth += (text[k] == ">") - (text[k] == "<")
                if depth == 0:
                    break
        while k > 0 and (text[k - 1].isalnum() or text[k - 1] in "_:"):
            k -= 1
        kernel = text[k:i]
        j = text.index(">>>", i)
        cfg = _split_top_level(text[i + 3:j])
        assert len(cfg) == 4 and text[j + 3] == "(", text[k:j + 40]
        depth, e = 0, j + 3
        while True:
            depth += (text[e] == "(") - (text[e] == ")")
            e += 1
            if depth == 0:
                break
        args = text[j + 4:e - 1]
        out.append(text[pos:k] + f"SIMT_LAUNCH(({kernel}), {cfg[0]}, {cfg[1]}, {cfg[2]}, {args})")
        pos = e
    out.append(text[pos:])
    return "".join(out)


def rewrite(text: str) -> str:
    text = _rewrite_launches(text)
    text = re.sub(r"extern __shared__ (\w+) (\w+)\[\];", lambda m: f"{m.group(1)}* {m.group(2)} = simt_dyn_smem<{m.group(1)}>();", text)
    text = text.replace('#include "thb_common.cuh"', '#include "simt_shim.h"').replace("#include <cuda_runtime.h>", '#include "simt_shim.h"')
    assert "<<<" not in text.replace("<<<...>>>", "") and "extern __shared__" not in text
    return text


def build(force: bool = False) -> str:
    os.makedirs(OUT_DIR, exist_ok=True)
    lib = os.path.join(OUT_DIR, "libthb_emu.so")
    texts = {f: rewrite(open(os.path.join(CSRC, f)).read()) for f in SOURCES + HEADERS}
    gens = {f: os.path.join(OUT_DIR, f.replace(".cuh", ".cuh").replace(".cu", "_emu.cpp") if f.endswith(".cu") else os.path.join(OUT_DIR, f)) for f in texts}
    fresh = (not force and os.path.exists(lib) and all(os.path.exists(g) and open(g).read() == texts[f] for f, g in gens.items())
             and os.path.getmtime(lib) >= os.path.getmtime(os.path.join(HERE, "simt_shim.h")))
    if fresh:
        return lib
    for f, g in gens.items():
        open(g, "w").write(texts[f])
    cmd = ["g++", "-std=c++20", "-O1", "-fPIC", "-shared", "-pthread", "-DTHB_SIMT_EMU", "-DTHB_ARCH=90", "-Wno-unknown-pragmas",
           # the CUDA library exports host stubs with the SAME mangled kernel names: bind this library's references to its own definitions
           "-Wl,-Bsymbolic", "-fno-semantic-interposition", "-I", HERE, "-I", OUT_DIR] + [gens[f] for f in SOURCES] + ["-o", lib]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ failed on the emulation build:\n" + r.stdout + r.stderr[-6000:])
    return lib


if __name__ == "__main__":
    print(build(force=True))
