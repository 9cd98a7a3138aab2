#!/usr/bin/env python
"""Builds oracle/_ref/libref_cs.so: the REFERENCE IMPORTER'S OWN C# packing code, compiled for the CPU.

Recipe (TEST INFRASTRUCTURE; nothing here is product code, nothing of the reference is copied into the repo):
  1. read the members named in KEEP (names only) from package/{Editor/GaussianSplatAssetCreator.cs,
     Editor/Utils/GaussianFileReader.cs, Runtime/GaussianUtils.cs, Runtime/GaussianSplatAsset.cs} where they lie under
     /root/reference;
  2. apply the purely syntactic rewrites of `rewrite()` (C# spelling -> C++ spelling; no expression is reordered):
       - attributes ([BurstCompile], [ReadOnly], [NativeDisable...]) and access / `unsafe` modifiers dropped,
       - `struct X : IJob...` / `: IComparer<..>` -> plain struct, `enum` -> `enum class`, `const` members -> constexpr,
       - `A.B` on a type or static class -> `A::B`, `float.PositiveInfinity` -> `float_PositiveInfinity`,
       - `new T(..)` -> `T(..)`, `T x = new(..)` -> `T x(..)`, `new T { a = x, .. }` -> an immediately-invoked lambda,
       - tuples: `(ulong, int)` -> `std::pair<ulong, int>`, `(a, b)` values -> `std::make_pair(a, b)`, Item1/2 -> first/second,
       - C# switch expressions -> chains of `?:` (the default arm keeps its `throw`),
       - property swizzles `v.xyz` -> `v.xyz()`, `var` -> `auto`, `var (a, b)` -> `auto [a, b]`, `= default` -> `= {}`,
         `null` -> `nullptr`,
       - `(uint)` / `(ulong)` / `(ushort)` casts -> `cs::conv<T>(..)`, which applies C#'s truncating float -> integer
         conversion and records every operand outside the target's range (see cs_shim.hpp),
       - `job.Schedule(n, batch).Complete()` -> `cs::RunParallelFor(job, n)` (Execute(0 .. n-1) in order);
  3. write the result to oracle/_ref/ref_cs_gen.inc (an intermediate, deleted after a successful build unless --keep is
     given) and compile ref_cs_harness.cpp, which includes it together with cs_shim.hpp, into oracle/_ref/libref_cs.so.
The GPU box has no /root/reference: it uses the prebuilt library that travels with the tree."""
from __future__ import annotations

import os
import re
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
OUT = HERE.parent / "_ref"
REF = Path("/root/reference/package")

# (file, class whose body holds the members or None for the file's namespace, kept member names or "*" for all)
KEEP = [
    ("Runtime/GaussianUtils.cs", "GaussianUtils", "*"),
    ("Runtime/GaussianSplatAsset.cs", "GaussianSplatAsset",
     ["kChunkSize", "kTextureWidth", "VectorFormat", "ColorFormat", "SHFormat", "SHTableItemFloat32", "SHTableItemFloat16",
      "SHTableItemNorm11", "SHTableItemNorm6", "ChunkInfo", "GetVectorSize", "GetColorSize", "GetOtherSizeNoSHIndex", "GetSHCount",
      "CalcTextureSize", "CalcPosDataSize", "CalcOtherDataSize", "CalcColorDataSize", "CalcSHDataSize", "CalcChunkDataSize"]),
    ("Editor/Utils/GaussianFileReader.cs", None, ["InputSplatData"]),
    ("Editor/Utils/GaussianFileReader.cs", "GaussianFileReader", ["LinearizeDataJob"]),
    ("Editor/GaussianSplatAssetCreator.cs", "GaussianSplatAssetCreator",
     ["CalcBoundsJob", "ReorderMortonJob", "OrderComparer", "ReorderMorton", "CalcChunkDataJob", "ConvertColorJob",
      "EncodeFloat3ToNorm16", "EncodeFloat3ToNorm11", "EncodeFloat3ToNorm655", "EncodeFloat3ToNorm565", "EncodeQuatToNorm10",
      "EmitEncodedVector", "CreatePositionsDataJob", "CreateOtherDataJob", "NextMultipleOf", "SplatIndexToTextureIndex",
      "CreateColorDataJob", "CreateSHDataJob"]),
]
SCOPES = ("GaussianSplatAsset", "GaussianUtils", "GaussianSplatAssetCreator", "GaussianFileReader", "math", "Allocator",
          "UnsafeUtility", "VectorFormat", "ColorFormat", "SHFormat")


def skip_to_match(text: str, i: int) -> int:
    """Index just past the brace that closes the one at text[i], skipping comments, strings and char literals."""
    depth, n = 0, len(text)
    while i < n:
        if text.startswith("//", i):
            i = text.find("\n", i)
            i = n if i < 0 else i
            continue
        if text.startswith("/*", i):
            i = text.find("*/", i) + 2
            continue
        c = text[i]
        if c in "\"'":
            j = i + 1
            while text[j] != c:
                j += 2 if text[j] == "\\" else 1
            i = j + 1
            continue
        if c == "{":
            depth += 1
        elif c == "}":
            depth -= 1
            if depth == 0:
                return i + 1
        i += 1
    raise ValueError("unbalanced braces")


def class_body(text: str, name: str) -> str:
    m = re.search(r"\b(?:class|struct)\s+%s\b[^{]*\{" % name, text)
    if not m:
        raise KeyError(name)
    start = m.end() - 1
    return text[start + 1:skip_to_match(text, start) - 1]


def member(body: str, name: str) -> str:
    """The text of member `name` of a class body: its attributes, declaration and body (or initializer)."""
    decl = re.compile(r"^[ \t]*(?:\[[^\]\n]*\][ \t]*\n?[ \t]*)*"
                      r"(?:(?:public|private|internal|static|unsafe|readonly|const)\s+)*"
                      r"(?:(?:struct|enum|class)\s+%s\b|[A-Za-z_][\w.<>(), ]*?\s+%s\s*(?:\(|=))" % (name, name), re.M)
    for m in decl.finditer(body):
        head_end = m.end()
        brace, semi = body.find("{", head_end), body.find(";", head_end)
        if re.search(r"=\s*$", m.group(0)) or (semi >= 0 and (brace < 0 or semi < brace)):
            return body[m.start():semi + 1]          # a constant
        return body[m.start():skip_to_match(body, brace)] + ("\n;" if re.search(r"\b(struct|enum)\s+%s\b" % name, m.group(0)) else "")
    raise KeyError(name)


def split_top(s: str, sep: str = ","):
    out, depth, cur = [], 0, ""
    for c in s:
        if c in "([{":
            depth += 1
        elif c in ")]}":
            depth -= 1
        if c == sep and depth == 0:
            out.append(cur)
            cur = ""
        else:
            cur += c
    if cur.strip():
        out.append(cur)
    return out


def object_initializers(text: str) -> str:
    """`new T { a = x, b = y }` -> `[&] { T _o; _o.a = x; _o.b = y; return _o; }()`."""
    pat = re.compile(r"\bnew\s+(\w+)\s*\{")
    while True:
        m = pat.search(text)
        if not m:
            return text
        end = skip_to_match(text, m.end() - 1)
        fields = [f.strip() for f in split_top(text[m.end():end - 1]) if f.strip()]
        assigns = " ".join("_o.%s;" % f for f in fields)
        text = text[:m.start()] + "[&] { %s _o; %s return _o; }()" % (m.group(1), assigns) + text[end:]


def switch_expressions(text: str) -> str:
    """`X switch { A => a, B => b, _ => c }` -> `(X == A) ? a : (X == B) ? b : c`."""
    pat = re.compile(r"(\w+)\s+switch\s*\{")
    while True:
        m = pat.search(text)
        if not m:
            return text
        end = skip_to_match(text, m.end() - 1)
        arms = [a.strip() for a in split_top(text[m.end():end - 1]) if a.strip()]
        expr = ""
        for arm in arms:
            lhs, rhs = (s.strip() for s in arm.split("=>", 1))
            expr += ("(%s)" % rhs) if lhs == "_" else "(%s == %s) ? (%s) : " % (m.group(1), lhs, rhs)
        text = text[:m.start()] + "(" + expr + ")" + text[end:]


def integer_casts(text: str) -> str:
    """`(uint) operand` -> `cs::conv<uint>(operand)`; the operand is a parenthesised group or a member/index chain."""
    pat = re.compile(r"\((uint|ulong|ushort)\)\s*")
    out, i = "", 0
    while True:
        m = pat.search(text, i)
        if not m:
            return out + text[i:]
        j = m.end()
        if text[j] == "(":
            depth, k = 0, j
            while True:
                depth += {"(": 1, ")": -1}.get(text[k], 0)
                k += 1
                if depth == 0:
                    break
        else:
            k = re.match(r"[\w.]+(?:\[[^\]]*\])*(?:\.\w+)*", text[j:]).end() + j
        out += text[i:m.start()] + "cs::conv<%s>(%s)" % (m.group(1), integer_casts(text[j:k]))
        i = k


def rewrite(text: str) -> str:
    text = re.sub(r"\[\s*(?:BurstCompile|ReadOnly|WriteOnly|NativeDisable\w+)[^\]]*\]", "", text)
    text = object_initializers(text)
    text = switch_expressions(text)
    text = re.sub(r"\(\s*ulong\s*,\s*int\s*\)", "std::pair<ulong, int>", text)
    text = re.sub(r"\(\s*int\s*,\s*int\s*\)", "std::pair<int, int>", text)
    text = re.sub(r"(=|return)\s*\((\w+),\s*(\w+)\)\s*;", r"\1 std::make_pair(\2, \3);", text)
    text = text.replace(".Item1", ".first").replace(".Item2", ".second")
    text = re.sub(r"\b(public|private|internal|protected|unsafe|readonly)\s+", "", text)
    text = re.sub(r"\bconst\s+(float|int|uint)\b", r"static constexpr \1", text)
    text = re.sub(r"\bstruct\s+(\w+)\s*:\s*I\w+(?:<[^{]*>)?", r"struct \1", text)
    text = re.sub(r"\benum\s+(\w+)", r"enum class \1", text)
    text = re.sub(r"(\S+)\s+(\w+)\s*=\s*new\s*\(", r"\1 \2(", text)
    text = re.sub(r"\bnew\s+(?=[A-Za-z_])", "", text)
    text = re.sub(r"(\w+)\.Schedule\(([^;]*?),\s*\d+\)\.Complete\(\)", r"cs::RunParallelFor(\1, \2)", text)
    text = re.sub(r"\bfloat\.(\w+)", r"float_\1", text)
    for _ in range(3):
        text = re.sub(r"\b(%s)\.(?=\w)" % "|".join(SCOPES), r"\1::", text)
    text = re.sub(r"\.(xyz|xyzw|yzwx|xzwy|xywz)\b(?!\s*\()", r".\1()", text)
    text = re.sub(r"\bvar\s*\((\w+),\s*(\w+)\)", r"auto [\1, \2]", text)   # deconstruction -> structured binding
    text = re.sub(r"\bvar\b", "auto", text)
    text = re.sub(r"\bnull\b", "nullptr", text)
    text = re.sub(r"=\s*default\s*;", "= {};", text)
    text = re.sub(r"(?<=\d)_(?=\d)", "", text)
    text = integer_casts(text)
    return text


def generate() -> str:
    parts = ["// GENERATED from the reference's importer sources by oracle/refcs/build_ref_cs.py; never committed"]
    for path, cls, names in KEEP:
        text = (REF / path).read_text()
        if cls is None:
            body = text
        else:
            body = class_body(text, cls)
        if names == "*":
            items = [body]
        else:
            # types first: a member function's signature may name a nested enum or struct declared later in the class
            order = sorted(names, key=lambda nm: 0 if re.search(r"\b(?:struct|enum)\s+%s\b|const\s+\w+\s+%s\b" % (nm, nm), body) else 1) \
                if cls == "GaussianSplatAsset" else names
            items = [member(body, nm) for nm in order]
        code = "\n\n".join(rewrite(it) for it in items)
        parts.append(code if cls is None else "struct %s {\n%s\n};" % (cls, code))
    return "\n\n".join(parts) + "\n"


def main() -> int:
    if not os.path.isdir(REF / "Editor"):   # absent, or not readable by this user
        print("build_ref_cs: %s not present (GPU box?): keeping the prebuilt library" % REF)
        return 0
    OUT.mkdir(exist_ok=True)
    inc = OUT / "ref_cs_gen.inc"
    inc.write_text(generate())
    cmd = ["/usr/bin/g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fno-strict-aliasing", "-fno-math-errno", "-fPIC", "-shared",
           "-w", "-I", str(HERE), "-I", str(OUT), "-o", str(OUT / "libref_cs.so"), str(HERE / "ref_cs_harness.cpp")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode == 0 and "--keep" not in sys.argv:
        inc.unlink()   # the rewritten reference text is a build intermediate: only the compiled library stays on disk
    if r.returncode != 0:
        sys.stderr.write(r.stdout[-6000:])
        return 1
    print("built", OUT / "libref_cs.so")
    return 0


if __name__ == "__main__":
    sys.exit(main())
