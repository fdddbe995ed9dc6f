"""The resolve paths of general patterns that look at or before an attempt's first byte (^, \\b, look-behinds: two outcomes per
candidate) and of class-repeat-led patterns (the chain with an attempt where a search resumes inside a run), on the CPU:
tests/model_check_start.cc runs the compiler and the resolve kernels' own source, extracted from resolve_kernels.cu and
compiled for the host, and compares with the oracle (no GPU)."""
import os
import subprocess

import test_gpu_random_patterns as R
import test_gpu_parity as P

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BEGIN = "// ---- device backtracking VM (general patterns) ----"
END = "// ---- 4. generic u32 block sums / exclusive scan (per-unit match counts -> output slots) ----"

HAND = [
    # reach 1: assertions and one-byte look-behinds at the attempt's first byte
    "\\bab\\b", "^a\\w*", "(?m)^a", "\\Ba", "(?<=a)b", "(?<![ab])\\w+", "\\ba", "\\Aab", "(?m)^ab|ba", "\\b\\w+@\\w+",
    "(?<=[ =])\\w+", "(?<!\\\\)\"", "(?<=[=:])\\d+", "\\b[ab]+c", "^\\w+", "(?m)^[ab]c*", "\\bc\\w*", "(?<=a)\\w", "\\B\\w+x",
    # reach 0 now (the back-looking construct runs behind the attempt's first byte)
    "a\\b", "ab\\b", "a(?<=a)b", "\\w+\\b", "c(?m)^", "a\\Bb",
    # reach above 1: still the per-unit walk (checked for soundness only)
    "(?<=ab)c", "a?\\bb", "(?<=\\ba)b",
    # class-repeat led
    "\\w+@\\w+", "[ab]+c", "\\w++b", "(?U)a+b", "[a-c]+\\.[0-9]", "\\w+@\\w+\\.c\\b", "[ab]+ ", "\\w+1", "[ab\\n]+c", "a+b+",
    "[^ ]+ a", "\\w{2,}_", "(?U)a+?b",
    # capturing groups (STRICT_REF: the first match that sets one ends the window)
    "\\b(a)b", "^(a)?b", "(?<=a)(b)|c", "\\b(?:a|(b))c", "(?m)^(a|b)c",
    "\\b(a)?b\\w*", "^a(b)?", "(?<=[ab])(c)?a", "\\b(?:(x)|a)b", "(?m)^(?:a|(c))b",
    # dense (no candidate filter): a match can begin with almost any byte
    "\\b\\w+@\\w+", "\\b.*c", "^.*b", "(?<=a).*c", "\\b\\w*x", "(?<= ).*a",
]


def test_start_sensitive_paths_through_the_launch_sequence_match_the_oracle(tmp_path):
    src = open(os.path.join(ROOT, "grab_b200", "csrc", "resolve_kernels.cu")).read()
    assert BEGIN in src and END in src
    snippet = src[src.index(BEGIN):src.index(END)]
    assert "k_vm_resume" in snippet and "k_two_blist" in snippet and "<<<" not in snippet
    (tmp_path / "vm_snippet.inc").write_text(snippet)
    pats = HAND + list(R.PATTERNS) + R.make_cases(400, 777) + list(P.DIFF_PATTERNS)
    (tmp_path / "patterns.txt").write_text("\n".join(p for p in pats if "\n" not in p) + "\n")
    exe = str(tmp_path / "model_check_start")
    subprocess.run(["gcc", "-O2", "-c", os.path.join(ROOT, "oracle", "grab_oracle.c"), "-o", str(tmp_path / "oracle.o")], check=True)
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")  # kernels.h names cudaError_t / cudaStream_t
    subprocess.run(["g++", "-O2", "-std=c++17", "-w", "-I", str(tmp_path), "-I", cuda_inc, os.path.join(HERE, "model_check_start.cc"),
                    os.path.join(ROOT, "grab_b200", "csrc", "pattern.cc"), str(tmp_path / "oracle.o"), "-I", os.path.join(ROOT, "include"),
                    "-o", exe], check=True)
    p = subprocess.run([exe, str(tmp_path / "patterns.txt")], stdout=subprocess.PIPE, timeout=900)
    out = p.stdout.decode()
    assert p.returncode == 0 and "model ok" in out, out[-3000:]
    tail = out.strip().splitlines()[-2]

    def count(label):
        return int(tail.split(label + " ")[1].split(";")[0].split(" ")[0])

    assert count("reach checks") >= 100000, tail
    # the soundness check must notice a reach reported one too small
    assert count("reach-1 patterns") >= 20 and count("under-reported reach caught") >= 20, tail
    for label in ("two-outcome checks", "dense two-outcome checks", "class-repeat chain checks", "two-unit checks"):
        assert count(label) >= 1000, (label, tail)
    assert count("strict programs") >= 5, tail
