#!/bin/bash
# Instruction histograms (cuobjdump -sass) of the kernels the roofline accounting rests on -> profiles/
# usage: tools/sass_hist.sh [round-tag]
set -e
tag=${1:-r02}
mkdir -p profiles
obj=noble-curves_b200/build/inst_bls381g1.o
hist() { grep -oE "^\s+/\*[0-9a-f]+\*/\s+[A-Z0-9_.]+" | awk '{print $2}' | sort | uniq -c | sort -rn; }
fn() { cuobjdump -sass "$obj" | awk -v pat="$1" '/Function : /{on=($0 ~ pat)} on'; }
{
  echo "# cuobjdump -sass $obj  (sm_90a, built by make -C noble-curves_b200)  -- k_accumulate<CurveBls381G1>"
  echo "# whole function (kernel body + the out-of-line mul_call / sqr_call subroutines it carries)"
  fn "k_accumulateINS_13CurveBls381G1E" | hist
} > profiles/${tag}_sass_k_accumulate_hist.txt
# mul_call / sqr_call: the subroutines are laid out after the kernel body; split at the RET instructions
python3 - "$obj" "$tag" <<'PY'
import re, subprocess, sys, collections
obj, tag = sys.argv[1], sys.argv[2]
sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
m = re.search(r"Function : (\S*k_accumulateINS_13CurveBls381G1E\S*)(.*?)(?=Function : |\Z)", sass, re.S)
lines = [l for l in m.group(2).splitlines() if re.match(r"\s+/\*[0-9a-f]{4}\*/", l)]
ops = [re.match(r"\s+/\*([0-9a-f]+)\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", l) for l in lines]
ops = [(int(o.group(1), 16), o.group(2)) for o in ops if o]
# segments: [start, first EXIT/RET ...]; find call targets
targets = sorted({int(t, 16) for t in re.findall(r"CALL\.REL\.NOINC\s+0x([0-9a-f]+)", m.group(2))})
out = open(f"profiles/{tag}_sass_mul_call_bls381.txt", "w")
out.write(f"# {obj}: out-of-line field subroutines inside k_accumulate<CurveBls381G1> (call targets of CALL.REL.NOINC)\n")
out.write("# mont_mul<FpBls381> = 2N^2+N = 300 IMAD.WIDE-equivalents for N = 12; mont_sqr = 234 (field.cuh)\n")
bounds = targets + [ops[-1][0] + 16]
body = collections.Counter(op for a, op in ops if a < targets[0]) if targets else collections.Counter()
out.write(f"\n## kernel body (before the first subroutine, {sum(body.values())} instructions)\n")
for op, c in body.most_common(): out.write(f"{c:7d} {op}\n")
for k, t in enumerate(targets):
    seg = collections.Counter(op for a, op in ops if t <= a < bounds[k + 1])
    wide = sum(c for op, c in seg.items() if op.startswith("IMAD.WIDE"))
    out.write(f"\n## subroutine at 0x{t:x} ({sum(seg.values())} instructions, {wide} IMAD.WIDE*)\n")
    for op, c in seg.most_common(): out.write(f"{c:7d} {op}\n")
PY
echo "wrote profiles/${tag}_sass_k_accumulate_hist.txt profiles/${tag}_sass_mul_call_bls381.txt"
