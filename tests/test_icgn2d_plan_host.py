"""CPU: the 2D launch plans (ocb::icgn2d_plan and ocb::nr2d1_plan, opencorr_b200/csrc/ocb_kernels.h) compiled for the host.
Every case of test_gpu_2d_geometry.py must land in the kernel instantiation, lane layout and row split it is meant to cover;
run with -s to see the plan of each case."""
import re

import test_gpu_2d_geometry as geometry


def test_icgn2d_plan_covers_every_branch(tmp_path):
    exe = geometry.build_plan_tool(str(tmp_path))
    out = geometry.run_plan_tool(exe)
    print(out.stdout)
    assert out.returncode == 0, out.stdout
    planned = set()
    for m in re.finditer(r"np=(\d+) r=\((\d+),(\d+)\) lm=(\d) wpp=(\d) n=\S+: (kernel (<[\d,]+>), .*?remainder (\S+),|rejected)", out.stdout):
        np_, rx, ry, lm, wpp = (int(v) for v in m.groups()[:5])
        planned.add((np_, rx, ry, lm, wpp))
    # every ICGN2D / ICLM2D case the GPU file runs is in the checked table
    missing = [c for c in geometry.ICGN2D_PLAN_CASES if c not in planned]
    assert not missing, "cases of test_gpu_2d_geometry.py without a checked plan (np, rx, ry, lm, wpp): %s" % missing
    nr = {(int(a), int(b)) for a, b in re.findall(r"^nr .*?r=\((\d+),(\d+)\)", out.stdout, re.M)}
    missing = [r for r in geometry.NR2D_PLAN_CASES if tuple(r) not in nr]
    assert not missing, "NR2D1 radii of test_gpu_2d_geometry.py without a checked plan: %s" % missing
    # every branch is reached: the twelve pair instantiations, remainders 0-3 in both warps, idle lanes and tail columns,
    # NR2D1 CTAs of 4, 2 and 1 warps with and without a tail, rejection
    kernels = set(re.findall(r"kernel (<[\d,]+>)", out.stdout))
    assert kernels == {"<%d,%d,%d,%d>" % (np_, rc, lm, w) for np_, rc, lm in
                       ((6, 0, 0), (6, 16, 0), (12, 0, 0), (12, 20, 0), (6, 0, 1), (12, 0, 1)) for w in (1, 2)}, kernels
    rems = re.findall(r"remainder (\d)/(\d)", out.stdout)
    assert {int(a) for a, _ in rems} == {0, 1, 2, 3} and {int(b) for _, b in rems} == {0, 1, 2, 3}
    assert re.search(r"[1-9]\d* idle lane", out.stdout) and re.search(r"[1-9]\d* tail column", out.stdout)
    nr_kinds = set(re.findall(r"(\d) warp\(s\) per CTA, \d+ CTA/SM, (\d+) tail", out.stdout))
    assert {(w, t != "0") for w, t in nr_kinds} == {(w, t) for w in "421" for t in (False, True)}, nr_kinds
    assert out.stdout.count("rejected") >= 2
