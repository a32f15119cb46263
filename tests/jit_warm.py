"""Plans the GPU parity tests run on plan-specialised (run-time compiled) kernels, and a parallel warm-up of the on-disk
kernel cache (b2_plan_precompile: NVRTC only, no GPU needed).  Each specialised kernel costs 5-15 s of NVRTC time; the
tests use ~70 of them one after the other.  __graft_entry__.build() compiles them here (the cache travels to the GPU box
with the library) and the GPU test session warms whatever is still missing on all host cores before the first test.

Test infrastructure: the recording `run` below answers with the oracle so that the check_* helpers walk all their plans."""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

import scenarios as sc
from tikv_b200 import ffi


def test_plans():
    import orc
    plans = []

    def rec(plan, ranges=None, region=None):
        plans.append(plan)
        return orc.dag_handle(plan, ranges if ranges is not None else sc.WHOLE, region)

    for fam in (sc.scalar_plans, sc.in_plans, sc.multi_group_plans, sc.real_sum_plans):
        plans += [p for _, p in fam()]
    plans += [p for n, p in sc.projection_plans() if n == "proj_real_chain"]
    plans += [p for n, p in sc.plans() if n in ("scan_all", "sel_lt_const", "count_star", "group_by_small", "group_filter_offsets")]
    plans += [p for n, p in sc.int_plans() if n in ("const_on_left", "eq_ne", "agg", "topn")]
    sc.check_like_known_answers(rec)
    plans += [p for n, p in sc.mixed_plans() if "like" in n or "decimal" in n]
    sc.check_scalar_known_answers(rec, error_labels=("int_divide(-9223372036854775808,-1)", "neg_uint(9223372036854775809)", "abs(-9223372036854775808)"))
    import test_gpu_group_tables
    plans += [p for _, p in test_gpu_group_tables.race_plans()]
    for fx in sc.reference_executor_fixtures():
        if fx[0] in ("hash_agg_fast_v2", "topn_integration_3", "topn_unsigned_col0_desc"):
            plans.append(fx[2])
    return plans


def warm_shard(plans, shard, n_shards):
    """Compile every n_shards-th plan into the on-disk cache.  Returns (compiled now, failures)."""
    L = ffi.lib()
    done, errs = 0, []
    for p in plans[shard::n_shards]:
        n = C.c_int32(0)
        if L.b2_plan_precompile(C.byref(p.c), C.byref(n)) == 0:
            done += n.value
        else:
            errs.append(L.b2_last_error_message().decode())
    return done, errs


def _host_gib():
    """GiB of host memory available (MemAvailable)."""
    try:
        for line in open("/proc/meminfo"):
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) >> 20
    except OSError:
        pass
    return 8


def warm(extra_modules=(), workers=None):
    """Warm the cache for test_plans() in `workers` processes (NVRTC serialises compilations inside one process)."""
    workers = workers or max(1, min(32, len(os.sched_getaffinity(0)), _host_gib() // 4))  # NVRTC takes up to a few GiB per compile
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests"), os.environ.get("PYTHONPATH", "")]))
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), str(i), str(workers)], env=env, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
             for i in range(workers)]
    done, errs = 0, []
    for p in procs:
        out, err = p.communicate()
        if p.returncode != 0:
            errs.append(err[-400:])
            continue
        last = out.strip().splitlines()[-1].split(" ", 1)
        done += int(last[0])
        if len(last) > 1 and last[1]:
            errs.append(last[1])
    return done, errs


if __name__ == "__main__":
    if len(sys.argv) < 3:  # python tests/jit_warm.py [workers]: warm everything from here
        sys.path.insert(0, ROOT)
        print(warm(workers=int(sys.argv[1]) if len(sys.argv) > 1 else None))
    else:
        d, e = warm_shard(test_plans(), int(sys.argv[1]), int(sys.argv[2]))
        print(d, e[0][:300].replace("\n", " ") if e else "")
