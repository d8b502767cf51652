"""Worker of test_kernel_selection in test_gpu_format_limits.py and test_gpu_mctf_limits.py: runs every case of the module's kernel_selection_cases() once
under torch.profiler, in a process of its own, and prints one JSON line per case: {"case": label, "ok": the case's expectation holds, "kernels": names of the
kernels in the trace}.
usage: python tests/_kernel_selection_run.py [test module, default test_gpu_format_limits]"""
import importlib, json, os, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch
import vvenc_b200 as V
import test_gpu_format_limits as F


def main():
    assert torch.cuda.is_available(), 'needs cuda:0'
    T = importlib.import_module(sys.argv[1] if len(sys.argv) > 1 else 'test_gpu_format_limits')
    eng = V.CostEngine(0)
    for label, setup in T.kernel_selection_cases():
        call, expect = setup(eng)
        _, names = F.kernel_names(call)
        names = sorted({n for n in names if '_kernel' in n})
        print(json.dumps({'case': label, 'ok': bool(expect(names)), 'kernels': names}), flush=True)
    eng.close()


if __name__ == '__main__':
    main()
