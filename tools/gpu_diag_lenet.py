"""GPU diagnostic: run every numerics self-check and print name / error / tolerance."""
import os
import sys
import traceback

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from distributedmnist_b200.ops import selfcheck  # noqa: E402


def main():
    os.makedirs("results", exist_ok=True)
    lines = []
    only = sys.argv[1:]
    for fn in selfcheck.ALL_CHECKS:
        if only and not any(o in fn.__name__ for o in only):
            continue
        try:
            for (name, err, tol) in fn():
                lines.append("%-44s err=%-12.5g tol=%-10.3g %s" % (name, err, tol, "ok" if err <= tol else "FAIL"))
            torch.cuda.synchronize()
        except Exception:  # noqa: BLE001
            lines.append("%s EXCEPTION\n%s" % (fn.__name__, traceback.format_exc()))
        print(lines[-1] if lines else "", flush=True)
    txt = "\n".join(lines)
    print("=" * 80 + "\n" + txt)
    open("results/lenet_diag.txt", "w").write(txt + "\n")


if __name__ == "__main__":
    main()
