"""Record tests/golden/schedule_cases.json on an H100: for every case of tests/test_schedule_gpu.py, the launches of one
eager training call and the sha256 of its outputs' bytes, with the device's name and SM count.  Run it with the build
whose schedule the tests pin (the file was written by the build before the side-stream reorder of the backward pass).

    python tests/golden/gen_schedule_golden.py [OUT]
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "stanford-ctc_b200"), os.path.join(ROOT, "tests")]


def main():
    import torch
    torch.cuda.set_device(0)
    from test_schedule_gpu import CASES, run_case
    props = torch.cuda.get_device_properties(0)
    out = {"device": props.name, "sms": props.multi_processor_count, "cases": {}}
    for name in CASES:
        launches, dig = run_case(name)
        out["cases"][name] = {"launches": launches, "outputs": dig}
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "schedule_cases.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
