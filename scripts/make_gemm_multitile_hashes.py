"""Writes tests/golden/gemm_epilogue_multitile_sha256.json: the SHA-256 of every output of the seeded multi-tile GEMM
launches in tests/gemm_multitile_cases.py, run on cuda:0 through the given build of the library.  Generate it from the
build whose epilogue bits are the standard, then check a change against it with
tests/test_gemm_epilogue_multitile_gpu.py.

    python scripts/make_gemm_multitile_hashes.py path/to/libvfeat.so [out.json]
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import gemm_epilogue_cases as gc  # noqa: E402
import gemm_multitile_cases as mc  # noqa: E402


def main():
    lib_path = sys.argv[1]
    out = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "tests", "golden",
                                                             "gemm_epilogue_multitile_sha256.json")
    dev = torch.device("cuda", 0)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    hashes = mc.all_hashes(gc.open_lib(lib_path), dev)
    doc = {"device": torch.cuda.get_device_name(dev), "sm_count": sms, "sha256": hashes}
    with open(out, "w") as fh:
        json.dump(doc, fh, indent=1, sort_keys=True)
        fh.write("\n")
    print(f"{len(hashes)} launches -> {out}")


if __name__ == "__main__":
    main()
