"""Multi-GPU parity check (run under torchrun on N GPUs): the SdBG stream / edges / counting produced by the
bucket-range partitioned build must be bit-identical to the reference fixtures (megahit_b200.multigpu.parity_check,
the same check bench.py --gpus N runs before timing)."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from megahit_b200 import lib, multigpu  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
lib.load().mhb_set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
import subprocess
import tempfile
tmp = [tempfile.mkdtemp(prefix="mhb_mgpu_") if rank == 0 else None]
dist.broadcast_object_list(tmp, src=0)
res = multigpu.parity_check(dev, verbose=True, files_dir=tmp[0])
# downstream acceptance of the multi-file output: the reference's `assemble` reads P.sdbg.<0..N-1> + P.sdbg_info
REF = os.path.join(ROOT, "oracle", "_ref", "megahit_core_ref")
if rank == 0 and os.path.exists(REF):
    ASM = ["--min_standalone", "300", "--prune_level", "2", "--merge_len", "20", "--merge_similar", "0.95", "--cleaning_rounds",
           "5", "--disconnect_ratio", "0.1", "--low_local_ratio", "0.2", "--min_depth", "2", "--bubble_level", "2",
           "--max_tip_len", "-1", "--careful_bubble"]
    for c in res["cases"]:
        if not c["case"].startswith("syn150_k27") and not c["case"].startswith("lowcov"):
            continue
        name, k = c["case"].rsplit("-k", 1)
        case = os.path.join(ROOT, "tests", "golden", name)
        m = json.load(open(os.path.join(case, "golden.json")))["m"]
        rp = os.path.join(tmp[0], "ref_" + c["case"])
        subprocess.run([REF, "count", "-k", k, "-m", str(m), "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", rp,
                        "--num_cpu_threads", "4", "--read_lib_file", os.path.join(case, "reads.lib")], check=True, capture_output=True)
        subprocess.run([REF, "seq2sdbg", "--host_mem", "1e9", "--mem_flag", "1", "--output_prefix", rp, "--num_cpu_threads", "4",
                        "-k", k, "--kmer_from", "0", "--input_prefix", rp, "--need_mercy"], check=True, capture_output=True)
        outs = []
        for tag, p in (("ref", rp), ("ours", c["prefix"])):
            cp = os.path.join(tmp[0], f"contigs_{tag}_{c['case']}")
            r = subprocess.run([REF, "assemble", "-s", p, "-o", cp, "-t", "1"] + ASM, capture_output=True, text=True)
            outs.append((r.returncode, open(cp + ".contigs.fa", "rb").read() if r.returncode == 0 else r.stderr[-500:]))
        c["assemble"] = bool(outs[0][0] == 0 and outs[1][0] == 0 and outs[0][1] == outs[1][1] and len(outs[1][1]) > 0)
        res["ok"] = bool(res["ok"] and c["assemble"])
        print("reference assemble on the", world, "file SdBG of", c["case"], "->", "identical contigs" if c["assemble"] else outs, flush=True)
if rank == 0:
    os.makedirs(os.path.join(ROOT, "scripts", "out"), exist_ok=True)
    json.dump(res, open(os.path.join(ROOT, "scripts", "out", f"mgpu_parity_n{world}.json"), "w"), indent=1)
    print("MGPU PARITY", "PASS" if res["ok"] else "FAIL", flush=True)
dist.destroy_process_group()
sys.exit(0 if res["ok"] else 1)
