"""Driver contract checks that do not need a GPU."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_contract_on_cpu():
    """Without a GPU the reference arm says so (one JSON line, exit 0); with ``--allow_cpu --tiny`` the same code path —
    HuggingFace GPT2DoubleHeadsModel + torch DDP + AdamW + clip, the reference's step body — runs over gloo and prints
    the full bench line without importing anything of this repository."""
    import torch

    base = [sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "1", "--steps", "2", "--warmup", "1"]
    if not torch.cuda.is_available():
        r = subprocess.run(base, capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr
        rec = json.loads(r.stdout.strip().splitlines()[-1])
        assert rec["impl"] == "reference" and "unavailable" in rec and len(rec["unavailable"]) > 20
    import socket

    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    r = subprocess.run(base + ["--tiny", "--allow_cpu", "--seq", "32"], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES="", MASTER_PORT=str(port)))
    assert r.returncode == 0, r.stderr[-2000:]
    rec = json.loads(r.stdout.strip().splitlines()[-1])
    assert rec["impl"] == "reference" and rec["metric"] == "gpt2_small_ddp_train_tokens_per_sec" and rec["value"] > 0
    assert rec["repo_code_on_path"] is False and "GPT2DoubleHeadsModel" in rec["reference_class"]
    assert rec["e2e"]["h2d_bytes_per_step"] > 0 and rec["e2e"]["d2h_bytes_per_step"] == 4
    assert rec["hyperparameters_from"]


def test_graft_entry_build_and_exports():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g

    g.build()
    from adapcc_b200.runtime.native import lib_path, load_library

    lib = load_library(build_if_missing=False)
    assert os.path.exists(lib_path())
    for sym in ("initThreads", "exitThreads", "allreduce", "reduce", "boardcast", "updateActive", "adapcc_allreduce",
                "adapcc_tree_collective", "adapcc_tree_relay_persistent", "adapcc_profile_links",
                "adapcc_detect_topology", "adapcc_fused_adamw", "adapcc_fused_ce", "adapcc_moe_exchange",
                "adapcc_alltoall", "adapcc_ln_fwd", "adapcc_pool_alloc"):
        assert hasattr(lib, sym), sym


def test_shipped_strategies_parse_and_validate():
    from adapcc_b200.strategy import Strategy

    d = os.path.join(ROOT, "strategy")
    files = [f for f in os.listdir(d) if f.endswith(".xml")]
    assert len(files) >= 10
    for f in files:
        s = Strategy.from_file(os.path.join(d, f), None)
        assert s.trees
        world = len(s.ranks())
        s.validate(world)


def test_sass_of_the_built_library_contains_the_hardware_paths():
    """The evidence the design rests on, checked on the build box (cuobjdump needs no GPU): in-switch reductions
    (LDGMC = multimem.ld_reduce), multicast stores, 128-bit peer accesses, system-scope release/acquire flags, and the
    tensor-core path of the GEMM (HGMMA = wgmma, UTMALDG = TMA load, .MULTICAST = cluster multicast, SYNCS.PHASECHK =
    mbarrier wait, USETMAXREG = setmaxnreg)."""
    import re
    import shutil
    import subprocess

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    from adapcc_b200.build import build

    lib = build()
    sass = subprocess.run(["cuobjdump", "-sass", str(lib)], capture_output=True, text=True, timeout=600).stdout
    assert "sm_90a" in sass
    blocks = dict(zip(re.findall(r"Function : (\S+)", sass), re.split(r"\n\s*Function : \S+\n", sass)[1:]))

    def ops_of(substr):
        text = "\n".join(b for n, b in blocks.items() if substr in n)
        assert text, f"no kernel matching {substr}"
        return text

    direct = ops_of("allreduce_direct_kernel")
    for m in ("LDGMC", "STG.E.128.STRONG.SYS", "LDG.E.NA.128", "MEMBAR.ALL.SYS", "CCTL.IVALL"):
        assert m in direct, m
    tree = ops_of("tree_collective_kernel")
    assert "LDG.E.64.STRONG.SYS" in tree and "STG.E.64.STRONG.SYS" in tree          # 64-bit chunk tokens
    gemm = ops_of("gemm_bias_act_wgmma")
    for m in ("HGMMA.64x256x16.F32.BF16", "UTMALDG.2D", "UTMALDG.2D.MULTICAST", "SYNCS.PHASECHK", "USETMAXREG"):
        assert m in gemm, m
    assert "STG.E.128.STRONG.SYS" in ops_of("zero_adamw_bcast_kernel")              # parameters leave through multimem.st
    assert "LD.E.128.STRONG.SYS" in ops_of("allreduce_ll_kernel") or "LDG.E.128.STRONG.SYS" in ops_of("allreduce_ll_kernel")


def test_drop_in_import_shims():
    """``from adapcc import *`` (how the reference's train_ddp.py imports the library) and ``python launcher.py``."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = "import sys; sys.path.insert(0, %r); from adapcc import *; print(AdapCC.__name__, ALLREDUCE, REDUCE, BOARDCAST, DETECT, PROFILE)" % root
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.split() == ["AdapCC", "0", "1", "2", "6", "7"], out.stderr[-500:]
    out = subprocess.run([sys.executable, os.path.join(root, "launcher.py"), "--num-process", "2", "--ips", "127.0.0.1:2",
                          "--exec-file", "train_ddp.py", "--dry-run"], capture_output=True, text=True, timeout=120, cwd=root)
    assert out.returncode == 0 and "torch.distributed.run" in out.stdout, out.stderr[-500:]


def test_launch_report_tool_on_a_sample_ncu_csv(tmp_path):
    """tools/launch_report.py: ncu launch list (CSV with ==PROF== noise lines, mixed units) -> per-family table of the
    last step, our kernels marked."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    rows = ['==PROF== Connected to process 1', '"ID","Kernel Name","Metric Name","Metric Unit","Metric Value"']
    k = 0
    for step in range(2):
        for name, unit, val in (("void adapcc::ln_fwd_kernel<3, true>(const __nv_bfloat16*)", "us", "12.5"),
                                ("nvjet_tst_192x256_64x5_2x2_2cta_v_bz_NNT", "us", "30.0"),
                                ("void at::native::vectorized_elementwise_kernel<4, F>(int)", "ns", "7,500"),
                                ("void adapcc::adamw_kernel<__nv_bfloat16, __nv_bfloat16>(float*)", "ms", "0.5")):
            rows.append(f'"{k}","{name}","gpu__time_duration.sum","{unit}","{val}"')
            k += 1
    src = tmp_path / "launches.csv"
    src.write_text("\n".join(rows) + "\n")
    out = tmp_path / "report.md"
    r = subprocess.run([sys.executable, os.path.join(root, "tools", "launch_report.py"), str(src), "2", str(out), "sample"],
                       capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-500:]
    text = out.read_text()
    assert "the last step (4 launches, 0.55 ms" in text
    assert "**adapcc::adamw_kernel** (ours) | 1 | 0.500" in text and "**adapcc::ln_fwd_kernel** (ours) | 1 | 0.013" in text
    assert "Our kernels: 93.2%" in text
