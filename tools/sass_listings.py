"""Writes profiles/sass/<kernel>.sass: the full ``cuobjdump -sass`` listing of ONE instantiation per hot kernel family
(the one the GPT-2 bench / the sweeps actually launch), so the instruction-level evidence — NVLS multimem ops, peer
128-bit loads/stores, system-scope flag protocol, wgmma / TMA / mbarrier — can be read next to the counts in
profiles/sass_summary.md. Run on the build box (no GPU needed): ``python tools/sass_listings.py``."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "adapcc_b200", "_C", "libadapcc.so")
# (file name, regex on the demangled name): first match wins
WANT = [
    ("allreduce_direct_nvls_bf16", r"allreduce_direct_kernel<__nv_bfloat16, __nv_bfloat16, 0, 3, 2>"),
    ("allreduce_direct_two_shot_bf16_8", r"allreduce_direct_kernel<__nv_bfloat16, __nv_bfloat16, 0, 2, 8>"),
    ("allreduce_direct_one_shot_f32_8", r"allreduce_direct_kernel<float, float, 0, 1, 8>"),
    ("allreduce_ll_f32", r"allreduce_ll_kernel<float, 0>"),
    ("broadcast_direct_bf16", r"broadcast_direct_kernel<__nv_bfloat16, __nv_bfloat16>"),
    ("alltoall_bf16", r"alltoall_kernel<__nv_bfloat16>"),
    ("tree_collective_f32", r"tree_collective_kernel<float, float, 0>"),
    ("tree_relay_persistent_bf16", r"tree_relay_persistent_kernel<__nv_bfloat16, 0>"),
    ("allreduce_pipelined_two_shot_f32", r"allreduce_pipelined_kernel<float, float, 0, 2, 8>"),
    ("zero_adamw_bcast", r"zero_adamw_bcast_kernel"),
    ("moe_push", r"moe_push_kernel"),
    ("gemm_cluster_gelu", r"gemm_bias_act_wgmma_kernel<256, 1, 2>"),
    ("gemm_cluster_dgelu", r"gemm_bias_act_wgmma_kernel<256, 2, 2>"),
    ("adamw_bf16", r"adamw_kernel<__nv_bfloat16, __nv_bfloat16>"),
    ("fused_ce_smem", r"fused_ce_smem_kernel"),
    ("embed_bwd_scatter", r"embed_bwd_scatter_kernel"),
    ("ln_fwd", r"\bln_fwd_kernel"),
]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    mangled = re.findall(r"Function : (\S+)", sass)
    names = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True).stdout.splitlines()
    blocks = re.split(r"\n\s*Function : \S+\n", sass)[1:]
    out_dir = os.path.join(ROOT, "profiles", "sass")
    os.makedirs(out_dir, exist_ok=True)
    index = ["# SASS listings (cuobjdump -sass adapcc_b200/_C/libadapcc.so, sm_90a), one instantiation per kernel family", ""]
    for fname, pat in WANT:
        for name, body in zip(names, blocks):
            if re.search(pat, name):
                lines = [ln.rstrip() for ln in body.splitlines()
                         if re.match(r"\s+/\*[0-9a-f]{4}\*/", ln) or ln.strip().startswith(".L_")]
                # keep the instruction column only (drop the encoding comment): smaller and diff-friendly
                lines = [re.sub(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", "", ln) for ln in lines]
                with open(os.path.join(out_dir, fname + ".sass"), "w") as f:
                    f.write(f"// {name}\n" + "\n".join(lines) + "\n")
                ops = re.findall(r"/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_.]+)", "\n".join(lines))
                key = [o for o in sorted(set(ops)) if re.match(r"LDGMC|UTC|UTMA|LDTM|SYNCS|MEMBAR|REDG|ATOMG|MUFU|CCTL|UCGABAR|STG\.E\.128|LDG\.E\..*128", o)]
                index.append(f"* `{fname}.sass` — `{name[:110]}`: {len(lines)} lines; notable: {', '.join(key[:14])}")
                break
        else:
            index.append(f"* {fname}: no instantiation matching /{pat}/ in the library")
    with open(os.path.join(out_dir, "README.md"), "w") as f:
        f.write("\n".join(index) + "\n")
    print("\n".join(index))


if __name__ == "__main__":
    sys.exit(main())
