"""Op-level determinism / correctness probe of the tensor-core encoder attention: the same QKV through the
kernel several times, against the SIMT kernel.
    python tools/attention_probe.py"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sam_road_b200 import _lib  # noqa: E402

DEV = "cuda:0"


def main():
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    out_all = {}
    for (B, s, win, heads, hd) in ((64, 16, 14, 12, 64), (64, 16, 16, 12, 64), (64, 32, 14, 12, 64), (16, 32, 32, 12, 64),
                                   (64, 16, 14, 16, 80), (64, 16, 16, 16, 80)):
        D = heads * hd
        g = torch.Generator().manual_seed(11)
        qkv16 = (torch.randn(B * s * s, 3 * D, generator=g) * 1.5).to(torch.float16).to(DEV)
        bias = (0.5 * torch.randn(3 * D, generator=g)).to(torch.float16).float().to(DEV)
        rel_h = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)
        rel_w = (0.3 * torch.randn(2 * win - 1, hd, generator=g)).to(DEV)

        def run(simt, hot):
            lib.samroad_debug_force_simt_attention(simt)
            out = torch.full((B * s * s, D), float("nan"), dtype=torch.float16, device=DEV)
            if hot:                      # rewrite the input right before: the kernel starts on L2-resident lines
                qkv16.copy_(qkv16.clone())
            _lib.check(lib.samroad_op_attention(qkv16.data_ptr(), bias.data_ptr(), rel_h.data_ptr(), rel_w.data_ptr(),
                                                B, s, win, heads, hd, out.data_ptr(), st), "attention")
            return out.float()

        ref = run(1, False)
        res = {}
        for hot in (False, True):
            outs = [run(0, hot) for _ in range(24)]
            torch.cuda.synchronize()
            res[f"hot{int(hot)}"] = {
                "runs_differing_from_first": sum(int(not torch.equal(outs[0], o)) for o in outs[1:]),
                "max_elems_differing": max(int((outs[0] != o).sum()) for o in outs[1:]),
                "max_err_vs_simt": max(float((o - ref).abs().max()) for o in outs),
                "nan": any(bool(torch.isnan(o).any()) for o in outs)}
        out_all[f"B{B}_s{s}_win{win}_hd{hd}"] = res
        print(f"B{B}_s{s}_win{win}_hd{hd}", json.dumps(res), flush=True)
    lib.samroad_debug_force_simt_attention(0)
    json.dump(out_all, open("gpurun_out/attention_probe.json", "w"), indent=1)


if __name__ == "__main__":
    main()
