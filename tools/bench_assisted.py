"""Time speculative decoding with a draft model (rmu_decoder_generate_assisted) against plain generation, in one run:

    python tools/bench_assisted.py [--target qwen3-32b,llama-3.1-8b | llama-3.1-70b] [--tokens 256] [--prompt 1024]
                                   [--ks 1,3,7,15] [--runs 3] [--layers N] [--draft-weights split,nf4]
                                   [--no-ceiling] [--json OUT]

Pairs, at full depth with seeded weights drawn on the device (tools/bench_generate.SeededLayers): Qwen3-32B (NF4) with
a Qwen3-0.6B draft, split and NF4; Llama-3.1-8B (NF4) with a Llama-3.2-3B draft (NF4); --target llama-3.1-70b adds
Llama-3.1-70B (NF4) with the Llama-3.2-3B draft.  Workload: a prompt of --prompt tokens and --tokens new tokens,
greedy and sampled at the reference's temperature 0.2, top-p 0.9 and repetition penalty 1.1.  Every call is timed
with the host clock around the whole call, which ends in a device synchronise; each figure is the median of --runs
warmed calls.

Measured, per pair and setting:
* the target's prefill (a one-token call) and plain step ((a --tokens call - the one-token call) / (tokens - 1));
* the target's verify pass at each k: rmu_debug_generate_drafts fed the plain reply as its drafts, so every pass keeps
  k + 1 tokens; (call - prefill) / passes;
* the draft's prefill and single-row step (its own plain generate), and its two-row pass (rmu_debug_generate_drafts
  at k = 1 on the draft): the draft chain's step and its steady-state catch-up;
* end to end, alternated with plain rmu_decoder_generate in the same process: a second handle of the target's own
  weights as the draft (every draft kept: the ceiling of the mechanics; skipped when two targets do not fit), and the
  small draft of another seed (nearly every draft rejected: the worst case).  Each reply's tokens must equal plain's.

Computed (labelled so): the draft's share of a pass, (worst-case call - both prefills) / passes - verify(k), and the
tokens per second a pass of k drafts gives at per-token acceptance rates between the two measured extremes, with the
expected tokens per pass (1 - a^(k+1)) / (1 - a).  Acceptance on real checkpoints needs their weights, which this run
does not hold: it is reported as "not measured".  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import gc
import json
import os
import statistics
import sys
import time
from dataclasses import replace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_generate import SeededLayers, card  # noqa: E402

DRAFTS = {"qwen3-32b": ("qwen3-0.6b", ("split", "nf4")), "llama-3.1-8b": ("llama-3.2-3b", ("nf4",)),
          "llama-3.1-70b": ("llama-3.2-3b", ("nf4",))}
RATES = (0.5, 0.7, 0.8, 0.9)


def handle(shape, weights, seed, layers=None):
    """a decoder of the preset shape with seeded weights and LM head, split or NF4 -> (config, encoder)"""
    from ragmeup_b200 import _lib
    from ragmeup_b200.encoder import BertEncoder
    from ragmeup_b200.weights import decoder_config
    cfg = replace(decoder_config("synthetic:" + shape), name=shape)
    if layers:
        cfg = replace(cfg, layers=min(layers, cfg.layers))
    src = SeededLayers(cfg, seed=seed)
    if weights == "nf4":
        enc = BertEncoder.nf4_decoder(src)
    else:
        w = dict(src.globals())
        for l in range(cfg.layers):
            w.update(src.layer(l))
        enc = BertEncoder(cfg, w, with_head=False)
        del w
    lm = SeededLayers(cfg, seed=seed + 100)._draw(0, [("lm_head", (cfg.vocab_size, cfg.hidden))])["lm_head"]
    _lib.check(_lib.lib().rmu_decoder_set_lm_head(enc._h, lm.ctypes.data), "rmu_decoder_set_lm_head")
    del lm
    return cfg, enc


def sampling(sampled: bool):
    from ragmeup_b200 import _lib
    return _lib.SamplingC(int(sampled), 0.2, 0.9, 1.1, 50, 0, (C.c_int32 * _lib.MAX_EOS)())


def plain(enc, ids, s, n):
    from ragmeup_b200 import _lib
    out, got = np.zeros(n, np.int32), C.c_int32(0)
    _lib.check(_lib.lib().rmu_decoder_generate(enc._h, ids.ctypes.data, len(ids), C.byref(s), 7, n, out.ctypes.data,
                                               C.byref(got), None, None), "rmu_decoder_generate")
    return out[:got.value].tolist()


def drafted(enc, ids, s, n, drafts, k):
    from ragmeup_b200 import _lib
    d = np.zeros(n, np.int32)
    d[:len(drafts)] = drafts
    out, got, passes = np.zeros(n, np.int32), C.c_int32(0), C.c_int32(0)
    _lib.check(_lib.lib().rmu_debug_generate_drafts(enc._h, ids.ctypes.data, len(ids), C.byref(s), 7, n, d.ctypes.data,
                                                    k, out.ctypes.data, C.byref(got), None, C.byref(passes), None),
               "rmu_debug_generate_drafts")
    return out[:got.value].tolist(), passes.value


def assisted(enc, draft, ids, s, n, k):
    from ragmeup_b200 import _lib
    out, got = np.zeros(n, np.int32), C.c_int32(0)
    passes, dr, kept = C.c_int32(0), C.c_int32(0), C.c_int32(0)
    _lib.check(_lib.lib().rmu_decoder_generate_assisted(enc._h, draft._h, ids.ctypes.data, len(ids), C.byref(s), 7, n,
                                                        k, 0, out.ctypes.data, C.byref(got), None, C.byref(passes),
                                                        C.byref(dr), C.byref(kept), None),
               "rmu_decoder_generate_assisted")
    return out[:got.value].tolist(), passes.value, dr.value, kept.value


def clock(fn):
    t0 = time.perf_counter()
    r = fn()
    return (time.perf_counter() - t0) * 1e3, r


def median_ms(fn, runs):
    fn()                                                    # warm
    return statistics.median(clock(fn)[0] for _ in range(runs))


def bench_pair(target, tcfg, enc, twin, draft_name, dweights, dcfg, dr, a, log):
    V = tcfg.vocab_size
    ids = np.random.default_rng(3).integers(0, V, a.prompt).astype(np.int32)
    N, runs = a.tokens, a.runs
    rows = []
    for sampled in (False, True):
        s = sampling(sampled)
        row = {"target": target, "draft": f"{draft_name} ({dweights})", "sampled": sampled}
        want = plain(enc, ids, s, N)
        t_pre = median_ms(lambda: plain(enc, ids, s, 1), runs)
        t_dpre = median_ms(lambda: plain(dr, ids, s, 1), runs)
        t_dplain = median_ms(lambda: plain(dr, ids, s, 33), runs)
        dwant = plain(dr, ids, s, 33)
        t_d2 = median_ms(lambda: drafted(dr, ids, s, 33, dwant, 1), runs)
        d2_passes = drafted(dr, ids, s, 33, dwant, 1)[1]
        row["measured_ms"] = {"target_prefill": t_pre, "draft_prefill": t_dpre,
                              "draft_step": (t_dplain - t_dpre) / 32,
                              "draft_two_row_pass": (t_d2 - t_dpre) / d2_passes}
        verify = {}
        for k in a.ks:
            toks, passes = drafted(enc, ids, s, N, want, k)
            assert toks == want
            verify[k] = (median_ms(lambda: drafted(enc, ids, s, N, want, k), runs) - t_pre) / passes
        row["measured_ms"]["verify_pass"] = verify
        # end to end, alternated with plain
        e2e = {k: {"plain": [], "ceiling": [], "worst": []} for k in a.ks}
        counts = {}
        for k in a.ks:
            for kind, d in (("ceiling", twin), ("worst", dr)):
                if d is not None:
                    toks, passes, nd, nk = assisted(enc, d, ids, s, N, k)      # warm, and the reply check
                    assert toks == want, (kind, k)
                    counts[(kind, k)] = {"passes": passes, "drafted": nd, "kept": nk}
            for _ in range(runs):
                e2e[k]["plain"].append(clock(lambda: plain(enc, ids, s, N))[0])
                for kind, d in (("ceiling", twin), ("worst", dr)):
                    if d is not None:
                        e2e[k][kind].append(clock(lambda: assisted(enc, d, ids, s, N, k))[0])
        row["end_to_end"] = {}
        row["computed"] = {}
        for k in a.ks:
            med = {kind: statistics.median(v) for kind, v in e2e[k].items() if v}
            row["end_to_end"][k] = {kind: {"ms": round(t, 1), "tok_per_s": round(N / t * 1e3, 1),
                                           **counts.get((kind, k), {})} for kind, t in med.items()}
            wc = counts[("worst", k)]
            draft_share = (med["worst"] - t_pre - t_dpre) / wc["passes"] - verify[k]
            pass_ms = verify[k] + draft_share
            row["computed"][k] = {"draft_ms_per_pass_COMPUTED": round(draft_share, 3),
                                  "tok_per_s_at_acceptance_COMPUTED": {
                                      str(r): round((1 - r ** (k + 1)) / (1 - r) / pass_ms * 1e3, 1) for r in RATES},
                                  "plain_tok_per_s_COMPUTED": round(1e3 / ((med["plain"] - t_pre) / (N - 1)), 1)}
        row["measured_ms"] = json.loads(json.dumps(row["measured_ms"], default=float))
        row["acceptance_on_real_checkpoints"] = "not measured"
        log(row)
        rows.append(row)
    return rows


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--target", default="qwen3-32b,llama-3.1-8b")
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--prompt", type=int, default=1024)
    ap.add_argument("--ks", default="1,3,7,15")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--layers", type=int, default=None, help="fewer layers per model (a rehearsal, not the table)")
    ap.add_argument("--draft-weights", default=None, help="split and / or nf4 (default: the pair's list)")
    ap.add_argument("--no-ceiling", action="store_true", help="skip the second handle of the target's weights")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    a.ks = [int(k) for k in a.ks.split(",")]
    res = {"card": card(), "tokens": a.tokens, "prompt": a.prompt, "layers": a.layers or "full", "rows": []}
    print(json.dumps(res["card"]), flush=True)

    def log(row):
        print(json.dumps(row), flush=True)

    for target in a.target.split(","):
        draft_name, dweights_all = DRAFTS[target]
        t0 = time.perf_counter()
        tcfg, enc = handle(target, "nf4", 0, a.layers)
        twin = None
        if target != "llama-3.1-70b" and not a.no_ceiling:
            twin = handle(target, "nf4", 0, a.layers)[1]
        print(json.dumps({"loaded": target, "s": round(time.perf_counter() - t0, 1)}), flush=True)
        for dweights in (a.draft_weights.split(",") if a.draft_weights else dweights_all):
            dcfg, dr = handle(draft_name, dweights, 1, a.layers)
            res["rows"] += bench_pair(target, tcfg, enc, twin, draft_name, dweights, dcfg, dr, a, log)
            del dr
            gc.collect()
        del enc, twin
        gc.collect()
        torch.cuda.empty_cache()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1, default=float)


if __name__ == "__main__":
    main()
