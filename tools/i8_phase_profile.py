#!/usr/bin/env python
"""
Phase split of the int8 decode-GEMM (tag 210) launches of the flagship token, from the in-kernel timeline stamps of the
bring-up build:

    EXL3B_LIB_SUFFIX=_dbg EXL3B_TC_DEBUG=1 python -m exllamav3_b200.build
    python tools/i8_phase_profile.py --library exllamav3_b200/libexl3b200_dbg.so [--reps 20] [--replay] [--out FILE]

Default (isolated): runs the launches of one Llama-3.1-8B layer as bench.py issues them (q+k+v fan-out, o, gate+up
exl3_mgemm, down) and the lm_head, each `reps` times after a warm-up, each launch alone after a synchronize, with the
timeline buffer set (exl3b_debug_tc_timeline).  Per CTA it splits a launch into
    ramp      kernel start -> the first decode warp has its first unit's weights   (stamps 0 -> 3)
      prologue  kernel start -> end of the CTA's row transform (bar.sync 2)        (stamps 0 -> 2)
      digits    prologue end -> the first unit's weights and digits (W_FULL)      (stamps 2 -> 4)
    steady    decode and MMA of the CTA's units, up to the last unit's MMAs        (stamps 3 -> 10)
    tail      epilogue and split-K exchange                                         (stamps 10 -> 8)
and prints one JSON line per launch with the median and the max over CTAs (pooled over the repetitions), in microseconds
(%globaltimer), plus the steady time per unit: the median steady time over the mean units per CTA.  Under "turns" it shows how
the two decode groups' k-half wgmma batches lie against each other, from the SM clock (%clock) at the issue and the retirement
of the first 16 batches of one warp per group (slots 16-47, see turn_stats): the issue offset between the groups, the share of
batches (and of batch time) during which the other group also had a batch in flight, the batch time, the gaps between batches
inside a unit and between units, and the cycle per k-half; unit_wait_clk is the decode group's wait for a unit's weights and
digits (slots 48-55).  The decode warps' stamps are SM clocks: one clock per SM, compared only inside a CTA.
"unit_gap_split" takes a group's step between units apart (a second timeline row per CTA, see unit_gap_split).  The stamps'
own global stores lie on that path, so the timeline build's steps are longer than the production kernel's.

--replay: what a launch costs between its predecessor and its first MMA inside the token, where PDL lets a launch start
before the previous one ends.  Captures two layers' launches and the lm_head into one CUDA graph exactly as bench.py issues
them (each launch with its own timeline buffer), replays it `reps` times, and reports for the second layer's launches and
the lm_head the boundary: this launch's first W_FULL per CTA (stamp 4) minus the previous launch's last CTA end (the
maximum of stamp 8 over its CTAs); median and max over CTAs, pooled over the replays.  %globaltimer is one clock per GPU.
"""
from __future__ import annotations
import argparse, ctypes, json, os, statistics, subprocess, sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLOTS = 64                                       # u64 stamps per CTA (gemm_tc_i8_body.cuh: p.dbg[blockIdx.x * 64 + slot])


def q(v):
    return {"median": round(statistics.median(v), 2), "max": round(max(v), 2)}


def launch_name(ln):
    return "+".join(m["name"] for m in ln["mats"])


def batch_windows(row, g):
    """(issue, retire) SM clocks of decode group g's first k-half batches in one CTA's timeline row (slots 16 + 16 g + i)."""
    out = []
    for v in row[16 + 16 * g: 32 + 16 * g]:
        if not v:
            break
        v &= (1 << 64) - 1
        out.append((v & 0xffffffff, v >> 32))
    return out


def turn_stats(rows):
    """How the two decode groups' wgmma batches lie against each other, from the batch windows of one warp per group:
    offset = group 1's i-th issue minus group 0's i-th issue (clocks), overlap_batches = share of batches during more than
    half of whose issue -> retire window the other group also had a batch in flight, overlap_time = the same as a share of
    all batch time, batch = issue -> retire, gap = retire of k-half 0 -> issue of k-half 1 of the same unit (the decode of
    a k-half), unit_gap = retire of k-half 1 -> issue of the group's next unit (its weight and digit waits, the hand-off and a
    decode), cycle = mean batch + mean gap of both kinds (clocks per k-half and group)."""
    off, batch, gap, gap_unit = [], [], [], []
    n_batches = n_over = 0
    t_all = t_over = 0
    for row in rows:
        w = [batch_windows(row, 0), batch_windows(row, 1)]
        if not w[0] or not w[1]:
            continue
        t0 = w[0][0][0]
        rel = lambda t: ((t - t0 + (1 << 31)) % (1 << 32)) - (1 << 31)      # 32-bit SM clock, relative to the first issue
        w = [[(rel(s), rel(e)) for s, e in wg] for wg in w]
        off += [b[0] - a[0] for a, b in zip(w[0], w[1])]
        for g in (0, 1):
            for i, (s, e) in enumerate(w[g]):
                d = max(e - s, 1)
                o = sum(max(0, min(e, e2) - max(s, s2)) for s2, e2 in w[1 - g])
                batch.append(e - s)
                if i + 1 < len(w[g]):
                    (gap if i % 2 == 0 else gap_unit).append(w[g][i + 1][0] - e)
                n_batches += 1
                n_over += o > d / 2
                t_all += d
                t_over += min(o, d)
    if not n_batches:
        return None
    return {"offset_clk": statistics.median(off), "overlap_batches": round(n_over / n_batches, 3),
            "overlap_time": round(t_over / t_all, 3), "batch_clk": statistics.median(batch), "gap_clk": statistics.median(gap),
            "unit_gap_clk": statistics.median(gap_unit) if gap_unit else None,
            "cycle_clk": round(statistics.mean(batch) + statistics.mean(gap + gap_unit), 1) if gap + gap_unit else None}


def unit_wait(rows):
    """Median SM clocks a decode group spends in its per-unit wait for the unit's weights and digits (one mbarrier, W_FULL),
    over the first four units of each group (slots 48-55: before the wait in the low word, after it in the high word)."""
    wait = []
    for row in rows:
        for v in row[48:56]:
            if v:
                v &= (1 << 64) - 1
                wait.append(((v >> 32) - (v & 0xffffffff)) % (1 << 32))
    return statistics.median(wait) if wait else None


SPLIT_SEGMENTS = ("fences", "arrive", "handoff", "step", "wait", "digit_sums", "lds", "decode", "fence_to_mma", "total")


def words32(row):
    """A timeline row (64 signed u64 slots) as 128 u32 words, low word first."""
    out = []
    for v in row:
        v &= (1 << 64) - 1
        out += [v & 0xffffffff, v >> 32]
    return out


def unit_gap_split(att_rows):
    """A decode group's step from k-half 1 of its unit j retired to the first wgmma of unit j + 1, split into segments
    (SM clocks of one warp per group, the first four steps of each group; words 8 + 12 (4 g + j) of the second timeline
    row of each CTA, see gemm_tc_i8_body.cuh):
        fences        wgmma_wait<0> retired -> the register fences at the end of i8_unit_mma passed
        arrive        __syncwarp and the W_EMPTY arrival
        handoff       accumulator hand-offs in the step (D_EMPTY wait included), 0 for most steps
        step          the rest of the loop step up to the W_FULL wait (hand-offs excluded)
        wait          the W_FULL wait; split into wait_ready (the first probe found the phase complete) and wait_backoff
                      (the try_wait loop ran; sleep_ns is the nanosleep time in it)
        digit_sums    wait -> the digit sums in a register (the digit-sum LDS and add where they come before the MMAs)
        lds           load_chunk, until the K + 1 weight words are in registers
        decode        decode16_i8 of k-half 0
        fence_to_mma  wgmma_fence -> the first wgmma issued
    Per segment the median and the mean (the means add up to the mean total)."""
    seg = {k: [] for k in SPLIT_SEGMENTS}
    ready, backoff, sleep_ns = [], [], []
    d = lambda a, b: (b - a) % (1 << 32)
    for row in att_rows:
        w = words32(row)
        for gj in range(8):
            a = w[8 + 12 * gj: 20 + 12 * gj]
            if a[11] != 1:
                continue
            t_ret, t_end, t_arr, t_ho, t_in, t_out, info, t_dsum, t_ld, t_iss, t_mma, _ = a
            seg["fences"].append(d(t_ret, t_end))
            seg["arrive"].append(d(t_end, t_arr))
            seg["handoff"].append(t_ho)
            seg["step"].append(d(t_arr, t_in) - t_ho)
            wt = d(t_in, t_out)
            seg["wait"].append(wt)
            (backoff if info >> 31 else ready).append(wt)
            if info >> 31:
                sleep_ns.append(info & 0x7fffffff)
            seg["digit_sums"].append(d(t_out, t_dsum))
            seg["lds"].append(d(t_dsum, t_ld))
            seg["decode"].append(d(t_ld, t_iss))
            seg["fence_to_mma"].append(d(t_iss, t_mma))
            seg["total"].append(d(t_ret, t_mma))
    if not seg["total"]:
        return None
    out = {k: {"median": statistics.median(v), "mean": round(statistics.mean(v), 1)} for k, v in seg.items()}
    n = len(seg["total"])
    out["wait_ready"] = {"share": round(len(ready) / n, 3), "median": statistics.median(ready) if ready else None}
    out["wait_backoff"] = {"share": round(len(backoff) / n, 3), "median": statistics.median(backoff) if backoff else None,
                           "sleep_ns_median": statistics.median(sleep_ns) if sleep_ns else None}
    out["steps"] = n
    return out


def isolated(tok, ext, buf, reps, library):
    import torch
    results = []
    for ln in tok.launches:
        mats = ln["mats"]
        units = sum((m["k"] // 128) * (m["n"] // 128) for m in mats)
        for _ in range(3):
            tok.run([ln])
        torch.cuda.synchronize()
        ph = {k: [] for k in ("ramp", "prologue", "digits", "steady", "tail", "total")}
        ctas, all_rows, att_rows = [], [], []
        ext.lib.exl3b_debug_tc_timeline(ctypes.c_void_p(buf.data_ptr()))
        try:
            for _ in range(reps):
                buf.zero_()
                tok.run([ln])
                torch.cuda.synchronize()
                full = buf.cpu().tolist()
                grid = sum(1 for r in full if r[0])          # every CTA stamps slot 0; rows grid .. 2 grid - 1: unit-gap split
                att_rows += full[grid: 2 * grid]
                rows = [r for r in full if r[0] and r[2] and r[3] and r[4] and r[10] and r[8]]
                ctas.append(len(rows))
                all_rows += rows
                for r in rows:
                    ph["ramp"].append((r[3] - r[0]) / 1e3)
                    ph["prologue"].append((r[2] - r[0]) / 1e3)
                    ph["digits"].append((r[4] - r[2]) / 1e3)
                    ph["steady"].append((r[10] - r[3]) / 1e3)
                    ph["tail"].append((r[8] - r[10]) / 1e3)
                    ph["total"].append((r[8] - r[0]) / 1e3)
        finally:
            ext.lib.exl3b_debug_tc_timeline(ctypes.c_void_p(0))
        torch.cuda.synchronize()
        assert ph["ramp"], f"{launch_name(ln)}: no timeline stamps (is {library} the EXL3B_TC_DEBUG build?)"
        n_cta = statistics.median(ctas)
        res = {"launch": launch_name(ln), "k": mats[0]["k"], "n": [m["n"] for m in mats], "K": mats[0]["K"], "units": units,
               "ctas": n_cta, "ramp_us": q(ph["ramp"]), "prologue_us": q(ph["prologue"]), "digits_us": q(ph["digits"]),
               "steady_us": q(ph["steady"]), "tail_us": q(ph["tail"]), "cta_total_us": q(ph["total"]),
               "steady_us_per_unit": round(statistics.median(ph["steady"]) / (units / n_cta), 3),
               "turns": turn_stats(all_rows), "unit_wait_clk": unit_wait(all_rows), "unit_gap_split": unit_gap_split(att_rows)}
        results.append(res)
        print(json.dumps(res), flush=True)
    return results


def replay(tok, ext, num_sms, reps):
    import torch
    launches = tok.launches
    bufs = [torch.zeros((4 * num_sms, SLOTS), dtype=torch.int64, device=tok.dev) for _ in launches]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for _ in range(3):
            tok.run()
    stream.synchronize()
    graph = torch.cuda.CUDAGraph()
    try:
        with torch.cuda.graph(graph, stream=stream):
            for ln, b in zip(launches, bufs):      # the buffer address is a kernel argument, set per launch at capture
                ext.lib.exl3b_debug_tc_timeline(ctypes.c_void_p(b.data_ptr()))
                tok.run([ln])
    finally:
        ext.lib.exl3b_debug_tc_timeline(ctypes.c_void_p(0))
    first = len(launches) - 5                      # the last layer's four launches and the lm_head
    bound = {i: [] for i in range(first, len(launches))}
    for _ in range(reps + 2):
        with torch.cuda.stream(stream):
            for b in bufs:
                b.zero_()
            graph.replay()
        stream.synchronize()
        st = [b.cpu().tolist() for b in bufs]
        if _ < 2:                                  # warm-up replays
            continue
        for i in bound:
            prev_end = max(r[8] for r in st[i - 1] if r[8])
            bound[i] += [(r[4] - prev_end) / 1e3 for r in st[i] if r[4]]
    del graph
    results = []
    for i, v in bound.items():
        assert v, f"{launch_name(launches[i])}: no timeline stamps"
        res = {"launch": launch_name(launches[i]), "after": launch_name(launches[i - 1]), "boundary_us": q(v)}
        results.append(res)
        print(json.dumps(res), flush=True)
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--library", required=True, help="bring-up build of libexl3b200 (EXL3B_TC_DEBUG)")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--replay", action="store_true", help="boundary times inside a replayed CUDA graph of the token's launches")
    ap.add_argument("--out", default=None, help="also write the results (JSON) here")
    args = ap.parse_args()
    os.environ["EXL3B_LIBRARY"] = os.path.abspath(args.library)
    sys.path.insert(0, ROOT)
    import torch
    import bench
    from exllamav3_b200 import ext

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = dict(bench.MODELS["llama-3.1-8b"], layers=2 if args.replay else 1)
    tok = bench.Token(cfg, 1, 0, dev)
    num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
    if args.replay:
        results = replay(tok, ext, num_sms, args.reps)
    else:
        buf = torch.zeros((4 * num_sms, SLOTS), dtype=torch.int64, device=dev)
        results = isolated(tok, ext, buf, args.reps, args.library)
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu, "library": os.path.basename(args.library), "mode": "replay" if args.replay else "isolated"}),
          flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"gpu": gpu, "library": os.path.basename(args.library), "mode": "replay" if args.replay else "isolated",
                       "launches": results}, f, indent=1)


if __name__ == "__main__":
    main()
