"""Camera pictures of many receivers in one batch, against the ways to decode them exactly without the receivers call.

    python -m libcimbar_b200.receivers_bench [--rounds R]

Workload: D receivers x k pictures (D in 16, 64, 256; k in 1, 4), picture i drawn round-robin from the camera_pipeline_bench pool
(the reference's samples/6bit/*.jpg with its 3584 x 2688 upscale) plus the two mode-B photographs (tests/golden/b__ex*.jpg), all in
device memory, and picture i belonging to receiver i % D.  Mode B (the mode whose CC_FIT fits matrices), SHARPEN_IF_NEEDED | CC_FIT
(the CLI's defaults); every receiver starts from a distinct active matrix.  Four runs, timed in turn with CUDA events, R rounds each:
  (a) `receivers`: one cb200_scan_extract_decode_chunks_receivers_dev call;
  (b) `per_receiver`: today's exact caller on one context: per receiver cb200_set_ccm, the pictures call on its k pictures,
      cb200_get_ccm (which waits for the call);
  (c) `contexts`: D contexts on D CUDA streams, each set to its receiver's state, one pictures call each;
  (d) `one_chain`: the same pictures as one plain pictures call -- one decoder for everybody: the cost of a single chain, not a
      correct result.
Prints one JSON line: per shape, pictures/s, GPU ms (events around the run) and host us (the host's time to issue it) of each run,
the device memory the D contexts of (c) hold, and whether (a), (b) and (c) gave identical records and states; the card's name and
power limit.  A context holds buffers sized for the largest batch and picture it has seen, and the exact walk's workspace, whatever
its max_frames, so (c) is run only where its D contexts fit in 80 % of the free device memory; the memory one context holds after
its call is reported for every shape.  Under mode B the 4C pictures of the pool run the whole path (scan, extract, deskew, decode)
but yield no chunks; the mode-B photographs decode."""
import argparse
import json
import time

import numpy as np

from libcimbar_b200.bench_support import card, entry_states, load_pictures, photographs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--receivers", type=int, nargs="*", default=[16, 64, 256])
    ap.add_argument("--per", type=int, nargs="*", default=[1, 4])
    args = ap.parse_args()
    import torch
    import libcimbar_b200 as cb
    torch.cuda.set_device(0)
    pool = [torch.from_numpy(p).cuda() for p in load_pictures() + photographs()]
    flags = cb.FLAG_SHARPEN_IF_NEEDED | cb.FLAG_CC_FIT
    stream = torch.cuda.Stream()

    def ev():
        return torch.cuda.Event(enable_timing=True)

    def timed(fn, s=None):
        s = s or stream
        t0, t1 = ev(), ev()
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        t0.record(s)
        fn()
        t1.record(s)
        host = time.perf_counter() - h0
        t1.synchronize()
        return t0.elapsed_time(t1), host * 1e6

    results = []
    for D in args.receivers:
        for k in args.per:
            n = D * k
            pics = [pool[i % len(pool)] for i in range(n)]
            of = np.arange(n, dtype=np.int32) % D
            mine = [np.flatnonzero(of == r) for r in range(D)]
            ents = entry_states(D)
            master = cb.receiver_states(ents)
            ctx = cb.Context(68, max_frames=n)
            ctx.set_stream(stream.cuda_stream)
            db = ctx.info.data_bytes
            chunks = torch.zeros((n, db), dtype=torch.uint8, device="cuda")
            mask = torch.zeros(n, dtype=torch.int32, device="cuda")
            status = torch.zeros(n, dtype=torch.int32, device="cuda")
            states = master.clone()

            def run_a():
                states.copy_(master)
                ctx.scan_extract_decode_chunks_receivers_dev(pics, of, states, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), flags=flags)

            def host_records():
                torch.cuda.synchronize()
                return chunks.cpu().numpy().copy(), mask.cpu().numpy().copy(), status.cpu().numpy().copy()

            per = cb.Context(68, max_frames=k)
            per.set_stream(stream.cuda_stream)
            exits_b = [None] * D

            bchunks = [torch.zeros((k, db), dtype=torch.uint8, device="cuda") for _ in range(D)]
            bmask = [torch.zeros(k, dtype=torch.int32, device="cuda") for _ in range(D)]
            bstatus = [torch.zeros(k, dtype=torch.int32, device="cuda") for _ in range(D)]

            def run_b_all():
                for r in range(D):
                    per.set_ccm(ents[r])
                    per.scan_extract_decode_chunks_pictures_dev([pics[i] for i in mine[r]], bchunks[r].data_ptr(), bmask[r].data_ptr(),
                                                                bstatus[r].data_ptr(), flags=flags)
                    exits_b[r] = per.get_ccm()

            def gathered(cs, ms, ss):
                c = np.zeros((n, db), np.uint8)
                m = np.zeros(n, np.int32)
                s = np.zeros(n, np.int32)
                for r in range(D):
                    c[mine[r]], m[mine[r]], s[mine[r]] = cs[r].cpu().numpy(), ms[r].cpu().numpy(), ss[r].cpu().numpy()
                return c, m, s

            def run_d():
                ctx.set_ccm(None)
                ctx.scan_extract_decode_chunks_pictures_dev(pics, chunks.data_ptr(), mask.data_ptr(), status.data_ptr(), flags=flags)

            entry = {"receivers": D, "per_receiver": k, "pictures": n}
            # (a) and its records
            run_a()
            a_rec = host_records()
            a_states = cb.read_receiver_states(states)
            ta = [timed(run_a) for _ in range(args.rounds)]
            # (b)
            run_b_all()
            b_rec = gathered(bchunks, bmask, bstatus)
            tb = [timed(run_b_all) for _ in range(args.rounds)]
            # (d)
            run_d()
            torch.cuda.synchronize()
            td = [timed(run_d) for _ in range(args.rounds)]
            per.close()
            # (c)
            free0, _ = torch.cuda.mem_get_info()
            probe = cb.Context(68, max_frames=k)
            s0 = torch.cuda.Stream()
            probe.set_stream(s0.cuda_stream)
            probe.scan_extract_decode_chunks_pictures_dev([pics[i] for i in mine[0]], bchunks[0].data_ptr(), bmask[0].data_ptr(),
                                                          bstatus[0].data_ptr(), flags=flags)
            probe.sync()
            one = free0 - torch.cuda.mem_get_info()[0]
            probe.close()
            c_ok = None
            entry["context_device_mb"] = round(one / 2**20, 1)
            if one * D < free0 * 0.8:
                torch.cuda.synchronize()
                f0 = torch.cuda.mem_get_info()[0]
                ctxs = [cb.Context(68, max_frames=k) for _ in range(D)]
                streams = [torch.cuda.Stream() for _ in range(D)]
                for c, s in zip(ctxs, streams):
                    c.set_stream(s.cuda_stream)

                def run_c():
                    start = torch.cuda.Event()
                    start.record(stream)
                    for r in range(D):
                        streams[r].wait_event(start)
                        ctxs[r].set_ccm(ents[r])
                        ctxs[r].scan_extract_decode_chunks_pictures_dev([pics[i] for i in mine[r]], bchunks[r].data_ptr(), bmask[r].data_ptr(),
                                                                        bstatus[r].data_ptr(), flags=flags)
                    for s in streams:
                        done = torch.cuda.Event()
                        done.record(s)
                        stream.wait_event(done)

                run_c()
                torch.cuda.synchronize()
                c_rec = gathered(bchunks, bmask, bstatus)
                c_states = [c.get_ccm() for c in ctxs]
                entry["contexts_device_mb"] = round((f0 - torch.cuda.mem_get_info()[0]) / 2**20, 1)
                tc = [timed(run_c) for _ in range(args.rounds)]
                entry["contexts"] = {"pictures_per_s": round(n / (min(t[0] for t in tc) / 1e3), 1), "gpu_ms": [round(t[0], 2) for t in tc],
                                     "host_us": [round(t[1]) for t in tc]}
                same_c = all(np.array_equal(x, y) for x, y in zip(a_rec, c_rec))
                c_ok = same_c and all(_same(a_states[r], c_states[r]) for r in range(D))
                for c in ctxs:
                    c.close()
                del ctxs, streams
            else:
                entry["contexts"] = "not run: %d contexts of %.0f MB each do not fit in 80 %% of the free memory" % (D, one / 2**20)
            for name, t in (("receivers", ta), ("per_receiver", tb), ("one_chain", td)):
                entry[name] = {"pictures_per_s": round(n / (min(x[0] for x in t) / 1e3), 1), "gpu_ms": [round(x[0], 2) for x in t],
                               "host_us": [round(x[1]) for x in t]}
            entry["a_equals_b"] = all(np.array_equal(x, y) for x, y in zip(a_rec, b_rec)) and \
                all(_same(a_states[r], exits_b[r]) for r in range(D))
            entry["a_equals_c"] = c_ok
            entry["decoded_pictures"] = int((a_rec[1] != 0).sum())
            results.append(entry)
            ctx.close()
            del chunks, mask, status, bchunks, bmask, bstatus
            torch.cuda.empty_cache()
    name, power = card()
    print(json.dumps({"bench": "receivers", "mode": 68, "flags": "SHARPEN_IF_NEEDED|CC_FIT", "rounds": args.rounds, "results": results,
                      "card": name, "power_limit": power}))


def _same(a, b):
    return (a is None) == (b is None) and (a is None or np.array_equal(a, b))


if __name__ == "__main__":
    main()
