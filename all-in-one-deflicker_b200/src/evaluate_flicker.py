"""Flicker of a video's sequences: the temporal warping error of the input, the stage-1 atlas reconstruction, the
neural filter's output and the final output, computed on the GPU (b200.flicker; DESIGN §4e).

    python src/evaluate_flicker.py --video_name NAME [--sequences input,atlas,filter,final] [--gpus N]
                                   [--clips [--clip_overlap V]] [--fidelity [--reference FOLDER]]

Run from the directory that holds data/test/NAME (the pipeline's working directory).  Pair t uses the flow pre-pass's
files data/test/NAME_flow/<t>_<t+1>.npy (F) and <t+1>_<t>.npy (B) of the input's sorted frames; missing pairs are
computed first with the pre-pass.  A sequence's frames are its sorted files, matched to the input's by position, and are
scored at their own resolution.  Writes results/NAME/flicker.json and prints a table.  With --gpus N the pairs are split
into contiguous blocks over N ranks and rank 0 writes the same bytes as a one-GPU run.

With --fidelity the frames the windows decode are also scored against a reference (b200.fidelity; DESIGN §4f): SSIM
and PSNR of each frame of each sequence against the reference frame at the same position, written to
results/NAME/fidelity.json with a second table.  The reference is the input frames (the input itself is then not
scored) or the frames of --reference FOLDER; flicker.json is the same with and without the flag."""
import argparse
import concurrent.futures as cf
import json
import math
import os
import sys
import time
from pathlib import Path

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

SEQUENCES = ("input", "atlas", "filter", "final")
CONFIG = os.path.join(os.path.dirname(os.path.abspath(__file__)), "config", "config_flow_100.json")
WINDOW_PAIRS = 8                    # with four sequences, one b200_warp_error call (B200_WARP_MAX_PAIRS = 32)
DECODERS = min(8, os.cpu_count() or 1)


def sequence_folders(name):
    return {"input": os.path.join("data", "test", name),
            "atlas": os.path.join("results", name, "stage_1", "output"),
            "filter": os.path.join("results", name, "neural_filter", "output"),
            "final": os.path.join("results", name, "final", "output")}


def frame_files(folder):
    """The frames of a sequence folder in order: *.png / *.jpg / *.jpeg, as the pre-pass lists them."""
    return sorted(Path(folder).glob('*.*g'))


def read_frame(path):
    """A frame file as (H, W, 3) uint8 or uint16 (cv2's BGR order: the metric sums over the channels); grey is
    repeated, a 4th channel dropped."""
    import cv2
    img = cv2.imread(str(path), cv2.IMREAD_UNCHANGED)
    if img is None:
        raise FileNotFoundError(f"cannot decode {path}")
    if img.dtype not in (np.uint8, np.uint16):
        raise ValueError(f"{path}: {img.dtype} pixels; frames are 8- or 16-bit")
    if img.ndim == 2:
        img = np.repeat(img[:, :, None], 3, axis=2)
    return np.ascontiguousarray(img[:, :, :3])


def pair_windows(p0, p1, k=WINDOW_PAIRS):
    return [(a, min(a + k, p1)) for a in range(p0, p1, k)]


def load_window(first, last, flow_dir, inputs, seq_frames):
    """Flows of pairs [first, last) and each sequence's frames first .. last (those it has, decoded on DECODERS
    threads), with the seconds spent loading flows and decoding frames.  No flows are read when flow_dir is None."""
    from src.preprocess_optical_flow import flow_files
    t0 = time.perf_counter()
    flows = [tuple(np.load(f).astype(np.float32, copy=False) for f in flow_files(flow_dir, inputs, p))
             for p in range(first, last)] if flow_dir is not None else []
    t1 = time.perf_counter()
    with cf.ThreadPoolExecutor(DECODERS) as pool:          # cv2 decodes without the GIL
        frames = {s: list(pool.map(read_frame, files[first:last + 1])) for s, files in seq_frames.items()}
    return flows, frames, t1 - t0, time.perf_counter() - t1


def score_pairs(p0, p1, flow_dir, inputs, seq_frames, score_window, stats=None, fidelity=None):
    """(squared-error sum, |M|) of pairs [p0, p1) for each sequence (pairs a sequence has both frames of), with each
    window's files read on a thread while the previous window is scored.

    With a FidelityJob, the frames the windows decode are also scored against the reference: frames [p0, p1) and,
    when the job owns the last frame, frame p1 too.  Its results go to fidelity.out; score_window may then be None
    (no flows are read and no pair is scored)."""
    out = {s: [] for s in seq_frames}
    windows = pair_windows(p0, p1)
    decode = seq_frames if fidelity is None else dict(seq_frames, **fidelity.extra)
    if fidelity is not None and fidelity.last and not windows:
        windows = [(p1, p1)]                               # a block of no pairs still owns the last frame
    if not windows:
        return out
    loader = cf.ThreadPoolExecutor(1)
    try:
        load = lambda w: loader.submit(load_window, w[0], w[1], flow_dir if score_window else None, inputs, decode)
        nxt = load(windows[0])
        for j in range(len(windows)):
            flows, frames, t_flow, t_decode = nxt.result()
            nxt = load(windows[j + 1]) if j + 1 < len(windows) else None
            if score_window is not None and windows[j][1] > windows[j][0]:
                for s, v in score_window(flows, {s: frames[s] for s in seq_frames}).items():
                    out[s] += v
            if fidelity is not None:
                fidelity.score(frames, windows[j][1] - windows[j][0] + (j + 1 == len(windows) and fidelity.last))
            if stats is not None:
                stats["flow_load"] += t_flow
                stats["decode"] += t_decode
    finally:
        loader.shutdown(wait=True, cancel_futures=True)
    return out


REFERENCE_KEY = "_reference"          # decoded beside the sequences when the reference is not one of them


class FidelityJob:
    """The fidelity part of a run (DESIGN §4f): which sequences are scored against which reference frames, and the
    (SSIM sum, squared-error sum) of each scored frame in order, filled window by window."""

    def __init__(self, score_frames, reference, ref_files, sequences, seq_frames, last):
        self.score_frames = score_frames
        self.reference = reference                                   # the reference folder as reported
        self.sequences = sequences
        self.ref_key = "input" if reference is None and "input" in seq_frames else REFERENCE_KEY
        self.extra = {} if self.ref_key == "input" else {REFERENCE_KEY: ref_files}
        self.last = last
        self.out = {s: [] for s in sequences}

    def score(self, frames, k):
        """Scores the first k frames of a window's decoded frames (those both a sequence and the reference have)."""
        refs = frames[self.ref_key][:k]
        for s, v in self.score_frames(refs, {s: frames[s][:len(refs)] for s in self.sequences}).items():
            self.out[s] += v


def clip_boundaries(n_frames, overlap=0):
    """The pairs of the seams of the plan stage 1's --clips (--clip_overlap V) fits an n_frames video in: for the
    frames [a, b) two clips share, the pairs t = a - 1 .. b - 1 (the step into the cross-fade, the V - 1 steps inside
    it and the step out).  With V = 0 that is the one pair (c1 - 1, c1) that straddles two clips."""
    from b200.atlas import clip_plan, clip_seams
    with open(CONFIG) as f:
        max_frames = json.load(f)["maximum_number_of_frames"]
    plan = clip_plan(n_frames, max_frames, overlap)
    return plan, [t for a, b in clip_seams(plan) for t in range(a - 1, b)]


def _mean(values):
    v = [x for x in values if not math.isnan(x)]
    return sum(v) / len(v) if v else None


def report(name, pairs, resolutions, folders, scores, clips=None):
    """The flicker.json document: per sequence its resolution, per-pair E(t) and |M| (E is null for an empty mask),
    E_warp (mean over the non-empty pairs; null when there is none) and the empty-pair count.  With clips, the
    boundary pairs and the means over boundary and interior pairs."""
    from b200.flicker import pair_value
    doc = {"video": name, "pairs": pairs, "sequences": {}}
    if clips is not None:
        doc["clips"] = {"plan": [list(c) for c in clips[0]], "boundary_pairs": clips[1]}
    for s, sc in scores.items():
        e = [pair_value(sse, n) for sse, n in sc]
        entry = {"folder": folders[s], "resolution": list(resolutions[s]),
                 "per_pair": [{"t": t, "E": None if math.isnan(v) else v, "mask": int(n)}
                              for t, (v, (_, n)) in enumerate(zip(e, sc))],
                 "E_warp": _mean(e), "empty_pairs": sum(1 for v in e if math.isnan(v))}
        if clips is not None:
            b = set(clips[1])
            entry["E_boundary"] = _mean([v for t, v in enumerate(e) if t in b])
            entry["E_interior"] = _mean([v for t, v in enumerate(e) if t not in b])
        doc["sequences"][s] = entry
    return doc


def table(doc):
    clips = "clips" in doc
    head = "%-8s %11s %6s %6s %12s" % ("sequence", "resolution", "pairs", "empty", "E_warp")
    lines = [head + (" %12s %12s" % ("E_boundary", "E_interior") if clips else "")]
    fmt = lambda v: "%12s" % "-" if v is None else "%12.6g" % v
    for s, e in doc["sequences"].items():
        line = "%-8s %11s %6d %6d %s" % (s, "%dx%d" % tuple(e["resolution"]), len(e["per_pair"]), e["empty_pairs"],
                                         fmt(e["E_warp"]))
        if clips:
            line += " %s %s" % (fmt(e["E_boundary"]), fmt(e["E_interior"]))
        lines.append(line)
    return "\n".join(lines)


def evaluate(name, sequences, score_window, rank=0, world=1, pg=None, clips=False, stats=None, clip_overlap=0):
    """Scores rank's block of pairs; under a process group the blocks are gathered in pair order.  Returns the
    flicker.json document on rank 0 (None on the other ranks)."""
    return _evaluate(name, sequences, score_window, rank, world, pg, clips, stats, clip_overlap)[0]


def evaluate_fidelity(name, sequences, score_window, score_frames, reference=None, rank=0, world=1, pg=None,
                      clips=False, stats=None, clip_overlap=0):
    """evaluate() plus the fidelity of the sequences to the reference (the input frames, or the frames of the folder
    `reference`), scored on the frames the warping error's windows decode.  Rank r scores frames [p0, p1) of its pair
    block, the last rank also frame T - 1; the frames are gathered in order.  Returns (flicker.json document,
    fidelity.json document) on rank 0, (None, None) elsewhere; with score_window None only the fidelity is scored
    (and the first document is None)."""
    return _evaluate(name, sequences, score_window, rank, world, pg, clips, stats, clip_overlap,
                     (score_frames, reference))


def _evaluate(name, sequences, score_window, rank, world, pg, clips, stats, clip_overlap, fidelity=None):
    folders = sequence_folders(name)
    inputs = frame_files(folders["input"])
    if len(inputs) < 2:
        raise FileNotFoundError(f"{folders['input']} holds {len(inputs)} frames; the warping error needs two")
    flow_dir = Path(folders["input"] + "_flow")
    seq_frames = {}
    for s in sequences:
        files = frame_files(folders[s])
        if s == "input" or len(files) >= 2:
            seq_frames[s] = files[:len(inputs)]
        elif rank == 0:
            print("evaluate_flicker: no %s frames in %s, skipped" % (s, folders[s]), flush=True)
    p0, p1 = 0, len(inputs) - 1
    if world > 1:
        from b200.launch import pair_block
        p0, p1 = pair_block(rank, world, len(inputs))
    job = None
    if fidelity is not None:
        score_frames, reference = fidelity
        ref_files = frame_files(reference if reference is not None else folders["input"])[:len(inputs)]
        if not ref_files:
            raise FileNotFoundError(f"{reference} holds no frames")
        # the input is its own default reference: it is scored only against a separate one
        scored = [s for s in seq_frames if s != "input" or reference is not None]
        job = FidelityJob(score_frames, reference, ref_files, scored, seq_frames, rank == world - 1)
    mine = score_pairs(p0, p1, flow_dir, inputs, seq_frames, score_window, stats, job)
    fmine = job.out if job is not None else None
    if world > 1:
        import torch.distributed as dist
        every = [None] * world
        dist.all_gather_object(every, mine if job is None else (mine, fmine), group=pg)
        if job is not None:
            fmine = {s: [v for r in range(world) for v in every[r][1][s]] for s in job.sequences}
            every = [e[0] for e in every]
        merged = {s: [v for r in range(world) for v in every[r][s]] for s in seq_frames}
    else:
        merged = mine
    if rank != 0:
        return None, None
    resolutions = {s: read_frame(files[0]).shape[:2] for s, files in seq_frames.items()}
    plan = clip_boundaries(len(inputs), clip_overlap) if clips else None
    doc = report(name, len(inputs) - 1, resolutions, folders, merged, plan) if score_window is not None else None
    if job is None:
        return doc, None
    fplan = clip_seam_frames(len(inputs), clip_overlap) if clips else None
    ref_res = read_frame(ref_files[0]).shape[:2]
    fdoc = report_fidelity(name, len(ref_files), job.reference or folders["input"], ref_res,
                           {s: resolutions[s] for s in job.sequences}, folders, fmine, fplan)
    return doc, fdoc


def clip_seam_frames(n_frames, overlap=0):
    """The seam frames of the plan stage 1's --clips (--clip_overlap V) fits an n_frames video in: the V frames each
    pair of consecutive clips shares (the cross-fade), or with V = 0 the first frame of each later clip."""
    from b200.atlas import clip_plan, clip_seams
    with open(CONFIG) as f:
        max_frames = json.load(f)["maximum_number_of_frames"]
    plan = clip_plan(n_frames, max_frames, overlap)
    if overlap == 0:
        return plan, [c[0] for c in plan[1:]]
    return plan, [t for a, b in clip_seams(plan) for t in range(a, b)]


def report_fidelity(name, n_frames, reference, ref_resolution, resolutions, folders, scores, clips=None):
    """The fidelity.json document: the video, the reference folder and its frame count; per sequence its folder,
    resolution and the reference's, per-frame S(t) and PSNR(t) (null for a frame equal to the reference), SSIM (mean
    of S(t)), PSNR (mean of the finite PSNR(t); null when there is none) and the identical-frame count.  With clips,
    the seam frames and the means over seam and interior frames."""
    from b200.fidelity import frame_values
    doc = {"video": name, "reference": reference, "frames": n_frames, "sequences": {}}
    if clips is not None:
        doc["clips"] = {"plan": [list(c) for c in clips[0]], "seam_frames": clips[1]}
    for s, sc in scores.items():
        H, W = resolutions[s]
        vals = [frame_values(a, b, H, W) for a, b in sc]
        ssim = [v[0] for v in vals]
        psnr = [float("nan") if v[1] is None else v[1] for v in vals]
        entry = {"folder": folders[s], "resolution": [H, W], "reference_resolution": list(ref_resolution),
                 "per_frame": [{"t": t, "ssim": a, "psnr": b} for t, (a, b) in enumerate(vals)],
                 "SSIM": _mean(ssim), "PSNR": _mean(psnr), "identical_frames": sum(1 for v in vals if v[1] is None)}
        if clips is not None:
            seam = set(clips[1])
            for part, keep in (("seam", lambda t: t in seam), ("interior", lambda t: t not in seam)):
                entry["SSIM_" + part] = _mean([v for t, v in enumerate(ssim) if keep(t)])
                entry["PSNR_" + part] = _mean([v for t, v in enumerate(psnr) if keep(t)])
        doc["sequences"][s] = entry
    return doc


def fidelity_table(doc):
    clips = "clips" in doc
    head = "%-8s %11s %6s %9s %10s %10s" % ("sequence", "resolution", "frames", "identical", "SSIM", "PSNR")
    lines = [head + (" %10s %10s %10s %10s" % ("SSIM_seam", "SSIM_int", "PSNR_seam", "PSNR_int") if clips else "")]
    fmt = lambda v: "%10s" % "-" if v is None else "%10.6g" % v
    for s, e in doc["sequences"].items():
        line = "%-8s %11s %6d %9d %s %s" % (s, "%dx%d" % tuple(e["resolution"]), len(e["per_frame"]),
                                            e["identical_frames"], fmt(e["SSIM"]), fmt(e["PSNR"]))
        if clips:
            line += " " + " ".join(fmt(e[k]) for k in ("SSIM_seam", "SSIM_interior", "PSNR_seam", "PSNR_interior"))
        lines.append(line)
    return "\n".join(lines)


def write(doc, name, file="flicker.json"):
    path = os.path.join("results", name, file)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write(json.dumps(doc, indent=1) + "\n")
    return path


def ensure_flows(name, rank=0, world=1):
    """Computes the flow pairs of the input that are missing, with the pre-pass (sharded over the ranks)."""
    from src import preprocess_optical_flow as P
    vid = Path(sequence_folders(name)["input"])
    frames = frame_files(vid)
    missing = P.pending_pairs(vid.parent / (vid.name + "_flow"), frames, 0, max(len(frames) - 1, 0))
    if world > 1:
        import torch.distributed as dist
        flag = [bool(missing)]
        dist.broadcast_object_list(flag, src=0)
        if flag[0]:
            P.preprocess_sharded(vid, rank, world)
    elif missing:
        P.preprocess(argparse.Namespace(vid_path=vid, max_long_edge=2000))


def main(argv=None):
    cli = argparse.ArgumentParser(description="temporal warping error of a video's sequences")
    cli.add_argument("--video_name", required=True)
    cli.add_argument("--sequences", default=",".join(SEQUENCES),
                     help="comma-separated subset of " + ",".join(SEQUENCES) + "; those whose folder has frames are scored")
    cli.add_argument("--gpu", type=int, default=0)
    cli.add_argument("--gpus", type=int, default=1, help="split the frame pairs over this many GPUs of the node")
    cli.add_argument("--clips", action="store_true",
                     help="list the pairs that straddle two of stage 1's --clips atlases apart")
    cli.add_argument("--clip_overlap", type=int, default=0,
                     help="with --clips: the frames consecutive clips share (stage 1's --clip_overlap); the pairs "
                          "into, inside and out of each cross-fade are listed")
    cli.add_argument("--fidelity", action="store_true",
                     help="also score SSIM and PSNR of each sequence against the reference (results/<name>/fidelity.json)")
    cli.add_argument("--reference", default=None,
                     help="with --fidelity: the folder of reference frames (default: the input frames, which are then "
                          "not scored)")
    opts = cli.parse_args(argv)
    if opts.clip_overlap != 0 and not opts.clips:
        cli.error("--clip_overlap is only meaningful with --clips")
    if opts.reference is not None and not opts.fidelity:
        cli.error("--reference is only meaningful with --fidelity")
    sequences = [s for s in opts.sequences.split(",") if s]
    bad = [s for s in sequences if s not in SEQUENCES]
    if bad or not sequences:
        cli.error("unknown sequence(s) %s; choose from %s" % (",".join(bad), ",".join(SEQUENCES)))
    from b200 import launch
    env = launch.torchrun_env()
    if env is None and opts.gpus > 1:
        return launch.relaunch(__file__, sys.argv[1:] if argv is None else argv, opts.gpus)
    if env is None:
        os.environ["CUDA_VISIBLE_DEVICES"] = str(opts.gpu)
        rank, world, device = 0, 1, "cuda:0"
    else:
        rank, world = env[0], env[1]
        device, _ = launch.init(env[2])
    from b200.flicker import FlickerScorer
    ensure_flows(opts.video_name, rank, world)
    scorer = FlickerScorer(device)
    fdoc = None
    if opts.fidelity:
        from b200.fidelity import FidelityScorer
        doc, fdoc = evaluate_fidelity(opts.video_name, sequences, scorer.score_window,
                                      FidelityScorer(device).score_frames, opts.reference, rank, world,
                                      clips=opts.clips, clip_overlap=opts.clip_overlap)
    else:
        doc = evaluate(opts.video_name, sequences, scorer.score_window, rank, world, clips=opts.clips,
                       clip_overlap=opts.clip_overlap)
    if rank == 0:
        print("wrote", write(doc, opts.video_name))
        print(table(doc), flush=True)
        if fdoc is not None:
            print("wrote", write(fdoc, opts.video_name, "fidelity.json"))
            print(fidelity_table(fdoc), flush=True)
    if env is not None:
        launch.finish()
    return 0


if __name__ == "__main__":
    sys.exit(main())
