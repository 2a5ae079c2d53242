"""Eval graphs (bts_b200.set_eval_graphs / BTS_B200_EVAL_GRAPH=1): BtsModel.forward serves eval forwards under no_grad
from a per-model cache of captured CUDA graphs.  Outputs are fresh tensors bit-identical to the eager forward's, also
while running statistics, weights, the state_dict, the precision mode or the parameters' storage change between calls;
a signature is captured on its second call, at most EVAL_GRAPH_KEYS are kept, and training, grad-enabled forwards,
captures in progress and DataParallel replicas run eager.  The unmodified bts_test.py writes the same PNG bytes with the
switch on and off, and the unmodified bts_main.py --do_online_eval reports the same metrics."""
import gc
import json
import os
import shutil
import subprocess
import sys
import types
import weakref

import numpy as np
import pytest
import torch

from test_dropin_gpu import ROOT, SCRIPTS, _make_dataset, _script_dir

pytestmark = pytest.mark.gpu


@pytest.fixture
def eval_graphs():
    """the switch on for one test; off again (freeing every graph) and the precision mode restored afterwards"""
    import bts_b200
    prev, mode = bts_b200.set_eval_graphs(True), bts_b200.get_precision()
    yield
    bts_b200.set_eval_graphs(prev)
    bts_b200.set_precision(mode)


def _model(enc, dataset="nyu"):
    import bts
    torch.manual_seed(0)
    p = types.SimpleNamespace(encoder=enc, max_depth=80.0 if dataset == "kitti" else 10.0, dataset=dataset, bts_size=512,
                              pretrained=False)
    m = bts.BtsModel(p)
    m.decoder.apply(bts.weights_init_xavier)
    return m.cuda().eval()


def _inputs(n, H, W, seed=1):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(1, 3, H, W, generator=g).cuda(), torch.tensor([700.0 + 10 * i], dtype=torch.float64).cuda())
            for i in range(n)]


def _eager(m, x, f):
    """the eager body of BtsModel.forward's inference branch, whatever the switch says"""
    from bts_b200 import conv
    with torch.no_grad(), conv.inference():
        return [t.clone() for t in m.decoder(m.encoder(x.contiguous(memory_format=torch.channels_last)), f)]


def _call(m, x, f):
    with torch.no_grad():
        return m(x, f)


def _same(a, b):
    return all(u.dtype == v.dtype and u.shape == v.shape and u.stride() == v.stride() and torch.equal(u, v)
               for u, v in zip(a, b)) and len(a) == len(b)


def _stats():
    from bts_b200 import graph
    return graph.eval_graph_stats()


def _delta(s0):
    s1 = _stats()
    return {k: s1[k] - s0[k] for k in s1}


@pytest.mark.parametrize("enc,dataset", [("densenet121_bts", "nyu"), ("resnext50_bts", "kitti"), ("mobilenetv2_bts", "kitti")])
def test_graphed_forwards_equal_eager_bit_for_bit(enc, dataset):
    """the same calls with the switch off and on; kitti scales the depth by focal, which changes from call to call"""
    import bts_b200
    from bts_b200 import _lib
    m = _model(enc, dataset)
    calls = _inputs(3, 96, 128)
    calls = calls + calls[:2]
    assert not bts_b200.get_eval_graphs()
    want = [[t.clone() for t in _call(m, x, f)] for x, f in calls]
    l0 = _lib.launches
    _call(m, *calls[0])
    per_forward = _lib.launches - l0
    prev = bts_b200.set_eval_graphs(True)
    try:
        s0 = _stats()
        got = [_call(m, x, f) for x, f in calls]
        assert _delta(s0) == {"captures": 1, "replays": 4, "evictions": 0, "recaptures": 0}
        l0 = _lib.launches
        _call(m, *calls[2])
        assert _lib.launches - l0 == per_forward            # a replay counts the native launches it runs
    finally:
        bts_b200.set_eval_graphs(prev)
    for g, w in zip(got, want):
        assert type(g) is tuple and _same(g, w)
        assert not any(t.requires_grad for t in g)


def test_outputs_are_fresh_tensors(eval_graphs):
    m = _model("densenet121_bts")
    (x0, f0), (x1, f1) = _inputs(2, 96, 128)
    for _ in range(2):
        _call(m, x0, f0)                        # seen, captured
    a = _call(m, x0, f0)
    a_copy = [t.clone() for t in a]
    b = _call(m, x1, f1)                        # the next replay does not write into what the caller holds
    assert _same(a, a_copy) and _same(b, _eager(m, x1, f1))
    for t in b:
        t.fill_(123.0)                          # and writing into an output changes nothing in the next call
    assert _same(_call(m, x1, f1), _eager(m, x1, f1))
    assert _same(_call(m, x0, f0), a_copy)


SHAPES = {"A": (64, 96), "B": (64, 128), "C": (96, 96), "D": (96, 128), "E": (64, 160), "F": (128, 96)}


def test_capture_policy_and_lru_eviction(eval_graphs):
    from bts_b200 import graph
    m = _model("mobilenetv2_bts")
    inp = {k: _inputs(1, H, W, seed=i)[0] for i, (k, (H, W)) in enumerate(SHAPES.items())}

    def run(seq):
        for k in seq:
            x, f = inp[k]
            assert _same(_call(m, x, f), _eager(m, x, f)), k

    def key(k):
        return next(kk for kk in m._eval_graph_cache.entries if kk[0][2:] == SHAPES[k])

    s0 = _stats()
    run("A")
    assert _delta(s0)["captures"] == 0                                       # once: eager, nothing captured
    run("AA")
    assert _delta(s0) == {"captures": 1, "replays": 2, "evictions": 0, "recaptures": 0}
    run("B")                                                                 # B is seen once and never captured
    run("CACADADA")
    entries = m._eval_graph_cache.entries
    assert len(entries) == graph.EVAL_GRAPH_KEYS == 4
    assert entries[key("B")] is None and all(entries[key(k)] is not None for k in "ACD")
    assert _delta(s0) == {"captures": 3, "replays": 8, "evictions": 0, "recaptures": 0}
    run("E")                                                                 # drops B, the least recently used key
    assert [kk[0][2:] for kk in entries] == [SHAPES[k] for k in "CDAE"]
    assert _delta(s0)["evictions"] == 0                                      # B held no graph
    c_graph = weakref.ref(entries[key("C")])
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    reserved = torch.cuda.memory_reserved()
    run("F")                                                                 # evicts C's graph
    assert [kk[0][2:] for kk in entries] == [SHAPES[k] for k in "DAEF"]
    assert _delta(s0) == {"captures": 3, "replays": 8, "evictions": 1, "recaptures": 0}
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert c_graph() is None and torch.cuda.memory_reserved() < reserved   # the graph and its pool are freed
    run("AAD")
    assert _delta(s0)["captures"] == 3                                      # the survivors still replay


def test_graphs_follow_the_model(eval_graphs):
    import bts
    import bts_b200
    m = _model("densenet121_bts")
    (x, f), (x2, _) = _inputs(2, 96, 128, seed=5)
    for _ in range(2):
        _call(m, x, f)
    s0 = _stats()

    def check(prev):
        got = _call(m, x, f)
        assert _same(got, _eager(m, x, f))
        assert prev is None or not _same(got, prev)
        return got

    g0 = check(None)
    # a train-mode forward moves the BatchNorm running statistics
    m.train()
    with torch.no_grad():
        m(x2 * 2 + 1, f)
    m.eval()
    g1 = check(g0)
    # an AdamW step
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3)
    m.train()
    gt = torch.rand(2, 1, 96, 128, generator=torch.Generator().manual_seed(6)).cuda() * 10
    out = m(torch.cat([x, x2]), f.repeat(2))
    bts.silog_loss(0.85)(out[4], gt, gt > 0.1).backward()
    opt.step()
    m.eval()
    g2 = check(g1)
    # load_state_dict
    m.load_state_dict(_model("densenet121_bts").state_dict())
    g3 = check(g2)
    assert _delta(s0) == {"captures": 0, "replays": 4, "evictions": 0, "recaptures": 0}
    # the precision mode is part of the key: tf32 forwards get their own graph, fp32 ones replay theirs again
    bts_b200.set_precision("tf32")
    for _ in range(3):
        t = check(g3)
    bts_b200.set_precision("fp32")
    g4 = check(t)
    assert _same(g4, g3)
    assert _delta(s0) == {"captures": 1, "replays": 7, "evictions": 0, "recaptures": 0}
    # replaced storage: the graph is captured again instead of raising
    w = m.decoder.conv5[0].weight
    w.data = w.data.clone()
    with torch.no_grad():
        w.mul_(1.5)
    check(g4)
    assert _delta(s0) == {"captures": 2, "replays": 8, "evictions": 0, "recaptures": 1}


def test_cache_not_taken(eval_graphs):
    import bts
    from bts_b200.graph import GraphedInference, GraphedTrainStep
    m = _model("mobilenetv2_bts")
    (x, f), = _inputs(1, 64, 96)
    s0 = _stats()
    # train mode, under no_grad
    m.train()
    for _ in range(3):
        _call(m, x, f)
    # eval mode with grad enabled and trainable parameters
    m.eval()
    for _ in range(3):
        out = m(x, f)
        assert out[4].requires_grad
    del out                                     # its autograd graph would stall the GraphedTrainStep capture below
    # the warm-up and capture of a GraphedInference, and its replays
    gi = GraphedInference(m, x, f)
    for _ in range(2):
        assert _same([t.clone() for t in gi(x, f)], _eager(m, x, f))
    # a GraphedTrainStep
    m.train()
    gt = torch.rand(2, 1, 64, 96, generator=torch.Generator().manual_seed(4)).cuda() * 10
    step = GraphedTrainStep(m, lambda o, g: bts.silog_loss(0.85)(o[4], g, g > 0.1),
                            ((x.repeat(2, 1, 1, 1), f.repeat(2)), (gt,)))
    step((x.repeat(2, 1, 1, 1), f.repeat(2)), (gt,))
    m.eval()
    # DataParallel replicas
    replica = torch.nn.parallel.replicate(m, [0], detach=True)[0]
    for _ in range(3):
        assert _same(_call(replica, x, f), _eager(m, x, f))
    assert _delta(s0) == {"captures": 0, "replays": 0, "evictions": 0, "recaptures": 0}
    assert "_eval_graph_cache" not in m.__dict__
    # a forward inside the caller's own capture runs the eager body even for a signature the cache has captured
    for _ in range(3):
        _call(m, x, f)
    s1 = _stats()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = _call(m, x, f)
    assert _delta(s1) == {"captures": 0, "replays": 0, "evictions": 0, "recaptures": 0}
    g.replay()
    assert _same(out, _eager(m, x, f))


# ---------------------------------------------------------------------------------------- the unmodified drivers
def _boot(script, args_file, cwd, graphs):
    """runs an unmodified reference script through tests/dropin/boot.py with seeded RNGs and BTS_B200_EVAL_GRAPH set;
    prints the eval-graph counters on exit"""
    code = ("import atexit, json, random, runpy, sys\n"
            "import numpy as np, torch\n"
            "random.seed(0); np.random.seed(0); torch.manual_seed(0)\n"
            "from bts_b200 import graph\n"
            "atexit.register(lambda: print('EVAL_GRAPH_STATS ' + json.dumps(graph.eval_graph_stats()), flush=True))\n"
            "sys.argv = [%r, %r, %r]\n"
            "runpy.run_path(sys.argv[0], run_name='__main__')\n") % (os.path.join(ROOT, "tests", "dropin", "boot.py"),
                                                                     script, args_file)
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="0",
               BTS_B200_PRETRAINED="0", BTS_B200_EVAL_GRAPH="1" if graphs else "0")
    r = subprocess.run([sys.executable, "-c", code], cwd=cwd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.stdout[-3000:], r.stderr[-3000:])
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("EVAL_GRAPH_STATS ")][-1]
    return r.stdout, json.loads(line.split(" ", 1)[1])


def _workdir(tmp_path, name):
    work = tmp_path / name
    work.mkdir()
    for s in SCRIPTS:
        shutil.copy(os.path.join(_script_dir(), s), work / s)
    shutil.copy(os.path.join(ROOT, "bts.py"), work / "bts.py")
    return work


@pytest.mark.skipif(_script_dir() is None, reason="reference scripts not available (`make -C oracle` copies them into oracle/_ref)")
def test_unmodified_bts_test_writes_identical_pngs(tmp_path):
    import cv2
    data = tmp_path / "data"
    data.mkdir()
    n = 6
    _make_dataset(str(data), n=n)
    # a checkpoint as bts_main.py writes it (DataParallel keys), with the BatchNorm statistics of two of the images
    m = _model("densenet121_bts").train()
    bns = [b for b in m.modules() if isinstance(b, torch.nn.BatchNorm2d)]
    for b in bns:
        b.momentum = 1.0
    mean, std = np.array([0.485, 0.456, 0.406], np.float32), np.array([0.229, 0.224, 0.225], np.float32)
    imgs = [(cv2.imread(str(data / "scene" / ("rgb_%d.png" % i)))[:, :, ::-1] / np.float32(255) - mean) / std
            for i in (0, 1)]                    # bts_dataloader's test-time input: RGB in [0, 1], ImageNet-normalised
    x = torch.from_numpy(np.stack(imgs)).permute(0, 3, 1, 2).contiguous().cuda()
    with torch.no_grad():
        m(x, torch.full((2,), 518.8579, device="cuda"))
    ckpt_dir = tmp_path / "ckpt"
    ckpt_dir.mkdir()
    shutil.copy(os.path.join(ROOT, "bts.py"), ckpt_dir / "bts_eg.py")
    torch.save({"global_step": 0, "model": {"module." + k: v.cpu() for k, v in m.state_dict().items()}},
               ckpt_dir / "model-0")
    args = """--model_name bts_eg
--encoder densenet121_bts
--data_path {d}/
--dataset nyu
--filenames_file {d}/files.txt
--checkpoint_path {c}
--input_height 480
--input_width 640
--max_depth 10
""".format(d=data, c=ckpt_dir / "model-0")
    pngs = {}
    for graphs in (False, True):
        work = _workdir(tmp_path, "work%d" % graphs)
        (work / "args_test.txt").write_text(args)
        out, stats = _boot("bts_test.py", "args_test.txt", work, graphs)
        assert "now testing %d files" % n in out and "Done." in out
        assert stats == ({"captures": 1, "replays": n - 1, "evictions": 0, "recaptures": 0} if graphs else
                         {"captures": 0, "replays": 0, "evictions": 0, "recaptures": 0})
        raw = sorted((work / "result_bts_eg" / "raw").glob("*.png"))
        assert len(raw) == n
        pngs[graphs] = [p.read_bytes() for p in raw]
        depth = cv2.imread(str(raw[-1]), -1)
        assert depth.dtype == np.uint16 and len(np.unique(depth)) > 10      # a depth map, not a constant
    assert pngs[True] == pngs[False]


@pytest.mark.skipif(_script_dir() is None, reason="reference scripts not available (`make -C oracle` copies them into oracle/_ref)")
def test_unmodified_bts_main_online_eval(tmp_path):
    """two training steps of batch 2 with --do_online_eval --eval_freq 1: one eval pass over the four images after the
    second step, with the DataParallel-wrapped model and the eval loader's pin-memory thread running during the capture"""
    data = tmp_path / "data"
    data.mkdir()
    _make_dataset(str(data))
    metrics = {}
    for graphs in (False, True):
        work = _workdir(tmp_path, "work%d" % graphs)
        log = tmp_path / ("log%d" % graphs)
        log.mkdir()
        (work / "args_train.txt").write_text("""--mode train
--model_name bts_eg
--encoder densenet121_bts
--dataset nyu
--data_path {d}/
--gt_path {d}/
--filenames_file {d}/files.txt
--batch_size 2
--num_epochs 1
--learning_rate 1e-4
--weight_decay 1e-2
--adam_eps 1e-3
--num_threads 1
--input_height 128
--input_width 160
--max_depth 10
--log_directory {l}
--log_freq 1000
--do_online_eval
--eval_freq 1
--data_path_eval {d}/
--gt_path_eval {d}/
--filenames_file_eval {d}/files.txt
--min_depth_eval 1e-3
--max_depth_eval 10
--eigen_crop
""".format(d=data, l=log))
        out, stats = _boot("bts_main.py", "args_train.txt", work, graphs)
        lines = out.splitlines()
        i = next(i for i, ln in enumerate(lines) if ln.startswith("Computing errors for 4 eval samples"))
        metrics[graphs] = lines[i + 2]
        vals = [float(v) for v in metrics[graphs].split(",")]
        assert len(vals) == 9 and np.all(np.isfinite(vals))
        assert stats == ({"captures": 1, "replays": 3, "evictions": 0, "recaptures": 0} if graphs else
                         {"captures": 0, "replays": 0, "evictions": 0, "recaptures": 0})
    assert metrics[True] == metrics[False]
