"""GPU: Pix2PixModel.run_inference -- the inference forward replayed from one CUDA graph -- against the eager
`model(batch, mode="inference")`, bit for bit, and test.py's output files with the graph on and off."""
import contextlib
import importlib.util
import io
import os
import shutil

import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from tests.golden.make_golden_data import FIXTURES  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# the reference README's test flags (batch sizes aside)
CONFIGS = {
    "ade20k": ["--dataset_mode", "ade20k", "--use_attention", "--maskmix", "--warp_mask_losstype", "direct", "--PONO",
               "--PONO_C"],
    "celebahq": ["--dataset_mode", "celebahq", "--use_attention", "--maskmix", "--warp_mask_losstype", "direct",
                 "--PONO", "--PONO_C", "--warp_bilinear", "--adaptor_kernel", "4"],
    "deepfashion": ["--dataset_mode", "deepfashion", "--use_attention", "--PONO", "--PONO_C", "--warp_bilinear",
                    "--no_flip", "--warp_patch", "--video_like", "--adaptor_kernel", "4"],
}
COMPARED = ("fake_image", "warp_out", "warp_mask")


@pytest.fixture(autouse=True)
def graphs_on(monkeypatch):
    monkeypatch.delenv("COCOS_CUDA_GRAPH", raising=False)


def converge_spectral_norms(model, iters=30):
    """Power-iterate every spectral norm's u, v to the top singular vectors, as a trained checkpoint has them.  In
    eval() no iteration runs, and with the freshly drawn u, v of a seeded init sigma can come out so small that the
    generator's SAGAN block overflows on the GPU (celebahq: non-finite fake_image)."""
    from torch.nn.utils.spectral_norm import SpectralNorm
    with torch.no_grad():
        for m in model.modules():
            for hook in m._forward_pre_hooks.values():
                if isinstance(hook, SpectralNorm):
                    for _ in range(iters):
                        hook.compute_weight(m, do_power_iteration=True)


def build(config, tmp_path, seed=0, extra=()):
    """Seeded test-time model (no checkpoint under tmp_path: the initialisation stays), in eval() on the GPU."""
    from cocosnet_b200.options import TestOptions
    from cocosnet_b200.pix2pix_model import Pix2PixModel
    opt = TestOptions().parse(CONFIGS[config] + list(extra) + ["--gpu_ids", "-1", "--batchSize", "2",
                                                                  "--checkpoints_dir", str(tmp_path / "none")],
                              save=False, verbose=False)
    opt.verbose_networks = False
    torch.manual_seed(seed)
    with contextlib.redirect_stdout(io.StringIO()):  # "not find model": the seeded weights stay
        model = Pix2PixModel(opt)
    converge_spectral_norms(model)
    opt.gpu_ids = [0]
    model.cuda().eval()
    return opt, model


def batch(opt, seed, n=2):
    from cocosnet_b200 import data as cdata
    return cdata.synthetic_batch(opt, n, seed=seed)


def graphed(model, data):
    """run_inference(data) and the number of C-ABI launches it enqueued from Python."""
    from cocosnet_b200 import _lib
    l0 = _lib.LAUNCHES
    out = model.run_inference(data)
    torch.cuda.synchronize()
    return out, _lib.LAUNCHES - l0


def assert_same(got, want):
    assert set(got) == set(want)
    for k in COMPARED:
        if want.get(k) is None:
            assert got.get(k) is None, k
            continue
        assert torch.isfinite(want[k]).all(), k
        assert torch.equal(got[k], want[k]), (k, float((got[k] - want[k]).abs().max()))


@pytest.mark.timeout(900)
@pytest.mark.parametrize("config", list(CONFIGS))
def test_replay_equals_eager_bit_for_bit(config, tmp_path):
    """Four different batches: warm-up, capture, two replays.  Every call equals the eager forward on the same batch;
    the replays enqueue no C-ABI launch, and the third call's tensors survive the fourth."""
    opt, model = build(config, tmp_path)
    returned, copies, launches = [], [], []
    for i in range(4):
        data = batch(opt, 500 + i)
        got, n = graphed(model, data)
        with torch.no_grad():
            want = model(data, mode="inference")
        assert_same(got, want)
        returned.append(got)
        copies.append({k: got[k].clone() for k in COMPARED if got.get(k) is not None})
        launches.append(n)
        if i == 1:
            assert model._infer["graph"] is not None, model.infer_graph_error
    print(config, "C-ABI launches per call:", launches)
    assert launches[0] > 0 and launches[2] == 0 and launches[3] == 0, launches
    assert not torch.equal(copies[2]["fake_image"], copies[3]["fake_image"])  # different batches, different images
    for k in copies[2]:  # no aliasing: what call 3 returned is untouched by call 4
        assert torch.equal(returned[2][k], copies[2][k]), k


@pytest.mark.timeout(900)
def test_other_batch_size_runs_eagerly_after_the_capture(tmp_path):
    opt, model = build("ade20k", tmp_path)
    for i in range(3):
        graphed(model, batch(opt, 600 + i))
    small = batch(opt, 610, n=1)
    got, n = graphed(model, small)
    assert n > 0  # eager: not the captured shapes
    with torch.no_grad():
        assert_same(got, model(small, mode="inference"))
    data = batch(opt, 611)
    got, n = graphed(model, data)
    assert n == 0  # the captured shape still replays
    with torch.no_grad():
        assert_same(got, model(data, mode="inference"))


@pytest.mark.timeout(900)
def test_in_place_weight_update_reaches_the_replay(tmp_path):
    opt, model = build("ade20k", tmp_path)
    for i in range(2):
        graphed(model, batch(opt, 700 + i))
    data = batch(opt, 710)
    before, _ = graphed(model, data)
    _, other = build("ade20k", tmp_path, seed=1)
    for k in ("netG", "netCorr"):
        model.net[k].load_state_dict(other.net[k].state_dict())
    got, n = graphed(model, data)
    assert n == 0  # same storage: no re-capture
    with torch.no_grad():
        want = model(data, mode="inference")
        assert_same(got, want)
        assert_same(got, other(data, mode="inference"))
    assert not torch.equal(got["fake_image"], before["fake_image"])

    # a replaced parameter tensor: the graph would read the old storage, so the signature changes -> warm-up, capture
    name = next(n for n, _ in model.net["netCorr"].named_parameters())
    owner, leaf = name.rsplit(".", 1) if "." in name else ("", name)
    mod = model.net["netCorr"].get_submodule(owner)
    setattr(mod, leaf, torch.nn.Parameter(getattr(mod, leaf).detach() * 0.5))
    with torch.no_grad():
        want = model(data, mode="inference")
    counts = []
    for _ in range(3):
        got, n = graphed(model, data)
        assert_same(got, want)
        counts.append(n)
    assert counts[0] > 0 and counts[2] == 0, counts


@pytest.mark.timeout(900)
def test_noise_for_mask_stays_eager(tmp_path):
    """--noise_for_mask draws random numbers inside the forward: never captured, and the same seed gives forward's
    output."""
    opt, model = build("ade20k", tmp_path, extra=["--noise_for_mask"])
    for i in range(4):
        data = batch(opt, 800 + i)
        torch.manual_seed(42 + i)
        got, n = graphed(model, data)
        torch.manual_seed(42 + i)
        with torch.no_grad():
            want = model(data, mode="inference")
        assert n > 0 and model._infer["graph"] is None
        assert_same(got, want)


@pytest.mark.timeout(900)
def test_celebahq_glasses_slot_is_checked_on_a_replay(tmp_path):
    opt, model = build("celebahq", tmp_path)
    for i in range(3):
        graphed(model, batch(opt, 900 + i))
    assert model._infer["graph"] is not None
    for key in ("label", "label_ref"):
        bad = batch(opt, 910)
        bad[key][1, 0, 100:120, 30:50] = opt.semantic_nc - 3  # id 16: the glasses slot
        with pytest.raises(AssertionError):
            model.run_inference(bad)
    good = batch(opt, 911)
    got, n = graphed(model, good)
    assert n == 0
    with torch.no_grad():
        assert_same(got, model(good, mode="inference"))


def _run_test_py(run_dir, ckpt, argv, monkeypatch, graph):
    """test.py's main() with a copy of the checkpoints under run_dir; returns {relative path: bytes} of its output."""
    shutil.copytree(ckpt, run_dir / "checkpoints")
    spec = importlib.util.spec_from_file_location("cocos_test_script", os.path.join(ROOT, "test.py"))
    script = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(script)
    monkeypatch.setenv("COCOS_CUDA_GRAPH", "1" if graph else "0")
    monkeypatch.setattr("sys.argv", ["test.py", "--checkpoints_dir", str(run_dir / "checkpoints")] + argv)
    with contextlib.redirect_stdout(io.StringIO()):
        script.main()
    out = run_dir / "output"
    return {str(p.relative_to(out)): p.read_bytes() for p in sorted(out.rglob("*")) if p.is_file()}


@pytest.mark.timeout(900)
@pytest.mark.parametrize("per_img", [False, True])
def test_test_py_files_equal_the_eager_run(per_img, tmp_path, monkeypatch):
    """The six ADE20k fixture pairs in batches of two (warm-up, capture, replay): the grids, or with --save_per_img the
    per-image JPEGs, are byte-identical to a run under COCOS_CUDA_GRAPH=0."""
    from cocosnet_b200 import util
    from tests.test_model_parity_cpu import build_inference_model
    monkeypatch.chdir(FIXTURES)  # the reference lists are read from ./data/
    ckpt = tmp_path / "ckpt"
    opt, model = build_inference_model("ade20k_infer_mk3")
    opt.checkpoints_dir, opt.name = str(ckpt), "ade20k_real"
    util.save_network(model.net["netG"], "G", "latest", opt)
    util.save_network(model.net["netCorr"], "Corr", "latest", opt)
    argv = ["--name", "ade20k_real", "--dataset_mode", "ade20k", "--dataroot", os.path.join(FIXTURES, "ade20k"),
            "--use_attention", "--maskmix", "--warp_mask_losstype", "direct", "--PONO", "--PONO_C", "--gpu_ids", "0",
            "--batchSize", "2", "--nThreads", "2"] + (["--save_per_img"] if per_img else [])
    graph = _run_test_py(tmp_path / "graph", ckpt, argv, monkeypatch, True)
    eager = _run_test_py(tmp_path / "eager", ckpt, argv, monkeypatch, False)
    if per_img:
        assert len(graph) == 6 and all(k.startswith("test_per_img/ade20k_real/ADE_val_") and k.endswith(".jpg")
                                       for k in graph), sorted(graph)
    else:
        assert sorted(graph) == ["ade20k_real/0.png", "ade20k_real/1.png", "ade20k_real/2.png"]
    assert sorted(graph) == sorted(eager)
    for k in graph:
        assert graph[k] == eager[k], k
