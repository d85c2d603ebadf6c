"""CPU: test.py --save_per_img on the ADE20k fixtures, the per-image file names, and the host-side check of the celebahq
glasses slot that Pix2PixModel.run_inference makes before a batch reaches the GPU."""
import contextlib
import importlib.util
import io
import os

import pytest
import torch
import torchvision.utils as vutils

from tests.golden.make_golden_data import FIXTURES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _script():
    spec = importlib.util.spec_from_file_location("cocos_test_script", os.path.join(ROOT, "test.py"))
    script = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(script)
    return script


def test_per_image_names_follow_the_reference():
    name = _script().per_image_name
    for path in ("/data/Dataset/DeepFashion/img/WOMEN/Dresses/id_00000244/02_1_front.jpg",
                 "tests/golden/data/DeepFashion/img/WOMEN/Dresses/id_00000244/02_1_front.jpg"):
        assert name(path, "deepfashion") == path.split("Dataset/DeepFashion/")[-1].replace("/", "_")  # test.py:44
    assert name("/data/Dataset/DeepFashion/img/WOMEN/Dresses/id_00000244/02_1_front.jpg", "deepfashion") == \
        "img_WOMEN_Dresses_id_00000244_02_1_front.jpg"
    assert name("tests/golden/data/DeepFashion/img/x/1.jpg", "deepfashion") == \
        "tests_golden_data_DeepFashion_img_x_1.jpg"
    assert name("/d/ADEChallengeData2016/images/validation/ADE_val_00001232.jpg", "ade20k") == "ADE_val_00001232.jpg"
    assert name("/d/celebahq/CelebA-HQ-img/12.jpg", "celebahq") == "12.jpg"


def _celebahq_model(tmp_path):
    from cocosnet_b200.options import TestOptions
    from cocosnet_b200.pix2pix_model import Pix2PixModel
    opt = TestOptions().parse(["--dataset_mode", "celebahq", "--use_attention", "--maskmix", "--warp_mask_losstype",
                               "direct", "--PONO", "--PONO_C", "--warp_bilinear", "--adaptor_kernel", "4",
                               "--gpu_ids", "-1", "--checkpoints_dir", str(tmp_path)], save=False, verbose=False)
    opt.verbose_networks = False
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        model = Pix2PixModel(opt)
    return opt, model.eval()


def test_celebahq_host_check_matches_preprocess_input(tmp_path):
    from cocosnet_b200 import data as cdata
    opt, model = _celebahq_model(tmp_path)
    good = cdata.synthetic_batch(opt, 2, seed=3)
    model.check_glasses_slot(good)
    model.preprocess_input(good)
    for key in ("label", "label_ref"):
        bad = cdata.synthetic_batch(opt, 2, seed=3)
        bad[key][0, 0, 10:20, 10:20] = opt.semantic_nc - 3  # id 16: the glasses slot
        with pytest.raises(AssertionError) as host:
            model.check_glasses_slot(bad)
        with pytest.raises(AssertionError) as device_side:
            model.preprocess_input(bad)
        assert type(host.value) is type(device_side.value) and str(host.value) == str(device_side.value)
        with pytest.raises(AssertionError):
            model.run_inference(bad)
    bad = cdata.synthetic_batch(opt, 2, seed=3)
    bad["label"][1, 1] = 1  # the glasses channel may be set: only the id channels are checked
    model.check_glasses_slot(bad)


@pytest.mark.timeout(900)
def test_test_py_save_per_img_on_cpu(tmp_path, monkeypatch):
    """Two ADE20k fixture pairs through test.py --save_per_img --gpu_ids -1: one JPEG per item, named after its path,
    no grid, and each file is save_image((fake + 1) / 2) of the eager forward on the same batch."""
    from cocosnet_b200 import data as cdata
    from cocosnet_b200 import util
    from cocosnet_b200.options import TestOptions
    from cocosnet_b200.pix2pix_model import Pix2PixModel
    from oracle import torch_port
    from tests.test_model_parity_cpu import build_inference_model
    monkeypatch.chdir(FIXTURES)  # the reference lists are read from ./data/
    ckpt = tmp_path / "checkpoints"
    opt, model = build_inference_model("ade20k_infer_mk3")
    opt.checkpoints_dir, opt.name = str(ckpt), "ade20k_real"
    util.save_network(model.net["netG"], "G", "latest", opt)
    util.save_network(model.net["netCorr"], "Corr", "latest", opt)
    argv = ["--name", "ade20k_real", "--dataset_mode", "ade20k", "--dataroot", os.path.join(FIXTURES, "ade20k"),
            "--checkpoints_dir", str(ckpt), "--use_attention", "--maskmix", "--PONO", "--PONO_C", "--gpu_ids", "-1",
            "--batchSize", "2", "--how_many", "2", "--nThreads", "0"]
    monkeypatch.setattr("sys.argv", ["test.py", "--save_per_img"] + argv)
    # the model on the CPU: K1 through the oracle's torch expressions, as in the other CPU tests
    with contextlib.redirect_stdout(io.StringIO()), torch_port.cpu_reference_mode():
        _script().main()
    out_dir = tmp_path / "output" / "test_per_img" / "ade20k_real"
    written = sorted(os.listdir(out_dir))
    assert sorted(os.listdir(tmp_path / "output")) == ["test_per_img"]  # no grid

    with contextlib.redirect_stdout(io.StringIO()):
        topt = TestOptions().parse(["--save_per_img"] + argv, save=False, verbose=False)
        torch.manual_seed(0)
        data = next(iter(cdata.create_dataloader(topt)))
        model = Pix2PixModel(topt).eval()
    names = [os.path.basename(p) for p in data["path"]]
    assert written == sorted(names) and all(n.startswith("ADE_val_") and n.endswith(".jpg") for n in names)
    with torch.no_grad(), torch_port.cpu_reference_mode():
        fake = model(data, mode="inference")["fake_image"]
    for j, n in enumerate(names):
        want = tmp_path / ("want_" + n)
        vutils.save_image((fake[j:j + 1] + 1) / 2, str(want), nrow=1, padding=0, normalize=False)
        assert (out_dir / n).read_bytes() == want.read_bytes(), n
