"""N1 / N3 (SURVEY.md section 8f): engine + conditioner glue and the frame writers behind the reference's inference.py
control flow. CPU tests cover the host logic; the GPU test runs the whole entry point on a shrunk copy of the reference
YAML."""
import os
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
CFG = str(ROOT / "tests" / "configs" / "tiny_inference.yaml")


def _engine():
    from panacea_b200.inference import load_config
    from panacea_b200.sgm.util import instantiate_from_config
    return instantiate_from_config(load_config([CFG])["model"])


def test_reference_yaml_structure_instantiates_the_engine_and_resolves_anchors():
    from panacea_b200.inference import load_config
    cfg = load_config([CFG], ["model.params.sampler_config.params.num_steps=7"])
    assert cfg["model"]["params"]["network_config"]["params"]["num_frames"] == 4
    assert cfg["model"]["params"]["sampler_config"]["params"]["num_steps"] == 7
    m = _engine()
    assert type(m).__name__ == "DiffusionEngine3D" and m.num_frames == 4 and m.share_noise_level == 0.07
    assert type(m.model).__name__ == "OpenAIWrapperControlLDM3D"
    assert [type(e).__name__ for e in m.conditioner.embedders] == ["FrozenOpenCLIPEmbedder", "IdentityEncoder", "VAEEmbedder"]
    assert m.conditioner.embedders[2].first_stage_model is m.first_stage_model      # diffusion.py:111-122


def test_conditioner_routing_matches_the_reference_rules():
    """modules.py:147-203: txt -> crossattn [b,77,D]; cond_img -> cond_feat flattened to (b t); final_cond_zero -> VAE latent
    'concat' (b t); the unconditional branch differs only in the text embedding (batch_uc['txt'] = '')."""
    from torch.utils.data import DataLoader
    from panacea_b200.inference import SyntheticBEVDataset
    m = _engine()

    class FakeFirstStage(torch.nn.Module):     # the routing is host logic; the native VAE encoder needs a GPU
        def encode(self, x):
            return torch.nn.functional.avg_pool2d(x, 8)[:, :1].repeat(1, 4, 1, 1)

    m.conditioner.embedders[2].first_stage_model = FakeFirstStage()
    batch = next(iter(DataLoader(SyntheticBEVDataset(2, 4, (64, 128), use_last_frame=True), batch_size=1)))
    bu = dict(batch)
    bu["txt"] = ["" for _ in batch["txt"]]
    c, uc = m.conditioner.get_unconditional_conditioning(batch, batch_uc=bu, force_uc_zero_embeddings=[])
    assert c["crossattn"].shape == (1, 77, 128) and c["cond_feat"].shape == (4, 19, 64, 768) and c["concat"].shape == (4, 4, 8, 96)
    assert not torch.equal(c["crossattn"], uc["crossattn"]) and torch.equal(c["concat"], uc["concat"]) and torch.equal(c["cond_feat"], uc["cond_feat"])
    # use_last_frame: the image-condition frames are zero except the last one (nuscenes_datasets_video.py:559-566)
    assert batch["final_cond_zero"][0, :-1].abs().max() == 0 and batch["final_cond_zero"][0, -1].abs().max() > 0
    _, uz = m.conditioner.get_unconditional_conditioning(batch, force_uc_zero_embeddings=["txt"])
    assert uz["crossattn"].abs().max() == 0


def test_frame_writers_produce_the_streampetr_layout(tmp_path):
    """inference.py:171-196: fake/<scene>_<file stem of the last frame per camera>/_{frame:06}.jpg, 6 cameras x T frames,
    camera i cropped from columns [w*i, w*i+w) with the reference's viewid table."""
    from PIL import Image
    from torch.utils.data import DataLoader
    from panacea_b200 import frame_io as IO
    from panacea_b200.inference import SyntheticBEVDataset
    batch = next(iter(DataLoader(SyntheticBEVDataset(1, 4, (32, 64)), batch_size=1)))
    jpgs = torch.zeros(4, 3, 32, 6 * 64)
    for i in range(6):
        jpgs[:, :, :, 64 * i:64 * i + 64] = -1.0 + 0.4 * i
    written = IO.logs_frames(jpgs, str(tmp_path / "fake"), batch["filenames"])
    assert len(written) == 24
    dirs = sorted(os.listdir(tmp_path / "fake"))
    assert len(dirs) == 6 and all(d.startswith("CAM_") for d in dirs)
    d = [x for x in dirs if x.startswith("CAM_BACK_RIGHT_")][0]
    assert sorted(os.listdir(tmp_path / "fake" / d)) == [f"_{k:06}.jpg" for k in range(4)]
    px = Image.open(tmp_path / "fake" / d / "_000000.jpg").getpixel((5, 5))
    assert abs(px[0] - round((0.4 * IO.VIEW_ID["CAM_BACK_RIGHT"]) / 2 * 255)) <= 3          # strip slot 5
    gifs = IO.logs_all_gifs({"samples": jpgs}, str(tmp_path / "gifs"), batch["filenames"], num_frames=4)
    pngs = IO.logs_all_images({"samples": jpgs}, str(tmp_path / "all"), batch["filenames"])
    assert len(gifs) == 1 and len(pngs) == 1 and Image.open(pngs[0]).size == (384, 128)


@pytest.mark.gpu
def test_inference_entry_point_end_to_end(tmp_path):
    """The whole main(): YAML -> engine -> DistributedSampler/bs=1 loop -> log_images (conditioner, VAE-stub encode,
    share-noise init, 3 Euler/CFG steps on the sm_90a path, decode) -> writers."""
    from panacea_b200 import inference as INF
    written = INF.main(["--name", "t", "--base", CFG, "--inferdir", str(tmp_path), "--num_sequences", "2", "--image_hw", "64", "128",
                        "--randomize_zero_init"])
    jpgs = [w for w in written if w.endswith(".jpg")]
    assert len(jpgs) == 2 * 6 * 4 and all(os.path.getsize(w) > 0 for w in jpgs)
    assert any(w.endswith(".gif") for w in written) and any(w.endswith(".png") for w in written)
