"""Drop-in proven by RUNNING an unmodified reference script: sampler/autoencoding_eval.py (its Sampler class: NCCL init,
DistributedSampler + DataLoader, yaml configs, checkpoint loading with the reference's keys, getattr(decoder_module, ...),
copy.deepcopy(...).cuda(), GaussianDiffusion.representation_learning_autoencoding('ddim1000', 'ddim100', ...), the metric
classes) executes on the pdae_b200 kernels after `pdae_b200.dropin.install()`.

Only what the offline box lacks is stubbed -- matplotlib / lmdb / lpips (third-party imports of utils/utils.py and
metric/lpips, SURVEY D9), a synthetic in-memory dataset registered under the reference's `dataset` module, and a
synthetic checkpoint + config files.  Needs oracle/_ref (installed by __graft_entry__.build() from the original project's
sources, oracle/install_reference.py); skips without it."""
import json
import os
import socket
import subprocess
import sys
import textwrap

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")

SCRIPT = r'''
import argparse, json, os, sys, types
import torch
ROOT, REF, TMP = sys.argv[1], sys.argv[2], sys.argv[3]
sys.path.insert(0, ROOT)
# ---- third-party modules the offline image lacks (imported by utils/utils.py and metric/lpips/lpips_metric.py) ----
for name in ("matplotlib", "matplotlib.pyplot", "lmdb"):
    sys.modules.setdefault(name, types.ModuleType(name))
sys.modules["matplotlib"].pyplot = sys.modules["matplotlib.pyplot"]
lp = types.ModuleType("lpips")
class LPIPS(torch.nn.Module):
    def __init__(self, net="alex"):
        super().__init__()
    def forward(self, a, b):
        return (a - b).abs().mean(dim=[1, 2, 3]).reshape(-1, 1, 1, 1)
lp.LPIPS = LPIPS
sys.modules["lpips"] = lp
# ---- the drop-in: model.* / diffusion.* resolve to pdae_b200, everything else to the unmodified reference ----
import pdae_b200.dropin
pdae_b200.dropin.install()
pdae_b200.set_default_precision("fp32")
sys.path.insert(1, REF)
import dataset as dataset_module
from pdae_b200.utils.synth import fill_named_tensors_, synth_images
class SYNTH(torch.utils.data.Dataset):
    def __init__(self, config):
        self.x = synth_images(config["n"], 3, config["image_size"], 28)
    def __len__(self):
        return self.x.shape[0]
    def __getitem__(self, i):
        return {"x_0": self.x[i]}
    @staticmethod
    def collate_fn(batch):
        return {"x_0": torch.stack([b["x_0"] for b in batch])}
dataset_module.SYNTH = SYNTH
import yaml
tiny = dict(input_channel=3, base_channel=32, channel_multiplier=[1, 2, 2], num_residual_blocks_of_a_block=1,
            attention_resolutions=[2], num_heads=1, head_channel=-1, use_new_attention_order=False, dropout=0.0)
yaml.safe_dump({"diffusion_config": {"timesteps": 1000, "betas_type": "linear"},
                "encoder_config": {"model": "CELEBA64Encoder", "latent_dim": 512},
                "decoder_config": {"model": "CELEBA64Decoder", "latent_dim": 512}}, open(os.path.join(TMP, "config.yml"), "w"))
yaml.safe_dump({"denoise_fn_config": dict(tiny, model="CELEBA64DenoiseFn")}, open(os.path.join(TMP, "ddpm.yml"), "w"))
import model.representation_learning.encoder as encoder_module
import model.representation_learning.decoder as decoder_module
assert encoder_module.__name__.startswith("pdae_b200"), encoder_module.__name__
enc = encoder_module.CELEBA64Encoder(latent_dim=512)
dec = decoder_module.CELEBA64Decoder(latent_dim=512, **tiny)
esd, dsd = enc.state_dict(), dec.state_dict()
fill_named_tensors_(esd.items(), 7)
fill_named_tensors_(dsd.items(), 6)
torch.save({"ema_encoder": esd, "ema_decoder": dsd}, os.path.join(TMP, "checkpoint.pt"))

import sampler.autoencoding_eval as script            # the UNMODIFIED reference script
assert os.path.realpath(script.__file__).startswith(os.path.realpath(REF)), script.__file__
assert script.GaussianDiffusion.__module__.startswith("pdae_b200")
args = argparse.Namespace()
args.config = {"diffusion_config": {"timesteps": 1000, "betas_type": "linear"},
               "config_path": os.path.join(TMP, "config.yml"), "checkpoint_path": os.path.join(TMP, "checkpoint.pt"),
               "trained_ddpm_config_path": os.path.join(TMP, "ddpm.yml"),
               "dataset_config": {"dataset_name": "SYNTH", "n": 3, "image_channel": 3, "image_size": 64, "augmentation": False},
               "batch_size": 2, "num_workers": 0}
runner = script.Sampler(args)
assert type(runner.decoder).__module__.startswith("pdae_b200") and type(runner.encoder).__module__.startswith("pdae_b200")
runner.start()
res = {"mse": runner.mse_metric.results, "ssim": runner.ssim_metric.results, "lpips": runner.lpips_metric.results}
# the same call outside the script, for comparison
with torch.inference_mode():
    x0 = synth_images(3, 3, 64, 28).cuda()
    rec = runner.gaussian_diffusion.representation_learning_autoencoding("ddim1000", "ddim100", runner.encoder, runner.decoder, x0[:2])
    res["mse_direct"] = (((x0[:2] + 1) / 2 - (rec + 1) / 2) ** 2).mean(dim=[1, 2, 3]).tolist()
print("RESULT " + json.dumps(res))
torch.distributed.destroy_process_group()
'''


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_reference_autoencoding_eval_script_runs_on_native_kernels(tmp_path):
    if not os.path.exists(os.path.join(REF, "sampler", "autoencoding_eval.py")):
        pytest.skip("oracle/_ref not installed (__graft_entry__.build() installs it when the original project's sources are available)")
    script = tmp_path / "run_ref_script.py"
    script.write_text(textwrap.dedent(SCRIPT))
    env = dict(os.environ, RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", LOCAL_WORLD_SIZE="1", MASTER_ADDR="127.0.0.1",
               MASTER_PORT=str(_free_port()))
    r = subprocess.run([sys.executable, str(script), ROOT, REF, str(tmp_path)], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + "\n" + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1]
    res = json.loads(line[len("RESULT "):])
    assert len(res["mse"]) == len(res["ssim"]) == len(res["lpips"]) == 3          # 3 images in batches of 2 + 1
    assert all(0.0 <= m < 1.0 for m in res["mse"]) and all(-1.0 <= s <= 1.0 for s in res["ssim"])
    for a, b in zip(res["mse"][:2], res["mse_direct"]):
        assert abs(a - b) <= 1e-6 + 1e-3 * abs(b), (res["mse"], res["mse_direct"])
    assert "sampler initialized" in r.stdout
