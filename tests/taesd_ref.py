"""fp32 oracle of [3P] diffusers `AutoencoderTiny`'s decoder (`DecoderTiny`, `AutoencoderTinyBlock`), written from the
published structure in plain PyTorch (restated from memory like the other [3P] oracles, parity unpinned).  Same module
tree, so the same state-dict keys (`decoder.layers.*`) as diffusers and as imagharmony_b200.taesd."""
import torch
import torch.nn as nn


class AutoencoderTinyBlockRef(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(cin, cout, 3, padding=1), nn.ReLU(), nn.Conv2d(cout, cout, 3, padding=1),
                                  nn.ReLU(), nn.Conv2d(cout, cout, 3, padding=1))
        self.skip = nn.Conv2d(cin, cout, 1, bias=False) if cin != cout else nn.Identity()
        self.fuse = nn.ReLU()

    def forward(self, x):
        return self.fuse(self.conv(x) + self.skip(x))


class DecoderTinyRef(nn.Module):
    def __init__(self, in_channels, out_channels, num_blocks, block_out_channels, upsampling_scaling_factor=2):
        super().__init__()
        layers = [nn.Conv2d(in_channels, block_out_channels[0], 3, padding=1), nn.ReLU()]
        for i, num_block in enumerate(num_blocks):
            is_final_block = i == len(num_blocks) - 1
            c = block_out_channels[i]
            for _ in range(num_block):
                layers.append(AutoencoderTinyBlockRef(c, c))
            if not is_final_block:
                layers.append(nn.Upsample(scale_factor=upsampling_scaling_factor, mode="nearest"))
            layers.append(nn.Conv2d(c, c if not is_final_block else out_channels, 3, padding=1, bias=is_final_block))
        self.layers = nn.Sequential(*layers)

    def forward(self, x):
        x = torch.tanh(x / 3) * 3          # clamp
        x = self.layers(x)
        return x.mul(2).sub(1)             # [0, 1] -> [-1, 1]


class AutoencoderTinyRef(nn.Module):
    """The decoder half; `decode(latents)` = diffusers' pipelines' `vae.decode(latents / scaling_factor).sample`."""

    def __init__(self, cfg):
        super().__init__()
        self.scaling_factor = cfg.scaling_factor
        self.decoder = DecoderTinyRef(cfg.latent_channels, cfg.out_channels, cfg.num_decoder_blocks,
                                      cfg.decoder_block_out_channels)

    def decode(self, latents):
        return self.decoder(latents / self.scaling_factor)
