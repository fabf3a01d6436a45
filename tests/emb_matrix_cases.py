# coding=utf-8
"""The --emb_size matrix: one embedding width per cell row width cpad = roundup(E, 32) + 256 that E in
range(8, 257, 8) reaches (288 ... 512), each with an x block that fills its padding and one narrower than it
(cx < cxp: channels [cx, cxp) of the x block are padding that every kernel must keep inert).  Also the configurations
of the goldens of tests/golden/make_golden_emb_matrix.py (oracle.multiverse_ref.default_config overrides and
seeds)."""

HID = 256
# cpad: (x block that fills the 32-channel padding, x block narrower than it)
CPADS = {
    288: (32, 8),
    320: (64, 40),
    352: (96, 72),
    384: (128, 120),
    416: (160, 136),
    448: (192, 184),
    480: (224, 200),
    512: (256, 248),
}
# cpads that no earlier test launches: three x chunks (416, 448), four with a trailing 32-channel chunk (480)
NEW_CPADS = (416, 448, 480)
PADDED = [CPADS[c][1] for c in sorted(CPADS)]
# what tests/test_emb_matrix_gpu.py launches: the cell forward and the backward GEMMs at both x blocks of every new
# cpad and at every padded one (the other full x blocks run in test_emb_size_gpu.py and test_kernels_atsize_gpu.py)
MATRIX = sorted(set(PADDED) | {CPADS[c][0] for c in NEW_CPADS})


def cpad_of(e):
  """cpad of an x block of e channels (ops.cell_cpad, restated)."""
  return (e + 31) // 32 * 32 + HID


# name: (default_config overrides, seed)
ROLLOUTS = {
    # test.py --use_scene_enc --use_gnn --emb_size 40: greedy decode of both scales, 24 padded x channels (cpad 320)
    "greedy_two_scale_emb40": (dict(batch_size=3, emb_size=40, use_gnn=True), 97),
}
# name: (overrides, seed) of one Model + Trainer step (loss weights 1.0 / 0.2, wd 0.001, Adadelta at 0.3, clip 10)
TRAIN = {
    # train.py --emb_size 136 without --use_scene_enc: class encoder and both decoders at cpad 416, 24 padded channels
    "no_scene_enc_emb136": (dict(batch_size=2, emb_size=136, use_scene_enc=False, use_gnn=False), 98),
}
TRAIN_ARGS = dict(grid_loss_weight=1.0, grid_reg_loss_weight=0.2, wd=0.001, init_lr=0.3, clip_gradient_norm=10.0,
                  optimizer="adadelta")
