"""Host half of the device augmentation path: DevicePairDataset makes the same random draws as the unmodified
PairDataset with main_train.py's transforms (the torch, Python and NumPy generators end every item in the same state,
and the masks agree), and pair_collate packs what the kernels read."""
import contextlib
import io
import random

import numpy as np
import pytest
import torch

from oracle import ref_loader
from _augment_data import mask_generator, reference_dataset, write_dataset

pytestmark = pytest.mark.skipif(not ref_loader.available(), reason="reference tree not staged")


def _states():
    return torch.get_rng_state(), random.getstate(), np.random.get_state()[1].tobytes()


@pytest.mark.parametrize("train", [True, False])
def test_draws_match_pairdataset(tmp_path, train):
    from painter_b200.data_gpu import DevicePairDataset
    lists = write_dataset(str(tmp_path), per_type=2)
    with contextlib.redirect_stdout(io.StringIO()):
        ref = reference_dataset(str(tmp_path), lists, train=train, mask_generator=mask_generator())
    ours = DevicePairDataset(str(tmp_path), lists, input_size=(896, 448), min_random_scale=0.3, half_mask_ratio=0.3,
                             use_two_pairs=True, masked_position_generator=mask_generator(), train=train)
    assert ours.weights == ref.weights and ours.pairs == ref.pairs and ours.pair_type_dict == ref.pair_type_dict
    seen = set()
    for i in range(len(ref)):
        for rep in range(2):
            seed = 1000 * i + rep
            torch.manual_seed(seed)
            random.seed(seed)
            np.random.seed(seed)
            _, _, mref, _ = ref[i]
            want = _states()
            torch.manual_seed(seed)
            random.seed(seed)
            np.random.seed(seed)
            images, rec = ours[i]
            got = _states()
            assert torch.equal(want[0], got[0]) and want[1] == got[1] and want[2] == got[2], (i, rep)
            assert np.array_equal(rec["mask"], mref) and rec["mask"].dtype == mref.dtype
            assert len(images) == 4 and all(a.dtype == np.uint8 and a.ndim == 3 for a in images)
            seen.add(("half", rec["half"]))
            seen.add(("sec", rec["sec"] is not None))
            for p in rec["pairs"]:
                seen.add(("jit", p["jitter"] is not None))
                seen.add(("flip", p["flip"]))
    if train:
        assert seen == {(k, v) for k in ("half", "sec", "jit", "flip") for v in (True, False)}, seen


def test_unsupported_recipes_raise(tmp_path):
    from painter_b200.data_gpu import DevicePairDataset
    lists = write_dataset(str(tmp_path), per_type=1)
    with pytest.raises(NotImplementedError):
        DevicePairDataset(str(tmp_path), lists, masked_position_generator=mask_generator(), transforms=object())
    with pytest.raises(NotImplementedError):
        DevicePairDataset(str(tmp_path), lists, masked_position_generator=mask_generator(), use_two_pairs=False)


def test_pair_collate_packing(tmp_path):
    from painter_b200.data_gpu import DevicePairDataset, pair_collate
    lists = write_dataset(str(tmp_path), per_type=2)
    ds = DevicePairDataset(str(tmp_path), lists, masked_position_generator=mask_generator(), half_mask_ratio=0.3)
    torch.manual_seed(3)
    random.seed(3)
    items = [ds[i] for i in range(0, len(ds), 3)]
    pk = pair_collate(items)
    m = pk.meta
    B, P, S = len(items), 2, 448
    assert (m["B"], m["P"], m["S"], m["J"]) == (B, P, S, 4 * B)
    flat = pk.buf.numpy()
    tab = flat[:m["table_bytes"]].view(np.int32)
    o_crop, o_jit, o_sec, o_rule, o_thr, o_mask = m["offs"]
    crop = tab[o_crop:o_jit].reshape(-1, 12)
    tmp_need = 0
    for b, (imgs, rec) in enumerate(items):
        for p in range(P):
            for t in range(2):
                row = crop[(b * P + p) * 2 + t]
                a = imgs[2 * p + t]
                off = int(row[0]) | (int(row[1]) << 32)
                assert np.array_equal(flat[m["table_bytes"] + off:m["table_bytes"] + off + a.size], a.reshape(-1))
                assert tuple(row[2:4]) == a.shape[:2]
                assert tuple(row[4:8]) == rec["pairs"][p]["box"]
                assert row[8] == rec["modes"][t] and row[9] == rec["pairs"][p]["flip"]
                assert (int(row[10]) | (int(row[11]) << 32)) == tmp_need
                tmp_need += max(rec["pairs"][p]["box"][2:]) * S * 3 if rec["modes"][t] == 0 else 0
                if row[8] == 0:
                    assert 2 * int(np.ceil(2 * max(row[6] / S, row[7] / S, 1.0))) + 1 <= m["KP"]
    jit = tab[o_jit:o_sec].reshape(-1, 9)
    want = [(b * P + p) * 2 for b, (_, r) in enumerate(items) for p in range(P) if r["pairs"][p]["jitter"]]
    assert jit[:, 0].tolist() == want
    for row in jit:
        b, p = divmod(int(row[0]) // 2, P)
        order, fb, fc, fs, hue = items[b][1]["pairs"][p]["jitter"]
        assert row[1:5].tolist() == order and row[8] == hue
        assert row[5:8].view(np.float32).tolist() == np.float32([fb, fc, fs]).tolist()
    sec = tab[o_sec:o_rule].reshape(B, 2, 5)
    for b, (_, rec) in enumerate(items):
        for t in range(2):
            want = [*rec["sec"], rec["modes"][t]] if rec["sec"] else [0, 0, 2 * S, S, 1]
            assert sec[b, t].tolist() == want
    masks = tab[o_mask:o_mask + B * 56 * 28].reshape(B, 56, 28)
    assert all(np.array_equal(masks[b], rec["mask"]) for b, (_, rec) in enumerate(items))
    assert m["tmp_bytes"] == max(tmp_need, 1)
