"""Host side of the training augmentation on the device (fasterseg_b200.trainpre, fsb_train_pre) without a GPU: the worker's random
draws against the reference's, the arithmetic specification (the numpy stand-in) against every golden the reference wrote, which
loaders take the device path, the launcher's hook of the drivers' dataloader module, the rank-sharded sampler, and the marshalling
of the wrapper against the header."""
import ctypes as C
import os
import random
import re
import sys
import textwrap
import types

import numpy as np
import pytest
import torch
import torch.utils.data as tud

from fasterseg_b200 import _lib
from fasterseg_b200 import functional as F_
from fasterseg_b200 import launch
from fasterseg_b200 import trainpre
from oracle import make_golden_trainpre as G
from tests import trainpre_dataset, trainpre_standin
from tests.test_marshalling_cpu import fake  # noqa: F401  (fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.abspath(__file__)          # defines the BaseDataset below, which stands for the reference's
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "trainpre.npz"))
MEAN, STD = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])


def case(name):
    """-> (inputs, config, seed, draws) of a golden case"""
    H, W, k, ch, cw, g, seed, *draws = GOLDEN[name + "/meta"].tolist()
    scales = GOLDEN[name + "/scales"].tolist()
    cfg = G.config((ch, cw), scales if name != "no_scale_array" else None, g)
    return G.synthetic_pair(H, W, k), cfg, seed, tuple(draws)


def device_inputs(pairs, cfg, draws):
    """what collate + to_device hand to functional.train_pre for these (image, label) pairs and draws"""
    recs = [[img.shape[0], img.shape[1], *d, cfg.image_height, cfg.image_width, *trainpre.label_size(cfg)]
            for (img, _), d in zip(pairs, draws)]
    geom, (ch, cw, lh, lw) = trainpre.check_geometry(np.array(recs))
    src = torch.cat([torch.from_numpy(img).reshape(-1) for img, _ in pairs])
    gt = torch.cat([torch.from_numpy(g).reshape(-1) for _, g in pairs])
    return src, gt, geom, trainpre.normalization_lut(MEAN, STD), (ch, cw), (lh, lw)


def bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


ALL = list(GOLDEN["cases"])
SMALL = [n for n in ALL if n not in set(GOLDEN["full_cases"])]
FULL = list(GOLDEN["full_cases"])


# ---- the worker's draws ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ALL)
def test_draws_and_rng_consumption_match_the_reference(name):
    (img, gt), cfg, seed, draws = case(name)
    random.seed(seed)
    assert trainpre.draw(img.shape[0], img.shape[1], cfg) == draws
    assert random.random() == float(GOLDEN[name + "/next_random"])
    random.seed(seed)
    data, label, extra = trainpre.DeviceTrainPre(types.SimpleNamespace(config=cfg, img_mean=MEAN, img_std=STD))(img, gt)
    assert random.random() == float(GOLDEN[name + "/next_random"])
    assert data.size == 0 and label.size == 0 and not any("img" in k or "label" in k for k in extra)
    assert extra[trainpre.SRC_KEY] is img and extra[trainpre.GT_KEY] is gt
    assert extra[trainpre.GEOM_KEY].tolist()[2:7] == list(draws)


# ---- the arithmetic specification -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", SMALL)
def test_standin_is_bit_identical_to_the_reference(name):
    pair, cfg, _, draws = case(name)
    data, label = trainpre_standin.train_pre(*device_inputs([pair], cfg, [draws]))
    assert bits_equal(data[0].numpy(), GOLDEN[name + "/data"])
    assert bits_equal(label[0].numpy(), GOLDEN[name + "/label"])


@pytest.mark.parametrize("name", FULL)
def test_standin_full_size_digests(name):
    pair, cfg, _, draws = case(name)
    data, label = trainpre_standin.train_pre(*device_inputs([pair], cfg, [draws]))
    assert G.digest(data[0].numpy()) == str(GOLDEN[name + "/data_sha256"])
    assert G.digest(label[0].numpy()) == str(GOLDEN[name + "/label_sha256"])


def test_check_geometry_rejects_what_the_kernel_must_not_see():
    good = [37, 53, 1, 46, 66, 23, 35, 24, 32, 3, 4]
    geom, size = trainpre.check_geometry(np.array([good, good]))
    assert size == (24, 32, 3, 4) and geom[:, 7].tolist() == [0, 37 * 53] and geom.dtype == torch.int32
    for i, v in ((5, 46), (6, -1), (2, 2), (3, 0), (9, 25), (10, 0)):
        bad = list(good)
        bad[i] = v
        with pytest.raises(ValueError):
            trainpre.check_geometry(np.array([good, bad] if i < 7 else [bad]))
    other = list(good)
    other[8] = 48
    with pytest.raises(ValueError):
        trainpre.check_geometry(np.array([good, other]))


# ---- which loaders take the device path ----------------------------------------------------------------------------------------------
class TrainPre:
    def __init__(self, config, img_mean, img_std):
        self.config, self.img_mean, self.img_std = config, img_mean, img_std


class BaseDataset(tud.Dataset):
    """item protocol of tools/datasets/BaseDataset.py: preprocess -> tensors, extra_dict merged into the item"""

    def __init__(self, pairs, preprocess):
        self.pairs, self.preprocess = pairs, preprocess

    def __len__(self):
        return len(self.pairs)

    def __getitem__(self, i):
        img, gt = self.pairs[i]
        img, gt, extra = self.preprocess(img, gt)
        out = dict(data=torch.from_numpy(np.ascontiguousarray(img)).float(), label=torch.from_numpy(np.ascontiguousarray(gt)).long(),
                   fn="item%d" % i, n=len(self.pairs))
        for k, v in (extra or {}).items():
            out[k] = torch.from_numpy(np.ascontiguousarray(v))
        return out


class OwnItems(BaseDataset):
    def __getitem__(self, i):
        return super().__getitem__(i)


CFG = G.config((24, 32), [0.75, 1, 1.25], 8)
PAIRS = [G.synthetic_pair(37, 53, k) for k in range(3)] + [G.synthetic_pair(41, 47, 3)]


def _loader(pre=None, dataset=BaseDataset, **kw):
    return tud.DataLoader(dataset(PAIRS, pre or TrainPre(CFG, MEAN, STD)), batch_size=2, shuffle=True, drop_last=True, **kw)


@pytest.fixture
def cuda_host(monkeypatch):
    """pretend CUDA is present and run the device step on the CPU stand-in"""
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(trainpre, "_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(F_, "train_pre", trainpre_standin.train_pre)


def test_eligible_loader_is_wrapped_and_yields_the_reference_batches(cuda_host):
    loader = trainpre.wrap_loader(_loader(), TrainPre, HERE)
    assert isinstance(loader, trainpre.DeviceTrainLoader) and len(loader) == 2 and loader.batch_size == 2
    assert isinstance(loader.dataset.preprocess, trainpre.DeviceTrainPre) and loader.collate_fn is trainpre.collate
    random.seed(3)
    torch.manual_seed(3)
    it = iter(loader)
    batches = [it.next(), next(it)]
    with pytest.raises(StopIteration):
        next(it)
    assert sorted(fn for b in batches for fn in b["fn"]) == ["item%d" % i for i in range(4)]
    random.seed(3)                                      # no workers: the draws come from this process's stream, in batch order
    for b in batches:
        idx = [int(fn[4:]) for fn in b["fn"]]
        assert set(b) == {"data", "label", "fn", "n"} and b["n"].tolist() == [4, 4]
        assert b["data"].shape == (2, 3, 24, 32) and b["data"].dtype == torch.float32
        assert b["label"].shape == (2, 3, 4) and b["label"].dtype == torch.int64
        for j, i in enumerate(idx):
            img, gt = PAIRS[i]
            d = trainpre.draw(img.shape[0], img.shape[1], CFG)
            want = trainpre_standin.train_pre(*device_inputs([PAIRS[i]], CFG, [d]))
            assert torch.equal(b["data"][j], want[0][0]) and torch.equal(b["label"][j], want[1][0])


def test_foreign_preprocess_custom_collate_and_own_getitem_keep_the_reference_path(cuda_host):
    class OtherPre(TrainPre):
        pass

    for loader in (_loader(OtherPre(CFG, MEAN, STD)), _loader(dataset=OwnItems), _loader(collate_fn=lambda b: b)):
        pre = loader.dataset.preprocess
        assert trainpre.wrap_loader(loader, TrainPre, HERE) is loader and loader.dataset.preprocess is pre


def test_a_basedataset_from_another_file_keeps_the_reference_path(cuda_host, tmp_path):
    other = tmp_path / "BaseDataset.py"
    other.write_text("")
    loader = _loader()
    assert trainpre.wrap_loader(loader, TrainPre, str(other)) is loader and type(loader.dataset.preprocess) is TrainPre
    assert trainpre.wrap_loader(loader, TrainPre, None) is loader
    assert isinstance(trainpre.wrap_loader(_loader(), TrainPre, os.path.join(os.path.dirname(HERE), ".", os.path.basename(HERE))),
                      trainpre.DeviceTrainLoader)


def test_reference_base_dataset_is_found_next_to_the_dataloader_module():
    mod = types.SimpleNamespace(__file__="/x/FasterSeg/search/dataloader.py")
    assert trainpre.reference_base_dataset(mod) == "/x/FasterSeg/tools/datasets/BaseDataset.py"
    assert trainpre.reference_base_dataset(types.SimpleNamespace()) is None


def test_no_cuda_keeps_the_reference_path(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    loader = _loader()
    assert trainpre.wrap_loader(loader, TrainPre, HERE) is loader and type(loader.dataset.preprocess) is TrainPre


def test_rank_sharded_sampler_still_applies(cuda_host, monkeypatch):
    monkeypatch.setattr(tud.DataLoader, "__init__", tud.DataLoader.__init__)
    monkeypatch.delattr(tud.DataLoader, "_fsb_sharded", raising=False)
    launch.install_rank_sharded_loaders(1, 2)
    loader = trainpre.wrap_loader(_loader(), TrainPre, HERE)
    assert isinstance(loader, trainpre.DeviceTrainLoader) and isinstance(loader.sampler, launch.RankShardSampler)
    shard = list(iter(loader.sampler))
    loader.sampler.epoch = 0
    b = next(iter(loader))
    assert b["fn"] == ["item%d" % i for i in shard] and b["data"].shape == (2, 3, 24, 32)


def test_install_wraps_get_train_loader_once():
    calls = []
    mod = types.SimpleNamespace(TrainPre=TrainPre, get_train_loader=lambda *a, **k: calls.append((a, k)) or "loader")
    trainpre.install(mod)
    first = mod.get_train_loader
    trainpre.install(mod)
    assert mod.get_train_loader is first and first._fsb_original is not None
    assert first("cfg", "ds", portion=1) == "loader" and calls == [(("cfg", "ds"), {"portion": 1})]


# ---- launcher ------------------------------------------------------------------------------------------------------------------------
_STUB_DATALOADER = textwrap.dedent('''
    class TrainPre(object):
        pass

    def get_train_loader(config, dataset, portion=None, worker=None, test=False):
        return "reference loader"
''')


@pytest.fixture
def clean_import_state():
    path, meta = list(sys.path), list(sys.meta_path)
    saved = sys.modules.pop("dataloader", None)
    yield
    sys.path[:] = path
    sys.meta_path[:] = meta
    sys.modules.pop("dataloader", None)
    if saved is not None:
        sys.modules["dataloader"] = saved


@pytest.mark.parametrize("flavour", ["train", "search"])
def test_launcher_hooks_the_drivers_dataloader_module(tmp_path, clean_import_state, flavour):
    d = tmp_path / "FasterSeg" / flavour
    d.mkdir(parents=True)
    (d / "dataloader.py").write_text(_STUB_DATALOADER)
    finder = launch.install_dataloader_patch(str(d / "train.py"))
    assert finder is not None and sys.meta_path[0] is finder
    sys.path.insert(0, str(d))                                            # what runpy's script directory on sys.path does
    import dataloader
    assert dataloader.get_train_loader._fsb_original is not None
    assert dataloader.get_train_loader(None, None) == "reference loader"   # not a DataLoader over BaseDataset: unchanged


def test_launcher_changes_nothing_without_a_dataloader_module(tmp_path, clean_import_state):
    meta = list(sys.meta_path)
    assert launch.install_dataloader_patch(str(tmp_path / "train.py")) is None and sys.meta_path == meta


# ---- end to end: 4 PNG pairs, batch 2, 2 workers -------------------------------------------------------------------------------------
def write_e2e_pngs(root):
    import cv2
    lines = []
    for k in range(G.E2E["images"]):
        img, gt = G.synthetic_pair(G.E2E["H"], G.E2E["W"], k)
        cv2.imwrite(str(root / ("img%d.png" % k)), img[:, :, ::-1])
        cv2.imwrite(str(root / ("gt%d.png" % k)), gt)
        lines.append("img%d.png gt%d.png\n" % (k, k))
    (root / "train.txt").write_text("".join(lines))


def _iterate(loader, pin_memory):
    assert isinstance(loader, trainpre.DeviceTrainLoader) and loader.pin_memory
    loader.loader.pin_memory = pin_memory
    return list(iter(loader))


def e2e_batches(tmp_path, pin_memory=True):
    """the golden end-to-end case through the reference's own get_train_loader and Cityscapes dataset, wrapped as the launcher
    wraps them (skipped where no copy of the reference is available)"""
    from oracle import ref_harness
    if not ref_harness.reference_available():
        pytest.skip("no copy of the reference")
    ns, datasets = G.load_reference()
    write_e2e_pngs(tmp_path)
    trainpre.install(ns.dataloader)
    return _iterate(G.e2e_loader(ns.dataloader, datasets, str(tmp_path)), pin_memory)


def e2e_batches_standalone(tmp_path, pin_memory=True):
    """the same case through tests/trainpre_dataset.py's PNG dataset and DataLoader (the reference's item protocol and loader
    settings), with the same seeds: runs everywhere"""
    e = G.E2E
    write_e2e_pngs(tmp_path)
    random.seed(e["seed"])
    torch.manual_seed(e["seed"])
    pre = TrainPre(G.config(e["crop"], e["scales"], e["g"]), MEAN, STD)
    loader = trainpre_dataset.train_loader(str(tmp_path), pre, e["batch"], e["workers"])
    return _iterate(trainpre.wrap_loader(loader, TrainPre, trainpre_dataset.__file__), pin_memory)


def check_e2e(batches):
    assert len(batches) == int(GOLDEN["e2e_batches"])
    for i, b in enumerate(batches):
        assert set(b) == {"data", "label", "fn", "n"}
        assert bits_equal(b["data"].cpu().numpy(), GOLDEN["e2e_data_%d" % i])
        assert bits_equal(b["label"].cpu().numpy(), GOLDEN["e2e_label_%d" % i])
        assert list(b["fn"]) == GOLDEN["e2e_fn_%d" % i].tolist() and b["n"].tolist() == GOLDEN["e2e_n_%d" % i].tolist()


def test_end_to_end_loader_on_the_standin(tmp_path, cuda_host):
    check_e2e(e2e_batches(tmp_path, pin_memory=False))      # pinning needs a real CUDA device


def test_end_to_end_standalone_loader_on_the_standin(tmp_path, cuda_host):
    check_e2e(e2e_batches_standalone(tmp_path, pin_memory=False))


# ---- marshalling -----------------------------------------------------------------------------------------------------------------------
def test_signature_table_matches_the_header():
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "fsb200.h")).read(), flags=re.S)
    params = [p.strip() for p in re.search(r"int\s+fsb_train_pre\s*\(([^)]*)\)", src).group(1).split(",")]
    assert len(params) == 8 and params[0].startswith("const fsb_train_pre_desc*")
    res, args = _lib._SIGS["fsb_train_pre"]
    assert res is C.c_int and args[0] is C.POINTER(_lib.TrainPreDesc) and args[1:] == [C.c_void_p] * 7
    body = src[src.index("typedef struct fsb_train_pre_desc {"):src.index("} fsb_train_pre_desc;")]
    names = [n.strip() for decl in re.findall(r"int32_t\s+([^;]+);", body) for n in decl.split(",")]
    assert names == [f for f, _ in _lib.TrainPreDesc._fields_]


def test_train_pre_marshalling(fake):  # noqa: F811
    seen = []
    proto = C.CFUNCTYPE(C.c_int, C.POINTER(_lib.TrainPreDesc), *[C.c_void_p] * 7)

    def record(d, *ptrs):
        seen.append(([getattr(d.contents, f) for f, _ in _lib.TrainPreDesc._fields_], list(ptrs)))
        return 0

    fake.fsb_train_pre = proto(record)
    pair, cfg, _, draws = case("mirror_s125_edge_both")
    src, gt, geom, lut, crop, lab = device_inputs([pair, pair], cfg, [draws, draws])
    data, label = F_.train_pre(src, gt, geom, lut, crop, lab)
    assert data.shape == (2, 3, 24, 32) and data.dtype == torch.float32 and label.shape == (2, 3, 4) and label.dtype == torch.int64
    desc, ptrs = seen[-1]
    assert desc == [2, 24, 32, 3, 4]
    assert ptrs == [t.data_ptr() for t in (src, gt, geom, lut, data, label)] + [None]
    for bad in (dict(geom=geom.long()), dict(geom=geom[:, :7].contiguous()), dict(src=src.int()), dict(gt=gt.long()),
                dict(lut=lut[:2]), dict(lut=lut.double()), dict(out_img=data[:, :2]), dict(out_gt=label.int()),
                dict(lut=lut.to("meta"))):                                          # another device
        kw = dict(src=src, gt=gt, geom=geom, lut=lut, out_img=data, out_gt=label)
        kw.update(bad)
        with pytest.raises(ValueError):
            F_.train_pre(kw["src"], kw["gt"], kw["geom"], kw["lut"], crop, lab, out_img=kw["out_img"], out_gt=kw["out_gt"])
