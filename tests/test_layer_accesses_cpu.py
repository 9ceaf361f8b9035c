"""What each layer states about its forward (Layer::Accesses), and the storages and readers the net derives from it,
host only: nets are built without a device, as in test_net_cpu.py.

(a) The activation plan (its describe text, as a sha256) of all 23 shipped deploy nets, at their drivers' net sizes and
    one more row and column (odd extents: folded pools run themselves), batch 8, both precisions, keeping nothing and,
    where the net has it, conv4_3.  The plan is made from the layers' statements alone, so this pins every statement
    on every shipped layer.
(b) Net::last_reader("data") of every shipped net, and of two small nets where data is read only through a top that
    shares its bytes (a Dropout with its own top, a one-bottom Concat): the last reader is the Convolution behind it.
    An asynchronous input upload waits for that layer, so it must see through the alias.

The pinned values were taken before the layers stated their accesses, from a plan that restated each layer type's
accesses itself; make_layer_accesses_pins.py prints them again."""
import hashlib
import subprocess
import tarfile
from pathlib import Path

import pytest

from test_activation_reuse_cpu import _net_hw

ROOT = Path(__file__).resolve().parent.parent

PROBE = r"""
#include <cstdio>

#include "caffe/caffe.hpp"

using namespace caffe;

int main(int argc, char** argv) {
  Caffe::set_mode(Caffe::GPU);
  for (int a = 1; a < argc; ++a) {
    Net<float> net(argv[a], TEST);
    const int r = net.last_reader("data");
    std::printf("last_reader %s\n", r < 0 ? "-" : net.layer_names()[r].c_str());
  }
  return 0;
}
"""

_INPUT = 'layer { name: "input" type: "Input" top: "data" input_param { shape { dim: 1 dim: 64 dim: 8 dim: 8 } } }\n'
_CONV = ('layer { name: "conv" type: "Convolution" bottom: "%s" top: "conv"'
         ' convolution_param { num_output: 64 kernel_size: 3 pad: 1 } }\n')
ALIAS_NETS = {
    "dropout": _INPUT + 'layer { name: "drop" type: "Dropout" bottom: "data" top: "drop" }\n' + _CONV % "drop",
    "concat": _INPUT + 'layer { name: "cat" type: "Concat" bottom: "data" top: "cat" }\n' + _CONV % "cat",
}


def deploy_nets(d: Path) -> dict[str, Path]:
    """The shipped deploy nets, extracted under d, by dataset/model."""
    with tarfile.open(ROOT / "tests" / "golden" / "deploy.tar.xz") as t:
        t.extractall(d, filter="data")
    nets = {str(f.parent.relative_to(d / "deploy")): f for f in sorted((d / "deploy").glob("*/*/mscnn_deploy.prototxt"))}
    assert len(nets) == 23
    return nets


def plan_hashes(rel: str, prototxt: Path) -> dict[str, str]:
    """sha256 of the plan's describe text per case "precision HxW keep"."""
    from mscnn_b200 import net as mnet
    net = mnet.Net(str(prototxt))
    h, w = _net_hw(rel)
    keeps = [()] + ([("conv4_3",)] if "conv4_3" in net.blob_names else [])
    prev = mnet.get_precision()
    out = {}
    try:
        for hh, ww in ((h, w), (h + 1, w + 1)):
            net.reshape_input("data", 8, 3, hh, ww)
            for keep in keeps:
                net.set_activation_reuse(True, keep)
                for mode in ("fp32", "bf16"):
                    mnet.set_precision(mode)
                    text = net.activation_plan()
                    assert text
                    out[f"{mode} {hh}x{ww} {','.join(keep) or '-'}"] = hashlib.sha256(text.encode()).hexdigest()
    finally:
        mnet.set_precision(prev)
    return out


def last_readers(d: Path, prototxts: list[Path]) -> list[str]:
    """Net::last_reader("data") of each net, by layer name ("-": none), from a host built against the mirror."""
    from mscnn_b200 import capi
    capi.lib()                                      # raises if the library has not been built
    (d / "probe.cpp").write_text(PROBE)
    exe = d / "probe"
    cmd = ["g++", "-std=c++17", "-O1", "-I", str(ROOT / "include"), "-I", str(ROOT / "mscnn_b200/csrc/caffe_api"),
           "-I", str(ROOT / "mscnn_b200/csrc/proto_shared"), "-I", "/usr/local/cuda/include", str(d / "probe.cpp"),
           "-L", str(ROOT / "mscnn_b200"), "-lmscnn_b200", f"-Wl,-rpath,{ROOT / 'mscnn_b200'}", "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([str(exe), *map(str, prototxts)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [l.split(" ", 1)[1] for l in r.stdout.splitlines() if l.startswith("last_reader ")]
    assert len(lines) == len(prototxts)
    return lines


# printed by make_layer_accesses_pins.py: per net, the plan's sha256 per case, and its input's last reader
PLANS = {
    'caltech/mscnn-7s-480': {
        'fp32 720x960 -': '52f3063e418f284529237343701fcf7c3e262c1887a61175df4915ea5e952ab1',
        'bf16 720x960 -': 'd51ddfbd133c9e4affc4f26ca8547fb452e996ffe9eaea039be858c62aec7065',
        'fp32 720x960 conv4_3': '605e1a4a1943d23db0314681155029670c39a0d568c7d3ff993b2a0d9d28097b',
        'bf16 720x960 conv4_3': 'bd95bd4e2f38acb8820326d1e195eb4919e10316b9726c7683012ccf10c0308a',
        'fp32 721x961 -': 'db1e5981db8652458cf9679ca811ebe45e995ab890210ee4541adc65918eb7b5',
        'bf16 721x961 -': '6550761c9b78fab171424c1d5346a5b5fcdf781207a885471413981a19b31a8e',
        'fp32 721x961 conv4_3': '08ab9e6ae3429e1c66d975cc7e05bfb1d6c07ba94a570cb642039827f1005750',
        'bf16 721x961 conv4_3': '1ad1e024bbee4dc929134a40b2d884444cd2b5547ce0d374e31d585412fb2fdc',
    },
    'caltech/mscnn-7s-480-2x': {
        'fp32 720x960 -': '7ec6c34702dae8984b2e93b616879acab1f1e3e3353a04531f274a9b422314e0',
        'bf16 720x960 -': '99e597198e74917280170da393c10419fb6ee3eefa16ce198b9dc5cb41cbfae2',
        'fp32 720x960 conv4_3': '705291edd366dd08fedbb7a2a1aec8b07f8841fef415347d9c35f84f958eef54',
        'bf16 720x960 conv4_3': '08c8e95f2bec72548f626035fee2d9a56251d2541b8fec723391fd15652b5f96',
        'fp32 721x961 -': 'd4592ccbb742658ea2bfe0307765cfdfca70a86b45b6048ef5b3380ada82f221',
        'bf16 721x961 -': 'cf1ed65b0f10172a9081e4c4314529472d95219a70399976d996018d385454d1',
        'fp32 721x961 conv4_3': 'cf30a2aaa62388c7b809b8f3d8961471e77009b5fd9f7682a10ff96da6a2bab8',
        'bf16 721x961 conv4_3': '6b017b6324591fab81b841984c966e5c8b754e10fa17ade3098d9023788f4eae',
    },
    'caltech/mscnn-7s-720': {
        'fp32 720x960 -': '52f3063e418f284529237343701fcf7c3e262c1887a61175df4915ea5e952ab1',
        'bf16 720x960 -': 'd51ddfbd133c9e4affc4f26ca8547fb452e996ffe9eaea039be858c62aec7065',
        'fp32 720x960 conv4_3': '605e1a4a1943d23db0314681155029670c39a0d568c7d3ff993b2a0d9d28097b',
        'bf16 720x960 conv4_3': 'bd95bd4e2f38acb8820326d1e195eb4919e10316b9726c7683012ccf10c0308a',
        'fp32 721x961 -': 'db1e5981db8652458cf9679ca811ebe45e995ab890210ee4541adc65918eb7b5',
        'bf16 721x961 -': '6550761c9b78fab171424c1d5346a5b5fcdf781207a885471413981a19b31a8e',
        'fp32 721x961 conv4_3': '08ab9e6ae3429e1c66d975cc7e05bfb1d6c07ba94a570cb642039827f1005750',
        'bf16 721x961 conv4_3': '1ad1e024bbee4dc929134a40b2d884444cd2b5547ce0d374e31d585412fb2fdc',
    },
    'citypersons/cascade-mscnn-8s-1344-2x': {
        'fp32 1344x2688 -': '89d6302d42e19f9e5f112f9643e65b95d8ce818b8ec8f1a581c017e8cdc7e883',
        'bf16 1344x2688 -': '56bb207f14a1555db449f09b74ed0ddcd6fd1cd4de034a7ed4eecd1038433832',
        'fp32 1344x2688 conv4_3': '8e24d8d1f9a0d5c1df84b74ee094807e31af300f29af949ed98c64a110f090c4',
        'bf16 1344x2688 conv4_3': '02c291e834ef20f1917ab73cf60b44caf25841eac146851ae6130415e9cecfb8',
        'fp32 1345x2689 -': 'c391b180a5c4809ade417fb288c41bc572f86f1574fa863bc9036f261cf7c9dd',
        'bf16 1345x2689 -': 'a3d2f4ae5e4f6c14e1c7c0427ed567292c3164d6ac503c6a2353c6d352b4baaf',
        'fp32 1345x2689 conv4_3': 'ceaddf429b0515f42450c48fee2ef9d0de9a078c6217dcff918ec82c7119425a',
        'bf16 1345x2689 conv4_3': '904d2dbdc5ee65afa6f8b76568ce204fb99f1a82717cced74409608e964c4966',
    },
    'citypersons/mscnn-8s-1344-2x': {
        'fp32 1344x2688 -': 'a92d319a4d43cd57157800310d3c4250b66f55a298d96e4822fc9ee3ac79c933',
        'bf16 1344x2688 -': '5e249bd71e47691b9a0f45d192b614423f179022c5252ee093be9b5a0baaee9a',
        'fp32 1344x2688 conv4_3': '6c1bf387f7d91d2011d488fb4aca429a8361c37f9cfbab38cc85e697e875099c',
        'bf16 1344x2688 conv4_3': '441092d9b8696097238e3f9b5d207427dc7aef0d7a7ea6c5fb0b399f566a2dcb',
        'fp32 1345x2689 -': '6c4550a4b16ffdb65e51c31a9b335fa1c1e744ee2dc709138be03ce19e2d9a10',
        'bf16 1345x2689 -': 'c835e474a3190f1d6d03ccbf8157914edc23214752f9abfacee78e71c415f47a',
        'fp32 1345x2689 conv4_3': '2b10fba904958ad778529278f1f8ca7aee7df7ed6c5e6af887abec110f5b5ccf',
        'bf16 1345x2689 conv4_3': '8964a1fdbdeb11d0c3000b96dcf8e9faf245ae1d037d63cc2aea1f1d0d362c8c',
    },
    'citypersons/mscnn-8s-1344-2x-trainval': {
        'fp32 1344x2688 -': 'a92d319a4d43cd57157800310d3c4250b66f55a298d96e4822fc9ee3ac79c933',
        'bf16 1344x2688 -': '5e249bd71e47691b9a0f45d192b614423f179022c5252ee093be9b5a0baaee9a',
        'fp32 1344x2688 conv4_3': '6c1bf387f7d91d2011d488fb4aca429a8361c37f9cfbab38cc85e697e875099c',
        'bf16 1344x2688 conv4_3': '441092d9b8696097238e3f9b5d207427dc7aef0d7a7ea6c5fb0b399f566a2dcb',
        'fp32 1345x2689 -': '6c4550a4b16ffdb65e51c31a9b335fa1c1e744ee2dc709138be03ce19e2d9a10',
        'bf16 1345x2689 -': 'c835e474a3190f1d6d03ccbf8157914edc23214752f9abfacee78e71c415f47a',
        'fp32 1345x2689 conv4_3': '2b10fba904958ad778529278f1f8ca7aee7df7ed6c5e6af887abec110f5b5ccf',
        'bf16 1345x2689 conv4_3': '8964a1fdbdeb11d0c3000b96dcf8e9faf245ae1d037d63cc2aea1f1d0d362c8c',
    },
    'kitti_car/cascade-mscnn-7s-576-2x': {
        'fp32 576x1920 -': '7c5fdcd948914a8541a313c0acbdd4cf9e62aed425b600016876efb4dd930eb3',
        'bf16 576x1920 -': 'abb6f24c225da055f95a7231abd4448704a5a31e7a1f5b608b52ce4698487050',
        'fp32 576x1920 conv4_3': 'acaac35994cb345a604aa5e0ed8ac15a0cd2709951bda8e296a53c091ced43c1',
        'bf16 576x1920 conv4_3': 'b74c1d8919009afc5741917ce1c8a8faabf9d573ec8ab3f36ab276e69a20bfba',
        'fp32 577x1921 -': 'ce52dc37bbab1808b205f8ef66f9f6db2d56b51deae927c0ddb918605b2824ce',
        'bf16 577x1921 -': '6faaee3801c2b6fbf422ce27e0d2d86374cd52a26a462aa0fac5aaa612ac6538',
        'fp32 577x1921 conv4_3': 'e40b7f13037182e2d98c8aa5045354685027ace944dfd9dc36c2140fe962ca6e',
        'bf16 577x1921 conv4_3': '097a890ff6ab18a1b271c046d97ea75092f5d655f414af33c9b92cf0a51d467a',
    },
    'kitti_car/cascade-mscnn-7s-576-2x-trainval': {
        'fp32 576x1920 -': '7c5fdcd948914a8541a313c0acbdd4cf9e62aed425b600016876efb4dd930eb3',
        'bf16 576x1920 -': 'abb6f24c225da055f95a7231abd4448704a5a31e7a1f5b608b52ce4698487050',
        'fp32 576x1920 conv4_3': 'acaac35994cb345a604aa5e0ed8ac15a0cd2709951bda8e296a53c091ced43c1',
        'bf16 576x1920 conv4_3': 'b74c1d8919009afc5741917ce1c8a8faabf9d573ec8ab3f36ab276e69a20bfba',
        'fp32 577x1921 -': 'ce52dc37bbab1808b205f8ef66f9f6db2d56b51deae927c0ddb918605b2824ce',
        'bf16 577x1921 -': '6faaee3801c2b6fbf422ce27e0d2d86374cd52a26a462aa0fac5aaa612ac6538',
        'fp32 577x1921 conv4_3': 'e40b7f13037182e2d98c8aa5045354685027ace944dfd9dc36c2140fe962ca6e',
        'bf16 577x1921 conv4_3': '097a890ff6ab18a1b271c046d97ea75092f5d655f414af33c9b92cf0a51d467a',
    },
    'kitti_car/mscnn-7s-384': {
        'fp32 768x2560 -': 'ad1ea99fb326081ddd20fb2a798a7aa406a3018a91ea7e5dc20adc5899394463',
        'bf16 768x2560 -': 'cafe42c706ab994bcdd56bccb71df8ae6661afd5f2d01736ac41048a754caea6',
        'fp32 768x2560 conv4_3': '28b0c2a8252c2c95fbfc3703408b26cd936a09a5128433988eaa2b5f0de16760',
        'bf16 768x2560 conv4_3': '76b8f7bca3c1201295a22161c2e51b13625c4ea6d7f7a7e6a91ffff7dc0873af',
        'fp32 769x2561 -': '9b25d0d773afb39eb75304079dcc3b75240d884123941f9b8a3957c45edcdb43',
        'bf16 769x2561 -': '434f883d65abc6f0e487a917d633aae92645d99dd2de28a321aa8bbe9534611d',
        'fp32 769x2561 conv4_3': '62343acc7189136110d99c08ec3237d8f121807407d7d8f282322a7761b20efb',
        'bf16 769x2561 conv4_3': 'c14169f2833c4160d5f0bd256ab547331f04401dffdb6a98e686769fb902ef0b',
    },
    'kitti_car/mscnn-7s-384-2x': {
        'fp32 768x2560 -': 'd4231f013d989f39002d8e87fcdbdab60ad8c273f200f0fa0661232d420c73bc',
        'bf16 768x2560 -': 'e3cbd3063158150fb9b0deee759130c4b078fe07924a5e2b3d779f92db3405d3',
        'fp32 768x2560 conv4_3': 'be18532efe4cf4767cf4c7ad3ffafbddc5413884a27af0932a69529475a9dea0',
        'bf16 768x2560 conv4_3': 'aea32a7afe40ee0a4136df99240123fe3194f797303a178a3cb5c7c483c97598',
        'fp32 769x2561 -': 'c9e4bcfef7a5e92fb20dac0cab24203a65cc4166ef3a03d63fea3bfb06ff042d',
        'bf16 769x2561 -': '8c845d5e243e72c071cb82ec31d6ae85e01dfcc383d2c1fd3fb4fec1c04305e6',
        'fp32 769x2561 conv4_3': 'ba96ad93f4b68b6cb449dc7e565e86f07fa284c68ea14482a82058c29b3541df',
        'bf16 769x2561 conv4_3': 'f1ab718e27a2a98aa871bef3ae160379b254f44237cad27c546c89476c60e04a',
    },
    'kitti_car/mscnn-7s-576': {
        'fp32 768x2560 -': 'ad1ea99fb326081ddd20fb2a798a7aa406a3018a91ea7e5dc20adc5899394463',
        'bf16 768x2560 -': 'cafe42c706ab994bcdd56bccb71df8ae6661afd5f2d01736ac41048a754caea6',
        'fp32 768x2560 conv4_3': '28b0c2a8252c2c95fbfc3703408b26cd936a09a5128433988eaa2b5f0de16760',
        'bf16 768x2560 conv4_3': '76b8f7bca3c1201295a22161c2e51b13625c4ea6d7f7a7e6a91ffff7dc0873af',
        'fp32 769x2561 -': '9b25d0d773afb39eb75304079dcc3b75240d884123941f9b8a3957c45edcdb43',
        'bf16 769x2561 -': '434f883d65abc6f0e487a917d633aae92645d99dd2de28a321aa8bbe9534611d',
        'fp32 769x2561 conv4_3': '62343acc7189136110d99c08ec3237d8f121807407d7d8f282322a7761b20efb',
        'bf16 769x2561 conv4_3': 'c14169f2833c4160d5f0bd256ab547331f04401dffdb6a98e686769fb902ef0b',
    },
    'kitti_car/mscnn-7s-576-2x': {
        'fp32 768x2560 -': 'd4231f013d989f39002d8e87fcdbdab60ad8c273f200f0fa0661232d420c73bc',
        'bf16 768x2560 -': 'e3cbd3063158150fb9b0deee759130c4b078fe07924a5e2b3d779f92db3405d3',
        'fp32 768x2560 conv4_3': 'be18532efe4cf4767cf4c7ad3ffafbddc5413884a27af0932a69529475a9dea0',
        'bf16 768x2560 conv4_3': 'aea32a7afe40ee0a4136df99240123fe3194f797303a178a3cb5c7c483c97598',
        'fp32 769x2561 -': 'c9e4bcfef7a5e92fb20dac0cab24203a65cc4166ef3a03d63fea3bfb06ff042d',
        'bf16 769x2561 -': '8c845d5e243e72c071cb82ec31d6ae85e01dfcc383d2c1fd3fb4fec1c04305e6',
        'fp32 769x2561 conv4_3': 'ba96ad93f4b68b6cb449dc7e565e86f07fa284c68ea14482a82058c29b3541df',
        'bf16 769x2561 conv4_3': 'f1ab718e27a2a98aa871bef3ae160379b254f44237cad27c546c89476c60e04a',
    },
    'kitti_car/mscnn-7s-576-2x-trainval': {
        'fp32 768x2560 -': 'd4231f013d989f39002d8e87fcdbdab60ad8c273f200f0fa0661232d420c73bc',
        'bf16 768x2560 -': 'e3cbd3063158150fb9b0deee759130c4b078fe07924a5e2b3d779f92db3405d3',
        'fp32 768x2560 conv4_3': 'be18532efe4cf4767cf4c7ad3ffafbddc5413884a27af0932a69529475a9dea0',
        'bf16 768x2560 conv4_3': 'aea32a7afe40ee0a4136df99240123fe3194f797303a178a3cb5c7c483c97598',
        'fp32 769x2561 -': 'c9e4bcfef7a5e92fb20dac0cab24203a65cc4166ef3a03d63fea3bfb06ff042d',
        'bf16 769x2561 -': '8c845d5e243e72c071cb82ec31d6ae85e01dfcc383d2c1fd3fb4fec1c04305e6',
        'fp32 769x2561 conv4_3': 'ba96ad93f4b68b6cb449dc7e565e86f07fa284c68ea14482a82058c29b3541df',
        'bf16 769x2561 conv4_3': 'f1ab718e27a2a98aa871bef3ae160379b254f44237cad27c546c89476c60e04a',
    },
    'kitti_car/mscnn-8s-768-trainval': {
        'fp32 768x2560 -': 'a5fc6f4fc0c21cd1719175f5b1376c50bce89ce2fdc4e8c14c50080693857f6c',
        'bf16 768x2560 -': '466b4bccdfea52f19ab3795a887cfbdba3d7cc8751a104d34c9cabc6db5266a1',
        'fp32 768x2560 conv4_3': 'de7160ba89193cc62087b9d17c70401ee6c691eecc47a14f88ea11a84ff485fd',
        'bf16 768x2560 conv4_3': '0ac69cee693b6d04a5f2e8e42540cba0a16c1bf558a48e37f992ce870f702ad0',
        'fp32 769x2561 -': '0f2e71033912a7f63f0ba09534d748385a295f0d15f955c51f7ae8a65def3265',
        'bf16 769x2561 -': '17a5dfe2d4620db6a1e64108d5d084bdb0165af9c0993d529a72cc29a5e5cc7f',
        'fp32 769x2561 conv4_3': 'bf0e006bdad91b843be1f7a12da186448d7048da4ff4625ff6642ca01c2ccd9c',
        'bf16 769x2561 conv4_3': 'c08b2cc0b2cf96b324970a6f98550d8139ae067216e2c95131f6614a5033c6cb',
    },
    'kitti_ped_cyc/mscnn-7s-384': {
        'fp32 768x2560 -': '737e9b1adfa4728f53b8e9e02f88b262fdcc40ce25c0235f809878149bba5eab',
        'bf16 768x2560 -': '9fb3e1af15f78b7ebb876b0cb8fda71b7bd78120fdd6637712146f1d1d7659c9',
        'fp32 768x2560 conv4_3': '6ded3db6bd8794417502737213b9b29f2bd35a55cb095218d0bfe0a757417a32',
        'bf16 768x2560 conv4_3': 'ec830867f099575bf1d3956a88a38f5cedcc7c140a127bb9142b973aecba2a4f',
        'fp32 769x2561 -': 'd6170f9a4c7865690fc9d0926121ab37684c1a88dfe7074d2250d4ec2fc5d0a5',
        'bf16 769x2561 -': '9fd0bf9e6dd96704eeba4853d09e933d1f5409ae135081fc31dfcedf16645424',
        'fp32 769x2561 conv4_3': '84ca5bdf9982298edbc58ccf837b302626a8d9d253002465e5a4d657cb2f8e59',
        'bf16 769x2561 conv4_3': 'c18e2d3269e5cc25a6773453fdce09f912613ca637029c3feac234d174f36a3e',
    },
    'kitti_ped_cyc/mscnn-7s-384-2x': {
        'fp32 768x2560 -': '0bc9db13bbd08d552d77e434dd9ee1cefd94b1ea22b1b148c3859ddf3e6bdfb5',
        'bf16 768x2560 -': '264dd4e95dffe31d25182ed84d6dda98aa90e5ea4ec78fea2f1827bf6bcb91b0',
        'fp32 768x2560 conv4_3': 'b683c6739248c71909aeb68f1f1b9c071c79455ee5bba56eb0859803cb60ede0',
        'bf16 768x2560 conv4_3': '15456895619932bb844c7e14a952d78cd07c59cbef6c1653791091d8be3fc3af',
        'fp32 769x2561 -': '2f87a6a5c0e17f355cd688c16b79a9e7d182cb5f4860c8bd827c3b8aadf830a9',
        'bf16 769x2561 -': 'dedd556dd01284a12def50cd9a265e4593cf229a5bf96dd3b54436ad1d0bba60',
        'fp32 769x2561 conv4_3': '587880d23bbe0fd7a8d4df3d3a532e79698a32888f808a73a6088c1cf71b13d4',
        'bf16 769x2561 conv4_3': '61b2a1fe7662112dcccfd9815e956c5dfda27506402bbd5285fd3d3d890abbc2',
    },
    'kitti_ped_cyc/mscnn-7s-576': {
        'fp32 768x2560 -': '737e9b1adfa4728f53b8e9e02f88b262fdcc40ce25c0235f809878149bba5eab',
        'bf16 768x2560 -': '9fb3e1af15f78b7ebb876b0cb8fda71b7bd78120fdd6637712146f1d1d7659c9',
        'fp32 768x2560 conv4_3': '6ded3db6bd8794417502737213b9b29f2bd35a55cb095218d0bfe0a757417a32',
        'bf16 768x2560 conv4_3': 'ec830867f099575bf1d3956a88a38f5cedcc7c140a127bb9142b973aecba2a4f',
        'fp32 769x2561 -': 'd6170f9a4c7865690fc9d0926121ab37684c1a88dfe7074d2250d4ec2fc5d0a5',
        'bf16 769x2561 -': '9fd0bf9e6dd96704eeba4853d09e933d1f5409ae135081fc31dfcedf16645424',
        'fp32 769x2561 conv4_3': '84ca5bdf9982298edbc58ccf837b302626a8d9d253002465e5a4d657cb2f8e59',
        'bf16 769x2561 conv4_3': 'c18e2d3269e5cc25a6773453fdce09f912613ca637029c3feac234d174f36a3e',
    },
    'kitti_ped_cyc/mscnn-7s-576-2x': {
        'fp32 768x2560 -': '0bc9db13bbd08d552d77e434dd9ee1cefd94b1ea22b1b148c3859ddf3e6bdfb5',
        'bf16 768x2560 -': '264dd4e95dffe31d25182ed84d6dda98aa90e5ea4ec78fea2f1827bf6bcb91b0',
        'fp32 768x2560 conv4_3': 'b683c6739248c71909aeb68f1f1b9c071c79455ee5bba56eb0859803cb60ede0',
        'bf16 768x2560 conv4_3': '15456895619932bb844c7e14a952d78cd07c59cbef6c1653791091d8be3fc3af',
        'fp32 769x2561 -': '2f87a6a5c0e17f355cd688c16b79a9e7d182cb5f4860c8bd827c3b8aadf830a9',
        'bf16 769x2561 -': 'dedd556dd01284a12def50cd9a265e4593cf229a5bf96dd3b54436ad1d0bba60',
        'fp32 769x2561 conv4_3': '587880d23bbe0fd7a8d4df3d3a532e79698a32888f808a73a6088c1cf71b13d4',
        'bf16 769x2561 conv4_3': '61b2a1fe7662112dcccfd9815e956c5dfda27506402bbd5285fd3d3d890abbc2',
    },
    'kitti_ped_cyc/mscnn-7s-576-2x-trainval': {
        'fp32 768x2560 -': '0bc9db13bbd08d552d77e434dd9ee1cefd94b1ea22b1b148c3859ddf3e6bdfb5',
        'bf16 768x2560 -': '264dd4e95dffe31d25182ed84d6dda98aa90e5ea4ec78fea2f1827bf6bcb91b0',
        'fp32 768x2560 conv4_3': 'b683c6739248c71909aeb68f1f1b9c071c79455ee5bba56eb0859803cb60ede0',
        'bf16 768x2560 conv4_3': '15456895619932bb844c7e14a952d78cd07c59cbef6c1653791091d8be3fc3af',
        'fp32 769x2561 -': '2f87a6a5c0e17f355cd688c16b79a9e7d182cb5f4860c8bd827c3b8aadf830a9',
        'bf16 769x2561 -': 'dedd556dd01284a12def50cd9a265e4593cf229a5bf96dd3b54436ad1d0bba60',
        'fp32 769x2561 conv4_3': '587880d23bbe0fd7a8d4df3d3a532e79698a32888f808a73a6088c1cf71b13d4',
        'bf16 769x2561 conv4_3': '61b2a1fe7662112dcccfd9815e956c5dfda27506402bbd5285fd3d3d890abbc2',
    },
    'kitti_ped_cyc/mscnn-8s-768-trainval': {
        'fp32 768x2560 -': '1bee3d98be8b8bb1446ae762f1933d7840879d2f888f02a950b992f26391cfd7',
        'bf16 768x2560 -': '0655fee048e7265a69423757e36b011b20da00501c033d0182202e8af237368d',
        'fp32 768x2560 conv4_3': 'e3931ff385ba502301f7590a87050519249ae9335a9d63445cfb4006f642f7d8',
        'bf16 768x2560 conv4_3': '1d12ecf07731a60f942fede175649b4b7d4cf72a23077ab2e10e1993279c3590',
        'fp32 769x2561 -': '344d56d74b8ce521b963ce134b1364ed1e476e2eee7085c7b08643943078f917',
        'bf16 769x2561 -': '4987d9b3c9c7d475826aad2bd98571f8290f7d7c7118d353eadb616dc86ec1c0',
        'fp32 769x2561 conv4_3': '666103edcd474d90f6dbb332d54cc6ebc183a7c8cf8df55aa60b0f17e64042f6',
        'bf16 769x2561 conv4_3': '0b52e86eccf313d8f1420f261651452b8b1a3862fbb214bd317d85c7d2c1fb97',
    },
    'widerface/cascade-mscnn-12s-align': {
        'fp32 1024x768 -': '86c9c1fd005ecb4906aa5985cc520404cdb921e14c553ac3d9d1b211d39e1024',
        'bf16 1024x768 -': '21d3cd898f77757c961a772866c045e5b7ef4b0e618d1575886ee36096ae5656',
        'fp32 1024x768 conv4_3': 'e351688cbc71017f6e37f74208b6d40727788cddb801b45a6c95929bada40db3',
        'bf16 1024x768 conv4_3': 'ab437417b7d10c694c206be0df4d60677e059baf9c3ea5b9baf5e9324f32c8d3',
        'fp32 1025x769 -': 'bcae35a20f6de3da7e9ddd35d5de512d8a19ffcf05f16b921d9404da777c7410',
        'bf16 1025x769 -': '452933268764c5dd294c86e884031723a85c5f918f5111a00bab05a77516273f',
        'fp32 1025x769 conv4_3': '2a567f0d5e5e2ef81655edf32ab4a30b4fa544ef882aaf1364b52f3ddfbcca25',
        'bf16 1025x769 conv4_3': 'c9236cfbd681d1fc4071944725d9a8c5986d8371031bbde1126f06bdd0c2b554',
    },
    'widerface/mscnn-12s-2x': {
        'fp32 1024x768 -': '837206f338fc282c777184eebdfbb694f2e50665b9b2f15ae221f0908fff50ed',
        'bf16 1024x768 -': 'f7d00f178ec4a6bee14be862a3d0949c43570cc1e6ae0ab13c666de9c58ac135',
        'fp32 1024x768 conv4_3': 'e999980be345e6bd925b1846f9f47b30ad64ead6fd387e6eb61e03d83a5f5d04',
        'bf16 1024x768 conv4_3': '02f344783281b2aac9c4faab7b1c092c7cd42d45f515a58bc9039082f5073cc1',
        'fp32 1025x769 -': '0a70d396286834de8a779d1bbb2b7b60f73e731494b6c8afd2fc4afc15496fa1',
        'bf16 1025x769 -': 'e5d4fe4a651d8024a342e4a48ee80778992cc5600dfc18109d1f012fdbd4b980',
        'fp32 1025x769 conv4_3': '3ecc5e4b53b8425c804994bc1b4033d5f803d6f0f13b9970a14de99a2c566ba9',
        'bf16 1025x769 conv4_3': 'd28e94683dfc6eaf3495dd37fb7c4fa2b2d0f9c31be2e13f3581c4f1ca393639',
    },
    'widerface/mscnn-12s-2x-trainval': {
        'fp32 1024x768 -': '837206f338fc282c777184eebdfbb694f2e50665b9b2f15ae221f0908fff50ed',
        'bf16 1024x768 -': 'f7d00f178ec4a6bee14be862a3d0949c43570cc1e6ae0ab13c666de9c58ac135',
        'fp32 1024x768 conv4_3': 'e999980be345e6bd925b1846f9f47b30ad64ead6fd387e6eb61e03d83a5f5d04',
        'bf16 1024x768 conv4_3': '02f344783281b2aac9c4faab7b1c092c7cd42d45f515a58bc9039082f5073cc1',
        'fp32 1025x769 -': '0a70d396286834de8a779d1bbb2b7b60f73e731494b6c8afd2fc4afc15496fa1',
        'bf16 1025x769 -': 'e5d4fe4a651d8024a342e4a48ee80778992cc5600dfc18109d1f012fdbd4b980',
        'fp32 1025x769 conv4_3': '3ecc5e4b53b8425c804994bc1b4033d5f803d6f0f13b9970a14de99a2c566ba9',
        'bf16 1025x769 conv4_3': 'd28e94683dfc6eaf3495dd37fb7c4fa2b2d0f9c31be2e13f3581c4f1ca393639',
    },
}
LAST_READER = {
    'caltech/mscnn-7s-480': 'conv1_1',
    'caltech/mscnn-7s-480-2x': 'conv1_1',
    'caltech/mscnn-7s-720': 'conv1_1',
    'citypersons/cascade-mscnn-8s-1344-2x': 'conv1_1',
    'citypersons/mscnn-8s-1344-2x': 'conv1_1',
    'citypersons/mscnn-8s-1344-2x-trainval': 'conv1_1',
    'kitti_car/cascade-mscnn-7s-576-2x': 'conv1_1',
    'kitti_car/cascade-mscnn-7s-576-2x-trainval': 'conv1_1',
    'kitti_car/mscnn-7s-384': 'conv1_1',
    'kitti_car/mscnn-7s-384-2x': 'conv1_1',
    'kitti_car/mscnn-7s-576': 'conv1_1',
    'kitti_car/mscnn-7s-576-2x': 'conv1_1',
    'kitti_car/mscnn-7s-576-2x-trainval': 'conv1_1',
    'kitti_car/mscnn-8s-768-trainval': 'conv1_1',
    'kitti_ped_cyc/mscnn-7s-384': 'conv1_1',
    'kitti_ped_cyc/mscnn-7s-384-2x': 'conv1_1',
    'kitti_ped_cyc/mscnn-7s-576': 'conv1_1',
    'kitti_ped_cyc/mscnn-7s-576-2x': 'conv1_1',
    'kitti_ped_cyc/mscnn-7s-576-2x-trainval': 'conv1_1',
    'kitti_ped_cyc/mscnn-8s-768-trainval': 'conv1_1',
    'widerface/cascade-mscnn-12s-align': 'conv1_1',
    'widerface/mscnn-12s-2x': 'conv1_1',
    'widerface/mscnn-12s-2x-trainval': 'conv1_1',
}


@pytest.fixture(scope="module")
def nets(tmp_path_factory):
    return deploy_nets(tmp_path_factory.mktemp("deploy"))


def test_every_net_is_pinned(nets):
    assert sorted(nets) == sorted(PLANS) == sorted(LAST_READER)


@pytest.mark.parametrize("rel", sorted(PLANS))
def test_activation_plan_is_pinned(nets, rel):
    assert plan_hashes(rel, nets[rel]) == PLANS[rel]


def test_last_reader_of_the_input_is_pinned(nets, tmp_path):
    rels = sorted(nets)
    assert dict(zip(rels, last_readers(tmp_path, [nets[r] for r in rels]))) == LAST_READER


def test_last_reader_follows_a_shared_top(tmp_path):
    files = []
    for name, text in ALIAS_NETS.items():
        files.append(tmp_path / f"{name}.prototxt")
        files[-1].write_text(f'name: "{name}"\n' + text)
    assert last_readers(tmp_path, files) == ["conv"] * len(files)

