"""The fusion pass's decisions on every shipped deploy net and on the generated nets: which layer does a folded layer's
work (Net::fused_producer: a Pooling -> its convolution, a ROIPooling -> the leader of its Concat group), which in-place
ReLUs fold into their producer and which Concats their ROIPooling producers write.  The decisions are made when the net
is built, so they are visible without a GPU.  ReLU and Concat fusion show only through the C++ layer classes, so a small
host written against the Caffe-API mirror prints them, one line per net."""
import os
import subprocess
import tarfile
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent

PROBE = r"""
#include <cstdio>
#include <string>

#include "caffe/caffe.hpp"
#include "caffe/layers/mscnn_layers.hpp"

using namespace caffe;

int main(int argc, char** argv) {
  Caffe::set_mode(Caffe::GPU);
  for (int a = 1; a < argc; ++a) {
    Net<float> net(argv[a], TEST);
    std::string folded, relus, concats;
    int conv_relus = 0;
    for (size_t i = 0; i < net.layers().size(); ++i) {
      Layer<float>* l = net.layers()[i].get();
      const std::string name = net.layer_names()[i], type = l->type();
      const int p = net.fused_producer((int)i);
      if (p != (int)i) folded += " " + name + "<-" + net.layer_names()[p];
      if (type == "ReLU" && static_cast<ReLULayer<float>*>(l)->fused()) relus += " " + name;
      if (type == "Concat" && static_cast<ConcatLayer<float>*>(l)->fused()) concats += " " + name;
      if (type == "Convolution" && static_cast<ConvolutionLayer<float>*>(l)->fuse_relu()) ++conv_relus;
    }
    std::printf("fusion%s | relu%s | concat%s | conv+relu %d\n", folded.c_str(), relus.c_str(), concats.c_str(),
                conv_relus);
  }
  return 0;
}
"""

GENERATED = {
    "models.kitti_8s": ("kitti", (768, 2560, 8, False)),
    "models.kitti_7s": ("kitti", (576, 1920, 7, False)),
    "models.kitti_7s_2x": ("kitti", (576, 1920, 7, True)),
    "models.kitti_cascade": ("kitti_cascade", (576, 1920)),
    "models.widerface": ("widerface", (512, 512)),
    "models.widerface_cascade": ("widerface_cascade", (512, 512)),
}

# Literals recorded from the fusion pass as it stood when groups were still formed during the forward.
_TRUNK = "pool1<-conv1_2 pool2<-conv2_2 pool3<-conv3_3"
_RELU = "relu relu1_1 relu1_2 relu2_1 relu2_2 relu3_1 relu3_2 relu3_3 relu4_1 relu4_2 relu4_3"
_MSCNN = (f"{_TRUNK} roi_pool_ctx<-roi_pool_org | {_RELU} loss_relu1 relu5_1 relu5_2 relu5_3 relu6_1 roi_c1_relu relu6"
          " | concat roi_pool | conv+relu 16")
_CASCADE_STAGES = "roi_pool_ctx<-roi_pool_org roi_pool_ctx_2nd<-roi_pool_org_2nd roi_pool_ctx_3rd<-roi_pool_org_3rd"
_CASCADE_KITTI = (f"{_TRUNK} {_CASCADE_STAGES} | {_RELU} loss_relu1 relu5_1 relu5_2 relu5_3 relu6_1 roi_c1_relu relu6"
                  " roi_c1_relu_2nd relu6_2nd roi_c1_relu_3rd relu6_3rd | concat roi_pool roi_pool_2nd roi_pool_3rd"
                  " | conv+relu 18")
_CASCADE_CITYPERSONS = (f"{_TRUNK} {_CASCADE_STAGES} | {_RELU} loss_relu1 relu5_1 relu5_2 relu5_3 relu6_1 roi_c1_relu"
                        " relu6 roi_c1_relu_2nd relu6_2nd roi_c1_relu_1st_3rd relu6_1st_3rd roi_c1_relu_2nd_3rd"
                        " relu6_2nd_3rd roi_c1_relu_3rd relu6_3rd | concat roi_pool roi_pool_2nd roi_pool_3rd"
                        " | conv+relu 20")
_WIDER_RELU = f"{_RELU} rpn_1_relu relu5_1 relu5_2 relu5_3 rpn_2_relu rpn_3_relu rpn_4_relu roi_c1_relu relu6"
_WIDER = f"{_TRUNK} roi_pool_ctx<-roi_pool_org | {_WIDER_RELU} | concat roi_pool | conv+relu 18"
# ROIAlign, not ROIPooling: nothing is grouped
_WIDER_CASCADE = (f"{_TRUNK} | {_WIDER_RELU} roi_c1_relu_2nd relu6_2nd roi_c1_relu_1st_3rd relu6_1st_3rd"
                  " roi_c1_relu_2nd_3rd relu6_2nd_3rd roi_c1_relu_3rd relu6_3rd | concat | conv+relu 22")

EXPECTED = {
    **{f"caltech/{m}": _MSCNN for m in ("mscnn-7s-480", "mscnn-7s-480-2x", "mscnn-7s-720")},
    **{f"citypersons/{m}": _MSCNN for m in ("mscnn-8s-1344-2x", "mscnn-8s-1344-2x-trainval")},
    **{f"{d}/{m}": _MSCNN for d in ("kitti_car", "kitti_ped_cyc")
       for m in ("mscnn-7s-384", "mscnn-7s-384-2x", "mscnn-7s-576", "mscnn-7s-576-2x", "mscnn-7s-576-2x-trainval",
                 "mscnn-8s-768-trainval")},
    "models.kitti_7s": _MSCNN,
    "models.kitti_7s_2x": _MSCNN,
    "models.kitti_8s": _MSCNN,
    "citypersons/cascade-mscnn-8s-1344-2x": _CASCADE_CITYPERSONS,
    "kitti_car/cascade-mscnn-7s-576-2x": _CASCADE_KITTI,
    "kitti_car/cascade-mscnn-7s-576-2x-trainval": _CASCADE_KITTI,
    "models.kitti_cascade": _CASCADE_KITTI,
    "widerface/mscnn-12s-2x": _WIDER,
    "widerface/mscnn-12s-2x-trainval": _WIDER,
    "models.widerface": _WIDER,
    "widerface/cascade-mscnn-12s-align": _WIDER_CASCADE,
    "models.widerface_cascade": _WIDER_CASCADE,
}


@pytest.fixture(scope="module")
def fusion(tmp_path_factory):
    from mscnn_b200 import capi, models
    capi.lib()                                      # raises if the library has not been built
    d = tmp_path_factory.mktemp("fusion")
    (d / "probe.cpp").write_text(PROBE)
    exe = d / "probe"
    cmd = ["g++", "-std=c++17", "-O1", "-I", str(ROOT / "include"), "-I", str(ROOT / "mscnn_b200/csrc/caffe_api"),
           "-I", str(ROOT / "mscnn_b200/csrc/proto_shared"), "-I", "/usr/local/cuda/include", str(d / "probe.cpp"),
           "-L", str(ROOT / "mscnn_b200"), "-lmscnn_b200", f"-Wl,-rpath,{ROOT / 'mscnn_b200'}", "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    with tarfile.open(ROOT / "tests" / "golden" / "deploy.tar.xz") as t:
        t.extractall(d, filter="data")
    nets = {str(f.parent.relative_to(d / "deploy")): f for f in sorted((d / "deploy").glob("*/*/mscnn_deploy.prototxt"))}
    assert len(nets) == 23
    for key, (fn, args) in GENERATED.items():
        nets[key] = d / f"{key}.prototxt"
        nets[key].write_text(getattr(models, fn)(*args))
    env = {k: v for k, v in os.environ.items() if k not in ("MSCNN_NO_FUSION", "MSCNN_NO_POOL_FUSION")}
    r = subprocess.run([str(exe), *map(str, nets.values())], capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [l[len("fusion"):].strip() for l in r.stdout.splitlines() if l.startswith("fusion")]
    assert len(lines) == len(nets)
    return dict(zip(nets, lines))


def test_every_net_is_pinned(fusion):
    assert sorted(fusion) == sorted(EXPECTED)


@pytest.mark.parametrize("net", sorted(EXPECTED))
def test_fusion_decisions(fusion, net):
    assert fusion[net] == EXPECTED[net]
