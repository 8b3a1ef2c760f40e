"""Regenerate config/model/*-b200.yaml from the reference's model yamls (run in the build container, where /root/reference exists).

Each output is the reference file with ONLY the model-class `_target_`s swapped for the nabladft_b200 mirrors, so that
`run.py --config-name ... model=<name>-b200` instantiates the same Lightning task / optimizer / scheduler / losses / metrics
around the H100 engine (INTEGRATION.md section 1).  Everything that is not a model class keeps the reference's target.
"""
import os
import sys

REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference/config/model"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "config", "model")

SWAPS = {
    "painn": [("schnetpack.model.NeuralNetworkPotential", "nabladft_b200.spk.NeuralNetworkPotential"),
              ("schnetpack.representation.PaiNN", "nabladft_b200.spk.PaiNN"),
              ("schnetpack.nn.radial.GaussianRBF", "nabladft_b200.spk.GaussianRBF"),
              ("schnetpack.nn.cutoff.CosineCutoff", "nabladft_b200.spk.CosineCutoff"),
              ("schnetpack.atomistic.PairwiseDistances", "nabladft_b200.spk.PairwiseDistances"),
              ("schnetpack.atomistic.Atomwise", "nabladft_b200.spk.Atomwise"),
              ("schnetpack.atomistic.Forces", "nabladft_b200.spk.Forces"),
              ("schnetpack.transform.AddOffsets", "nabladft_b200.spk.AddOffsets")],
    "painn-oc": [("nablaDFT.painn_pyg.PaiNN", "nabladft_b200.painn_oc.PaiNN")],
    "qhnet": [("nablaDFT.qhnet.QHNet", "nabladft_b200.qhnet.QHNet")],
    "gemnet-oc": [("nablaDFT.gemnet_oc.GemNetOC", "nabladft_b200.gemnet_oc.GemNetOC")],
    "dimenetplusplus": [("nablaDFT.dimenetplusplus.DimeNetPlusPlusPotential", "nabladft_b200.dimenetplusplus.DimeNetPlusPlusPotential")],
}
SWAPS["schnet"] = [(a.replace("representation.PaiNN", "representation.SchNet"), b.replace("spk.PaiNN", "spk.SchNet")) for a, b in SWAPS["painn"]]

for name, swaps in SWAPS.items():
    text = open(os.path.join(REF, name + ".yaml")).read()
    for a, b in swaps:
        assert ("_target_: " + a) in text, (name, a)
        text = text.replace("_target_: " + a, "_target_: " + b)
    head = f"# Drop-in for nablaDFT config/model/{name}.yaml: model-class targets swapped for the nabladft_b200 mirrors, rest unchanged (tools/make_b200_yamls.py).\n"
    open(os.path.join(OUT, name + "-b200.yaml"), "w").write(head + text)
    print("wrote", name + "-b200.yaml")
