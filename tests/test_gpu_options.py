"""The option registry of each matcher type: every registered name is accepted, PrintOptions lists
exactly that type's names with the values that were set, and any other name is a CheckFailure."""
import numpy as np
import pytest

import staticmapping_b200 as smb

pytestmark = pytest.mark.gpu

# name -> (text to set, kind, expected value); kinds follow the engine's tables
ICP = {
    "knn_normal_estimate": ("9", "int", 9),
    "max_iteration": ("42", "int", 42),
    "dist_outlier_ratio": ("0.65", "float", 0.65),
    "knn_epsilon": ("2.5", "float", 2.5),
    "disable_convergence_check": ("true", "bool", True),
    "profile_kernels": (" 1", "bool", True),
    "use_graphs": ("no", "bool", False),
    "knn_queries_per_cta": ("64", "int", 64),
    "reading_sample_prob": ("0.8", "float", 0.8),
    "accept_min_score": ("0.55", "float", 0.55),
    "sample_seed": ("7", "int", 7),
}
NDT = {
    "max_iterations": ("20", "int", 20),
    "resolution": ("1.5", "float", 1.5),
    "step_size": ("0.05", "double", 0.05),
    "outlier_ratio": ("0.4", "double", 0.4),
    "transformation_epsilon": ("0.001", "double", 0.001),
}
NDT_GICP = {
    "use_ndt": ("false", "bool", False),
    "using_voxel_filter": ("0", "bool", False),
    "voxel_resolution": ("0.3", "float", 0.3),
}


def _set_xml(m, opts):
    m.InitWithXml("<registrator_options>" + "".join(
        f'<param name="{k}">{v}</param>' for k, v in opts.items()) + "</registrator_options>")


def _set_engine(m, opts):
    # Ndt and the IcpUsingPointMatcher stand-in register no XML option (InitWithXml raises for any
    # name, as the reference does); their engine options go through the same registry
    m.SetEngineOptions(**opts)


@pytest.mark.parametrize("cls,table,setter,foreign", [
    (smb.IcpFast, ICP, _set_xml, "max_iterations"),
    (smb.IcpUsingPointMatcher, ICP, _set_engine, "voxel_resolution"),
    (smb.Ndt, NDT, _set_engine, "max_iteration"),
    (smb.NdtWithGicp, NDT_GICP, _set_xml, "max_iteration"),
], ids=["IcpFast", "IcpUsingPointMatcher", "Ndt", "NdtWithGicp"])
def test_option_registry_per_type(cls, table, setter, foreign):
    m = cls()
    setter(m, {k: text for k, (text, _, _) in table.items()})
    printed = {}
    names = []
    for line in m.PrintOptions().splitlines():
        name, value = line.split(" -> ")
        names.append(name.strip())
        printed[name.strip()] = value
    assert names == list(table)
    for name, (_, kind, want) in table.items():
        got = printed[name]
        if kind == "int":
            assert int(got) == want, name
        elif kind == "float":
            assert np.float32(got) == np.float32(want), name
        elif kind == "double":
            assert float(got) == want, name
        else:
            assert got == ("true" if want else "false"), name
    for bad in ("bogus", foreign):
        with pytest.raises(smb.CheckFailure):
            setter(m, {bad: "1"})
