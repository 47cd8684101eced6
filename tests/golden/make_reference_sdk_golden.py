"""Regenerates reference_sdk_models.json from an unmodified checkout of the reference's Python SDK:

    python tests/golden/make_reference_sdk_golden.py <reference>/sdk/python/v2beta1 > tests/golden/reference_sdk_models.json

"v2beta1": openapi_types and attribute_map of the 9 MPIJob models.
"generic": for every other generated model file, its attribute_map, the attributes whose setter rejects None (required
fields) and the module name."""
import importlib
import inspect
import json
import pkgutil
import sys


def main(sdk_dir: str) -> None:
    sys.path.insert(0, sdk_dir)
    import mpijob.models as m
    v2 = {n: [getattr(m, n).openapi_types, getattr(m, n).attribute_map] for n in dir(m) if n.startswith("V2beta1")}
    generic = {}
    for info in pkgutil.iter_modules(m.__path__):  # every generated FILE (the package __init__ lists only half)
        mod = importlib.import_module("mpijob.models." + info.name)
        cs = [c for c in vars(mod).values() if inspect.isclass(c) and c.__module__ == mod.__name__ and hasattr(c, "attribute_map")]
        if len(cs) != 1 or cs[0].__name__.startswith("V2beta1"):
            continue
        c = cs[0]
        req = []
        for a in c.openapi_types:
            try:
                o = c.__new__(c)
                o.local_vars_configuration = type("C", (), {"client_side_validation": True})()
                setattr(o, a, None)
            except ValueError:
                req.append(a)
            except Exception:
                pass
        generic[c.__name__] = [c.attribute_map, sorted(req), c.__module__.rsplit(".", 1)[-1]]
    print(json.dumps({"v2beta1": v2, "generic": generic}, indent=1, sort_keys=True))


if __name__ == "__main__":
    main(sys.argv[1])
