"""Soil tables beyond the shipped presets, for the tests of tests/test_soil_space*.py: a writer of `.soil` text the
reference's loadsoil (io.h:7-230) and the library's parser both read, a seeded generator of random tables over the
parameter extremes, hand-made "sentinel" tables in which a soil type can reach the map through one mapping only, and
a table of SM_MAX_SOILS (64) soils.

A table is a plain dict: {"name", "scale", "soils": [soil dicts, Air excluded], "layers": [layer dicts],
"declare": bool}.  A soil dict holds "name", the four chain fields as soil names ("transports", "erodes", "cascades",
"abrades") and the float fields of FLOATS; a layer dict holds "soil" (a name) and the fields of LAYER_FLOATS.
Air is never written: both parsers pre-seed it as soil 0 (surface.h:41-57).  With "declare" the file opens with an
empty block per soil in table order, so soil i of the table is soil i + 1 of the parsed file; without it a chain
field that names a soil before its own block allocates that soil's index at the first mention (io.h:125-152)."""
import numpy as np

# file keyword -> table field, in the order they are written
FLOATS = (("DENSITY", "density"), ("POROSITY", "porosity"), ("SOLUBILITY", "solubility"),
          ("EQUILIBRIUM", "equrate"), ("FRICTION", "friction"), ("EROSIONRATE", "erosionrate"),
          ("MAXDIFF", "maxdiff"), ("SETTLING", "settling"), ("SUSPENSION", "suspension"), ("ABRASION", "abrasion"))
CHAINS = (("TRANSPORTS", "transports"), ("ERODES", "erodes"), ("CASCADES", "cascades"), ("ABRADES", "abrades"))
LAYER_FLOATS = (("MIN", "min"), ("BIAS", "bias"), ("SCALE", "scale"), ("OCTAVES", "octaves"),
                ("LACUNARITY", "lacunarity"), ("GAIN", "gain"), ("FREQUENCY", "frequency"))

SOIL_DEFAULTS = {"density": 1.0, "porosity": 0.3, "solubility": 1.0, "equrate": 0.5, "friction": 0.15,
                 "erosionrate": 0.0, "maxdiff": 0.01, "settling": 0.1, "suspension": 0.0, "abrasion": 0.0}
LAYER_DEFAULTS = {"min": 0.0, "bias": 0.0, "scale": 0.5, "octaves": 8.0, "lacunarity": 2.0, "gain": 0.5,
                  "frequency": 1.0}


def _num(v):
    """a float32 value in text that std::stof reads back to the same bits"""
    return "%.9g" % float(np.float32(v))


def soil(name, chain=None, color="808080", **kw):
    """a soil dict: every chain field names `chain` (default: the soil itself) unless given in kw"""
    s = dict(SOIL_DEFAULTS, name=name, color=color)
    for _, k in CHAINS:
        s[k] = chain or name
    s.update(kw)
    return s


def layer(soil_name, **kw):
    return dict(LAYER_DEFAULTS, soil=soil_name, **kw)


def soil_text(table):
    out = ["# %s (generated)" % table["name"], "", "WORLD {", "", "SCALE %d" % table["scale"],
           "SIZEX %d" % table.get("size", 64), "SIZEY %d" % table.get("size", 64), "", "}", ""]
    if table.get("declare", True):
        for s in table["soils"]:
            out += ["SOIL %s {" % s["name"], "}", ""]
    for s in table["soils"]:
        out += ["SOIL %s {" % s["name"], ""]
        out += ["%s %s" % (kw, s[k]) for kw, k in CHAINS]
        out += ["", "COLOR %s" % s["color"], "Ka 0.5", "Kd 0.8", "Ks 0.2", "Kk 8.0", ""]
        out += ["%s %s" % (kw, _num(s[k])) for kw, k in FLOATS]
        out += ["", "}", ""]
    for l in table["layers"]:
        out += ["LAYER %s {" % l["soil"], ""]
        out += ["%s %s" % (kw, _num(l[k])) for kw, k in LAYER_FLOATS]
        out += ["", "}", ""]
    return "\n".join(out) + "\n"


def write(table, directory):
    """writes `table` as <directory>/<name>.soil and returns the path"""
    path = str(directory) + "/" + table["name"] + ".soil"
    with open(path, "w") as f:
        f.write(soil_text(table))
    return path


# ---- generated tables -----------------------------------------------------------------------------------------
_WORDS = ("Loam", "Red Sand", "Clay", "Silt", "Scree", "Grit", "Peat", "Ash")


def random_table(seed):
    """2 to 5 soils with random chains and parameters drawn from the extremes the presets never use (friction 0 and
    1, maxdiff 0, settling 1, solubility 0 or above 1, erosionrate in (0, 0.95), porosity 0 and 1, suspension on
    several soils), 1 to 9 layers with MIN > 0, negative BIAS and fractional OCTAVES, scale 40 to 200"""
    rng = np.random.RandomState(seed)
    n = int(rng.randint(2, 6))
    names = ["%s %d" % (_WORDS[int(rng.randint(len(_WORDS)))], i) if rng.rand() < 0.6 else "S%d" % i for i in range(n)]

    def pick(*choices):
        c = choices[int(rng.randint(len(choices)))]
        return float(c(rng) if callable(c) else c)

    soils = []
    for i in range(n):
        s = soil(names[i], color="%02X%02X%02X" % tuple(rng.randint(0, 256, 3)))
        for _, k in CHAINS:
            s[k] = names[int(rng.randint(n))]
        s.update(density=pick(lambda r: 0.5 + r.rand(), 1.0),
                 porosity=pick(0.0, 1.0, lambda r: r.rand()),
                 solubility=pick(0.0, 1.0, 1.7, lambda r: r.rand()),
                 equrate=pick(0.2, 1.0, lambda r: 0.05 + 0.9 * r.rand()),
                 friction=pick(1.0, lambda r: 0.05 + 0.5 * r.rand(), lambda r: 0.05 + 0.5 * r.rand(), 0.0) if i else
                 pick(1.0, lambda r: 0.05 + 0.5 * r.rand()),
                 erosionrate=pick(0.0, lambda r: 0.95 * r.rand(), lambda r: 0.01 * r.rand()),
                 maxdiff=pick(0.0, 1.0, lambda r: 0.02 * r.rand()),
                 settling=pick(0.0, 1.0, lambda r: r.rand()),
                 suspension=pick(0.0, 0.0, lambda r: 0.02 * r.rand(), 0.01),
                 abrasion=pick(0.0, lambda r: r.rand()))
        soils.append(s)
    layers = []
    for j in range(int(rng.randint(1, 10))):
        layers.append(layer(names[int(rng.randint(n))],
                            min=pick(0.0, 0.0, lambda r: 0.1 * r.rand()),
                            bias=pick(0.0, lambda r: -0.3 * r.rand(), lambda r: 0.2 * r.rand()),
                            scale=pick(lambda r: 0.05 + 0.6 * r.rand(), 0.5),
                            octaves=pick(8.0, lambda r: 1.0 + 7.0 * r.rand()),
                            lacunarity=pick(2.0, lambda r: 1.5 + r.rand()),
                            gain=pick(0.5, lambda r: 0.3 + 0.4 * r.rand()),
                            frequency=pick(1.0, lambda r: 0.5 + 2.0 * r.rand())))
    return {"name": "gen%d" % seed, "scale": int(rng.choice([40, 80, 120, 160, 200])), "soils": soils,
            "layers": layers, "declare": bool(rng.rand() < 0.5)}


# ---- sentinel tables ----------------------------------------------------------------------------------------
def sentinel_water():
    """Base soil "Base" is the only layer.  A water particle's sediment is Base.transports = "Tr" (water.h:17,83),
    which turns into Tr.erodes = "Er" where the water frequency exceeds Tr.erosionrate = 0 (water.h:83-84: from the
    second frame on), and a cascade off Base deposits Base.cascades = "Ca" (particle.h:92).  Tr, Er and Ca map to
    themselves, so each of them is on the map only if its one mapping ran and its sediment was deposited."""
    soils = [soil("Base", transports="Tr", erodes="Base", cascades="Ca", abrades="Base", friction=0.2, maxdiff=0.002,
                  settling=0.4, porosity=0.4, equrate=0.6),
             soil("Tr", erodes="Er", friction=0.25, maxdiff=0.004, settling=0.2, erosionrate=0.0, equrate=0.7,
                  porosity=0.2),
             soil("Er", friction=0.3, maxdiff=0.004, settling=0.2, equrate=0.4, porosity=0.5),
             soil("Ca", friction=0.1, maxdiff=0.006, settling=0.3, equrate=0.5, porosity=0.1)]
    return {"name": "sentinel_water", "scale": 160, "soils": soils,
            "layers": [layer("Base", scale=0.9, octaves=5.5)], "declare": False}


def sentinel_wind():
    """Wind over two surfaces (wind.h:105 / :119).  "Dune" transports "Dust" (suspension > 0), so particles spawned on
    it carry Dust and lift Dune there; "Crust" transports itself, so a Dust particle over Crust picks nothing up but
    drops Dust, because Crust has suspension > 0 too; particles spawned on Crust carry Crust.  "Dust" can only reach
    the map from a wind particle's deposit."""
    soils = [soil("Dune", transports="Dust", suspension=0.008, friction=0.2, maxdiff=0.005, settling=0.05),
             soil("Crust", suspension=0.004, friction=0.15, maxdiff=0.01, settling=0.1),
             soil("Dust", suspension=0.012, friction=0.1, maxdiff=0.003, settling=0.2)]
    return {"name": "sentinel_wind", "scale": 80, "soils": soils,
            "layers": [layer("Crust", scale=0.6, octaves=6.25), layer("Dune", scale=0.5, bias=-0.2, min=0.02)]}


def friction0():
    """Every soil has friction 0: a water particle stops at its first step (water.h:56), so the batch is all stalls
    and every particle floods."""
    soils = [soil("Rock", friction=0.0, solubility=1.5, maxdiff=0.0, settling=1.0, porosity=0.0),
             soil("Mud", friction=0.0, porosity=1.0, settling=0.5, maxdiff=0.001)]
    return {"name": "friction0", "scale": 120, "soils": soils,
            "layers": [layer("Rock", scale=0.7, octaves=4.5), layer("Mud", scale=0.2, bias=-0.05, min=0.01)]}


def steep():
    """Steep, rough terrain at SCALE 200 of a soil with solubility 4 and equilibrium rate 1: the equilibrium
    concentration hits its clamp at 1 (water.h:72-74), a particle's sediment climbs to it and the evaporation step
    pushes it past 1, where water.h:117 cuts it off."""
    soils = [soil("Scarp", solubility=4.0, equrate=1.0, friction=0.35, maxdiff=0.0, settling=0.02, porosity=0.6),
             soil("Talus", solubility=0.0, equrate=1.0, friction=0.6, maxdiff=0.05, settling=1.0, porosity=1.0)]
    return {"name": "steep", "scale": 200, "soils": soils,
            "layers": [layer("Scarp", scale=3.0, octaves=6.5, frequency=2.5, gain=0.6),
                       layer("Talus", scale=0.3, bias=-0.1, min=0.0)]}


def table_64():
    """Air plus 63 soils chained i -> i + 1 (transports, erodes, cascades; soil 63 maps to itself), each with its
    own friction, maxdiff and settling, and layers that put soils 1, 21, 42, 61, 62 and 63 on the map."""
    names = ["Soil %02d" % i for i in range(1, 64)]
    soils = []
    for i, nm in enumerate(names):
        nxt = names[min(i + 1, 62)]
        soils.append(soil(nm, transports=nxt, erodes=nxt, cascades=nxt, abrades=nm,
                          friction=0.05 + 0.5 * ((i * 37) % 63) / 63.0, maxdiff=0.001 + 0.01 * ((i * 11) % 7) / 7.0,
                          settling=0.05 + 0.9 * ((i * 5) % 9) / 9.0, porosity=((i * 3) % 10) / 10.0,
                          equrate=0.2 + 0.7 * ((i * 13) % 17) / 17.0, erosionrate=0.0,
                          suspension=0.0 if i % 3 else 0.01))
    lay = [layer(names[62], scale=0.3, octaves=3.5), layer(names[0], scale=0.2), layer(names[20], scale=0.2),
           layer(names[41], scale=0.2, bias=-0.05), layer(names[60], scale=0.3), layer(names[61], scale=0.2, min=0.02)]
    return {"name": "soils64", "scale": 160, "soils": soils, "layers": lay}


SENTINELS = {"sentinel_water": sentinel_water, "sentinel_wind": sentinel_wind, "friction0": friction0, "steep": steep}
