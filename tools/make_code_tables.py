"""Build the product's code-table data files from the 3GPP / example-code DATA the reference ships.

Run once in the build container (needs /root/reference); the outputs are committed:
  sionna_b200/phy/fec/ldpc/codes/bg_tables.npz   38.212 Tables 5.3.2-2/-3 as COO triplets
        bg{1,2}_row, bg{1,2}_col : int16 [nnz]     base-graph row / column of each non-empty entry
        bg{1,2}_shift            : int16 [nnz, 8]  circulant shift V_{i,j} for set index i_LS = 0..7
  sionna_b200/phy/fec/ldpc/codes/example_pcms.npz  pcm0..pcm4 (uint8) small example codes
        ((7,4) Hamming, BCH(63,45), BCH(127,106), (3,6) LDPC n=100, 802.11n n=648)
Source data: /root/reference/src/sionna/phy/fec/ldpc/codes/{5G_bg1.csv,5G_bg2.csv,example_codes.npy}
(parsing rule of the csv: /root/reference/src/sionna/phy/fec/ldpc/encoding.py:305-318).
"""
import numpy as np, os
src = "/root/reference/src/sionna/phy/fec/ldpc/codes"
dst = os.path.join(os.path.dirname(__file__), "..", "sionna_b200", "phy", "fec", "ldpc", "codes")
out = {}
for bg in ("bg1", "bg2"):
    csv = np.genfromtxt(os.path.join(src, f"5G_{bg}.csv"), delimiter=";")
    rows, cols, shifts = [], [], []
    r_ind = 0
    for r in range(2, csv.shape[0]):
        if not np.isnan(csv[r, 0]):
            r_ind = int(csv[r, 0])
        rows.append(r_ind); cols.append(int(csv[r, 1])); shifts.append([int(v) for v in csv[r, 2:10]])
    out[f"{bg}_row"] = np.array(rows, np.int16)
    out[f"{bg}_col"] = np.array(cols, np.int16)
    out[f"{bg}_shift"] = np.array(shifts, np.int16)
    print(bg, len(rows), "entries", max(rows) + 1, "x", max(cols) + 1)
np.savez_compressed(os.path.join(dst, "bg_tables.npz"), **out)
pcms = np.load(os.path.join(src, "example_codes.npy"), allow_pickle=True)
np.savez_compressed(os.path.join(dst, "example_pcms.npz"), **{f"pcm{i}": np.array(p, np.uint8) for i, p in enumerate(pcms)})
for i, p in enumerate(pcms): print("pcm", i, np.array(p).shape)

# ---- TR 38.901 Table 7.7.2-1..5 TDL power delay profiles (normalised delays, powers in dB) --------------------------
import json
tdl = {}
mdir = "/root/reference/src/sionna/phy/channel/tr38901/models"
for m in ("A", "B", "C", "D", "E", "A30", "B100", "C300"):   # the last three: TS 38.104 Annex G, delays in ns
    with open(os.path.join(mdir, f"TDL-{m}.json")) as f:
        d = json.load(f)
    tdl[f"{m}_delays"] = np.array(d["delays"], np.float64)
    tdl[f"{m}_powers_db"] = np.array(d["powers"], np.float64)
    tdl[f"{m}_los"] = np.array(int(d["los"]))
    tdl[f"{m}_scale_delays"] = np.array(int(d["scale_delays"]))
    print("TDL-" + m, d["num_clusters"], "taps, los", d["los"])
np.savez_compressed(os.path.join(os.path.dirname(__file__), "..", "sionna_b200", "phy", "channel", "tdl_models.npz"), **tdl)

# ---- TR 38.901 Tables 7.7.1-1..5 CDL clusters (normalised delays, powers in dB, angles in degrees) -------------------
# Written as text (JSON, one object per model). Rows stay in table order (not delay order); for the LoS models D and E
# row 0 is the specular component.
cdl = {}
for m in ("A", "B", "C", "D", "E"):
    with open(os.path.join(mdir, f"CDL-{m}.json")) as f:
        d = json.load(f)
    t = {"los": int(d["los"]), "num_clusters": int(d["num_clusters"]),
         "delays": [float(v) for v in d["delays"]], "powers_db": [float(v) for v in d["powers"]]}
    for k in ("aod", "aoa", "zod", "zoa"):
        t[k] = [float(v) for v in d[k]]
    for k in ("cASD", "cASA", "cZSD", "cZSA"):
        t[k] = float(d[k])
    t["xpr_db"] = float(d["xpr"])
    cdl[m] = t
    print("CDL-" + m, d["num_clusters"], "clusters,", len(d["delays"]), "rows, los", d["los"])
with open(os.path.join(os.path.dirname(__file__), "..", "sionna_b200", "phy", "channel", "cdl_models.json"), "w") as f:
    json.dump(cdl, f, indent=1)
    f.write("\n")
