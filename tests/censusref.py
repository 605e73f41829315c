"""ClusterSimulation's proposal census (proposal_census=True) restated over simref's per-tag proposals (NOT a pytest module).

An interval's census groups the (receiver tag, proposal) pairs the oracle's receivers announced in it by proposal, in order of
the lowest ring-0 position that announced each; size is the proposal's length, down its members, up its registered joiners,
voters the receivers that announced it, representative the tag of the lowest.  A configuration's census merges its intervals'
classes by proposal in order of first appearance; against the decided cut, missing = |cut - proposal|, extra = |proposal - cut|,
decided = (proposal == cut); agreement = the decided proposal's voters over the configuration's announcers."""
from simref import OracleSimulation


class CensusOracleSimulation(OracleSimulation):
    def _new_configuration(self):
        super()._new_configuration()
        self.classes = {}                                         # frozenset(proposal) -> class of the configuration

    def _deliver(self, batches, cfg, i):
        new = super()._deliver(batches, cfg, i)
        pos = {t: p for p, t in enumerate(self.ring0)}
        members = set(self.tags)
        out, at = [], {}
        for tag, prop in sorted(new, key=lambda x: pos[x[0]]):
            k = frozenset(prop)
            if k not in at:
                down = sum(1 for t in prop if t in members)
                at[k] = len(out)
                out.append({"size": len(prop), "down": down, "up": len(prop) - down, "voters": 0, "representative": tag})
            out[at[k]]["voters"] += 1
        for k, c in at.items():
            if k in self.classes:
                self.classes[k]["voters"] += out[c]["voters"]
            else:
                self.classes[k] = {key: out[c][key] for key in ("size", "down", "up", "voters")}
        self.interval_census = out
        return new

    def interval(self):
        self.interval_census = None
        rec = super().interval()
        if rec["announced"]:
            rec["census"] = self.interval_census
        return rec

    def _view_change(self, path, value, i):
        cut = frozenset(value)
        census = [dict(c, decided=k == cut, missing=len(cut - k), extra=len(k - cut)) for k, c in self.classes.items()]
        total = sum(c["voters"] for c in census)
        agreement = sum(c["voters"] for c in census if c["decided"]) / total if total else None
        super()._view_change(path, value, i)
        self.history[-1]["census"], self.history[-1]["agreement"] = census, agreement
