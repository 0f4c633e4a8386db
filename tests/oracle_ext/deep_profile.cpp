// TEST INFRASTRUCTURE -- the oracle's error-profile estimator (oracle/pipeline.hpp ProfileEstimator, used unchanged) as the reference's
// --deepprofileonly (src/daccord.cpp:1442-1650, handleIndelEstimateDeep<8> :634-995), with the second-DB and --vard input handling of
// two_db.cpp; built by tests/test_deep_profile.py, never linked into the product.
//
// ProfileEstimator::handleRead only sums its windows.  read_windows below restates its window loop step for step on the estimator's own
// parts (selectOverlaps, computeTrace, advanceA / stringLengthUsed, the DebruijnGraph, the aligner) and records every window instead;
// every read is also run through the unchanged handleRead, and the summed records must equal what it adds up, or the driver fails.
// The [deep] lines are written through std::ostream as the reference writes them; the product formats them with printf, so the two
// formatters check each other.
#include "two_db.cpp"
#include <sstream>

namespace {

struct WinRec { uint32_t aread, astart, status, reserved; uint32_t cnt[4]; };     // dcu_profile_window's layout

// one window with a non-empty pile: status 0 fewer than 3 sequences, 1 a repeated 7-mer, 2 no trivial consensus, 3 consensus (stats =
// its alignment steps; their error rate is what --deepprofileonly collects, :945-955)
struct ProfileWindow { uint64_t aread, astart; int status; AlignStats stats; };

// ProfileEstimator::handleRead's window loop (oracle/pipeline.hpp), each window appended to W
void read_windows(ProfileEstimator& PE, uint64_t aread, std::vector<ProfileWindow>& W) {
  typedef ProfileEstimator PEs;
  std::vector<const OvlRec*> ita; PE.selectOverlaps(aread, ita);
  const uint64_t nintv = ita.size();
  if (!nintv) return;
  const std::string& A = PE.DB.reads[aread];
  double maxerate = 0.0, minerate = 1.0; uint64_t maxaepos = 0;
  std::vector<std::vector<uint8_t>> traces(nintv); std::vector<std::string> bseq(nintv);
  for (uint64_t z = 0; z < nintv; ++z) {
    const OvlRec& o = *ita[z];
    double er = (double)o.diffs / (double)(o.aepos - o.abpos);
    if (er > maxerate) maxerate = er;
    if (er < minerate) minerate = er;
    if ((uint64_t)o.aepos > maxaepos) maxaepos = (uint64_t)o.aepos;
    bseq[z] = (o.flags & 1) ? revcomp(PE.DB.reads[o.bread]) : PE.DB.reads[o.bread];
    PE.computeTrace(o, (const uint8_t*)A.data(), (const uint8_t*)bseq[z].data(), traces[z]);
  }
  const double ediv = (maxerate > minerate) ? (maxerate - minerate) : 1.0;
  typedef std::pair<uint64_t, uint64_t> upair;
  FiniteHeap<upair> E(1024);
  std::map<uint64_t, ActiveElement> activeset;
  std::vector<SeqRef> MA;
  const uint64_t ylimit = (maxaepos + PEs::EA >= PEs::EW) ? ((maxaepos + PEs::EA - PEs::EW) / PEs::EA) : 0;
  uint64_t z = 0;
  for (uint64_t y = 0; y < ylimit; ++y) {
    const uint64_t astart = y * PEs::EA, aend = astart + PEs::EW;
    while (z < nintv && (int64_t)astart >= ita[z]->abpos) {
      const OvlRec& o = *ita[z];
      if (o.aepos >= (int64_t)astart) {
        const uint64_t aoff = astart - (uint64_t)o.abpos;
        const uint8_t* ta = traces[z].data(); const uint8_t* te = ta + traces[z].size();
        auto adv = advanceA(ta, te, aoff);
        uint64_t uboff = (uint64_t)o.bbpos + stringLengthUsed(ta, ta + adv.second).second;
        ta += adv.second;
        double er = (double)o.diffs / (double)(o.aepos - o.abpos);
        uint64_t escore = (uint64_t)(((er - minerate) / ediv) * std::numeric_limits<uint32_t>::max());
        uint64_t eindex = (escore << 32) | z;
        activeset[eindex] = ActiveElement{(const uint8_t*)A.data() + astart, (const uint8_t*)bseq[z].data() + uboff, ta, te, uboff};
        E.pushBump(upair((uint64_t)o.aepos, eindex));
      }
      ++z;
    }
    while (!E.empty() && E.top().first <= aend) { upair UP = E.pop(); activeset.erase(UP.second); }
    MA.clear();
    for (auto& kv : activeset) {
      ActiveElement& AE = kv.second;
      auto adv = advanceA(AE.ta, AE.te, PEs::EW);
      uint64_t blen = stringLengthUsed(AE.ta, AE.ta + adv.second).second;
      if (MA.empty()) MA.push_back(SeqRef(AE.ua, PEs::EW));
      if (MA.size() < PE.maxalign) MA.push_back(SeqRef(AE.ub, blen));
      auto advadv = advanceA(AE.ta, AE.te, PEs::EA);
      uint64_t badv = stringLengthUsed(AE.ta, AE.ta + advadv.second).second;
      AE.ua += PEs::EA; AE.ta += advadv.second; AE.ub += badv; AE.uboff += badv;
    }
    if (MA.empty()) continue;
    if (MA.size() < 3) { W.push_back(ProfileWindow{aread, astart, 0, AlignStats()}); continue; }
    bool rep = false;
    for (auto& sr : MA) rep = hasRepeatedKmer(sr.first, sr.second, PEs::EK - 1) || rep;
    if (rep) { W.push_back(ProfileWindow{aread, astart, 1, AlignStats()}); continue; }
    PE.DG.setup(MA.data(), MA.size());
    PE.DG.filterFreq(2, MA.size());
    std::string cons;
    if (!PE.DG.traverseTrivial(cons)) { W.push_back(ProfileWindow{aread, astart, 2, AlignStats()}); continue; }
    AlignStats GAS;
    for (auto& sr : MA) {
      PE.NP.align((const uint8_t*)cons.data(), cons.size(), sr.first, sr.second);
      for (uint8_t st : PE.NP.trace) switch (st) {
        case STEP_MATCH: GAS.matches++; break; case STEP_MISMATCH: GAS.mismatches++; break;
        case STEP_INS: GAS.insertions++; break; default: GAS.deletions++; break; }
    }
    W.push_back(ProfileWindow{aread, astart, 3, GAS});
  }
}

// the estimator's windows of A-reads [first, top) (no cap on the count), in read order
std::vector<ProfileWindow> windows(const char* lasfn, const char* dbfn, const char* db2fn, int64_t first, int64_t top, uint64_t maxalign, uint64_t maxinput,
                                   uint64_t vard) {
  ReadDB DB; LasFile L;
  const uint64_t nA = load_inputs(lasfn, dbfn, db2fn, vard, DB, L);
  const uint64_t avg = vard ? average_read_length(DB) : 0;
  if (first < 0) first = 0;
  if (top < 0 || top > (int64_t)nA) top = (int64_t)nA;
  std::vector<ProfileWindow> W;
  ProfileEstimator PE(L, DB, maxalign, maxinput);
  for (int64_t r = first; r < top; ++r) {
    if (L.first[r] == L.first[r + 1]) continue;
    PE.maxinput = lmaxinput(DB.reads[r].size(), maxinput, vard, avg);
    const size_t w0 = W.size();
    read_windows(PE, (uint64_t)r, W);
    ProfileResult R, S;                                    // the unchanged estimator on the same read must sum to the records
    PE.handleRead((uint64_t)r, R);
    for (size_t i = w0; i < W.size(); ++i) {
      if (W[i].status == 1) S.unusable++;
      if (W[i].status >= 2) S.usable++;
      S.stats.add(W[i].stats);
    }
    if (R.usable != S.usable || R.unusable != S.unusable || R.stats.matches != S.stats.matches || R.stats.mismatches != S.stats.mismatches ||
        R.stats.insertions != S.stats.insertions || R.stats.deletions != S.stats.deletions)
      throw std::runtime_error("per-window restatement differs from ProfileEstimator::handleRead at read " + std::to_string(r));
  }
  return W;
}

}  // namespace

extern "C" {

// per-window records of A-reads [first, top): malloc'ed array of *n WinRec (free with two_db_free), NULL on error
void* deep_profile_windows(const char* lasfn, const char* dbfn, const char* db2fn, int64_t first, int64_t top, uint64_t maxalign, uint64_t maxinput, uint64_t vard,
                           uint64_t* n) {
  try {
    const std::vector<ProfileWindow> W = windows(lasfn, dbfn, db2fn, first, top, maxalign, maxinput, vard);
    WinRec* out = (WinRec*)malloc(std::max<size_t>(W.size(), 1) * sizeof(WinRec));
    for (size_t i = 0; i < W.size(); ++i) {
      const AlignStats& s = W[i].stats;
      out[i] = WinRec{(uint32_t)W[i].aread, (uint32_t)W[i].astart, (uint32_t)W[i].status, 0u,
                      {(uint32_t)s.matches, (uint32_t)s.mismatches, (uint32_t)s.insertions, (uint32_t)s.deletions}};
    }
    *n = W.size();
    return out;
  } catch (std::exception& e) { fprintf(stderr, "[oracle] %s\n", e.what()); return nullptr; }
}

// `daccord --deepprofileonly` over A-reads [first, min(top, first + 4096)): the [deep] lines (malloc'ed, *len bytes), NULL on error
char* deep_profile_text(const char* lasfn, const char* dbfn, const char* db2fn, int64_t first, int64_t top, uint64_t maxalign, uint64_t maxinput, uint64_t vard,
                        uint64_t* len) {
  try {
    if (first < 0) first = 0;
    if (top >= 0) top = std::min(top, first + 4096);
    else top = first + 4096;
    std::vector<uint32_t> vals;
    for (const ProfileWindow& w : windows(lasfn, dbfn, db2fn, first, top, maxalign, maxinput, vard)) {
      if (w.status != 3) continue;
      const double e = w.stats.errorRate();                                            // :945-955
      const uint64_t v = static_cast<uint64_t>(static_cast<double>(std::numeric_limits<uint32_t>::max()) * e + 0.5);
      vals.push_back(static_cast<uint32_t>(std::min(v, static_cast<uint64_t>(std::numeric_limits<uint32_t>::max()))));
    }
    std::sort(vals.begin(), vals.end());
    std::ostringstream os;                                                              // :1612-1646
    int64_t prevD = -1; uint64_t n = 0, s = 0;
    const double dcnt = vals.size();
    for (uint32_t d : vals) {
      if (static_cast<int64_t>(d) != prevD) {
        if (n) { s += n; os << "[deep]\t" << (prevD / static_cast<double>(std::numeric_limits<uint32_t>::max())) << "\t" << s / dcnt << "\n"; }
        prevD = static_cast<int64_t>(d); n = 0;
      }
      n += 1;
    }
    if (n) { s += n; os << "[deep]\t" << (prevD / static_cast<double>(std::numeric_limits<uint32_t>::max())) << "\t" << s / dcnt << "\n"; }
    const std::string out = os.str();
    char* buf = (char*)malloc(out.size() + 1); memcpy(buf, out.data(), out.size()); buf[out.size()] = 0;
    *len = out.size();
    return buf;
  } catch (std::exception& e) { fprintf(stderr, "[oracle] %s\n", e.what()); return nullptr; }
}

}  // extern "C"
