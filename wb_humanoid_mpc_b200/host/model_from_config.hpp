// Host layer (C++17, no dependencies): the reference's own config files -> HostModel (b200sqp_model_desc + reference-manager parameters).
//
// WBMpcInterface builds its OptimalControlProblem from URDF + task.info + reference.info + gait.info
// (humanoid_nmpc/humanoid_wb_mpc/src/WBMpcInterface.cpp:60-199) through Pinocchio's URDF importer, boost::property_tree and the term
// factories.  A GPU cannot consume those objects; this loader derives the flat description the C ABI takes from the SAME files, so that a node
// needs nothing but the paths it already passes to the interface (no Python, no intermediate model file):
//   * boost INFO subset of loadData::loadPtreeValue / loadEigenMatrix / loadStdVector (ocs2_core/include/ocs2_core/misc/LoadData.h);
//   * URDF subset urdfdom gives Pinocchio: <link><inertial>, <joint> origin / axis / limit / parent / child;
//   * the conventions of createCustomPinocchioInterface (humanoid_common_mpc/src/pinocchio_model/createPinocchioModel.cpp:60-182): joints not
//     in the MPC joint list are welded and their child inertias folded into the parent body, joints ordered depth first with children sorted
//     by joint name (urdfdom keeps them in a std::map), contact / collision frames attached to their parent joint's frame;
//   * the term constants of ModelSettings / HumanoidCostConstraintFactory / WBMpcInterface, field by field as
//     wb_humanoid_mpc_b200/model_loader.py documents them (each with its reference source line).
// Both MPCs: the whole-body one (WBMpcInterface) and, with centroidal = true, the centroidal one (CentroidalMpcInterface: other state layout and
// weights, the task-space link cost, ICP and leg-torque costs, and the nominal inertia of the single-rigid-body model type).
// tests/test_host_cpp.py compares every field with the flat model file derived by the Python loader.
#pragma once
#include <algorithm>
#include <cmath>
#include <functional>
#include <set>

#include "model_file.hpp"

namespace b200sqp::host {
namespace cfg {

// ---- boost::property_tree INFO subset ---------------------------------------------------------------------------------------------------
struct Info {
  std::string value;
  std::vector<std::pair<std::string, Info>> kids;
  const Info* find(const std::string& key) const {
    for (const auto& k : kids)
      if (k.first == key) return &k.second;
    return nullptr;
  }
  const Info& at(const std::string& dotted) const {
    const Info* n = this;
    size_t a = 0;
    while (a <= dotted.size()) {
      const size_t b = std::min(dotted.find('.', a), dotted.size());
      n = n->find(dotted.substr(a, b - a));
      if (!n) throw std::invalid_argument("[b200sqp::host] config key not found: " + dotted);
      a = b + 1;
    }
    return *n;
  }
  double num(const std::string& dotted) const {
    std::string v = at(dotted).value;
    while (!v.empty() && v.back() == ';') v.pop_back();
    return std::stod(v);
  }
  // loadStdVector: entries "[i] value"
  std::vector<std::string> list(const std::string& dotted) const {
    std::vector<std::pair<int, std::string>> items;
    for (const auto& k : at(dotted).kids)
      if (k.first.size() > 2 && k.first.front() == '[' && k.first.back() == ']') items.emplace_back(std::stoi(k.first.substr(1, k.first.size() - 2)), k.second.value);
    std::sort(items.begin(), items.end(), [](const auto& x, const auto& y) { return x.first < y.first; });
    std::vector<std::string> out;
    for (auto& it : items) out.push_back(it.second);
    return out;
  }
  // loadEigenMatrix: the diagonal of a matrix given by entries "(i,j) v" with an optional "scaling" (missing entries are zero)
  std::vector<double> diagonal(const std::string& name, int n) const {
    const Info& blk = at(name);
    std::vector<double> d(n, 0.0);
    const Info* sc = blk.find("scaling");
    const double scaling = sc ? std::stod(sc->value) : 1.0;
    for (const auto& k : blk.kids) {
      int i = -1, j = -1;
      if (std::sscanf(k.first.c_str(), "(%d,%d)", &i, &j) == 2 && i == j && i >= 0 && i < n) d[i] = std::stod(k.second.value) * scaling;
    }
    return d;
  }
  std::vector<double> column(const std::string& name, int n) const {
    const Info& blk = at(name);
    std::vector<double> d(n, 0.0);
    const Info* sc = blk.find("scaling");
    const double scaling = sc ? std::stod(sc->value) : 1.0;
    for (const auto& k : blk.kids) {
      int i = -1, j = -1;
      if (std::sscanf(k.first.c_str(), "(%d,%d)", &i, &j) == 2 && j == 0 && i >= 0 && i < n) d[i] = std::stod(k.second.value) * scaling;
    }
    return d;
  }
};

inline std::string readFile(const std::string& path) {
  std::ifstream in(path);
  if (!in) throw std::invalid_argument("[b200sqp::host] file not found: " + path);   // the reference interfaces throw std::invalid_argument too
  std::ostringstream ss;
  ss << in.rdbuf();
  return ss.str();
}

inline Info parseInfo(const std::string& path) {
  const std::string text = readFile(path);
  std::vector<std::string> toks;   // "\n" separates lines
  std::istringstream lines(text);
  std::string line;
  while (std::getline(lines, line)) {
    line = line.substr(0, line.find(';'));     // ';' starts a comment
    const size_t sl = line.find("//");         // '//' comments appear in the shipped task.info as well
    if (sl != std::string::npos) line = line.substr(0, sl);
    size_t i = 0;
    while (i < line.size()) {
      const char c = line[i];
      if (std::isspace(static_cast<unsigned char>(c))) {
        ++i;
      } else if (c == '{' || c == '}') {
        toks.emplace_back(1, c);
        ++i;
      } else if (c == '"') {
        const size_t e = line.find('"', i + 1);
        toks.push_back(line.substr(i + 1, (e == std::string::npos ? line.size() : e) - i - 1));
        i = (e == std::string::npos) ? line.size() : e + 1;
      } else {
        size_t e = i;
        while (e < line.size() && !std::isspace(static_cast<unsigned char>(line[e])) && line[e] != '{' && line[e] != '}') ++e;
        toks.push_back(line.substr(i, e - i));
        i = e;
      }
    }
    toks.emplace_back("\n");
  }
  size_t pos = 0;
  std::function<Info()> block = [&]() {
    Info node;
    while (pos < toks.size()) {
      const std::string t = toks[pos];
      if (t == "\n") {
        ++pos;
        continue;
      }
      if (t == "}") {
        ++pos;
        return node;
      }
      ++pos;
      Info child;
      if (pos < toks.size() && toks[pos] != "\n" && toks[pos] != "{" && toks[pos] != "}") {
        child.value = toks[pos++];
        while (pos < toks.size() && toks[pos] != "\n" && toks[pos] != "{" && toks[pos] != "}") ++pos;   // trailing tokens of the line
      }
      size_t save = pos;
      while (pos < toks.size() && toks[pos] == "\n") ++pos;
      if (pos < toks.size() && toks[pos] == "{") {
        ++pos;
        Info sub = block();
        sub.value = child.value;
        child = std::move(sub);
      } else {
        pos = save;
      }
      node.kids.emplace_back(t, std::move(child));
    }
    return node;
  };
  return block();
}

// ---- XML subset (elements, attributes; text, comments, declarations skipped) -----------------------------------------------------------------
struct Xml {
  std::string tag;
  std::map<std::string, std::string> attr;
  std::vector<Xml> kids;
  const Xml* child(const std::string& t) const {
    for (const auto& k : kids)
      if (k.tag == t) return &k;
    return nullptr;
  }
  std::string get(const std::string& a, const std::string& dflt = "") const {
    auto it = attr.find(a);
    return it == attr.end() ? dflt : it->second;
  }
};

inline Xml parseXml(const std::string& path) {
  const std::string s = readFile(path);
  size_t i = 0;
  Xml root;
  std::vector<Xml*> stack{&root};
  while ((i = s.find('<', i)) != std::string::npos) {
    if (s.compare(i, 4, "<!--") == 0) {
      i = s.find("-->", i);
      if (i == std::string::npos) break;
      i += 3;
      continue;
    }
    if (s[i + 1] == '?' || s[i + 1] == '!') {
      i = s.find('>', i);
      continue;
    }
    if (s[i + 1] == '/') {
      if (stack.size() > 1) stack.pop_back();
      i = s.find('>', i);
      continue;
    }
    size_t e = i + 1;
    while (e < s.size() && !std::isspace(static_cast<unsigned char>(s[e])) && s[e] != '>' && s[e] != '/') ++e;
    Xml el;
    el.tag = s.substr(i + 1, e - i - 1);
    bool selfClosing = false;
    while (e < s.size() && s[e] != '>') {
      if (s[e] == '/') {
        selfClosing = true;
        ++e;
        continue;
      }
      if (std::isspace(static_cast<unsigned char>(s[e]))) {
        ++e;
        continue;
      }
      size_t q = s.find('=', e);
      if (q == std::string::npos) break;
      std::string name = s.substr(e, q - e);
      while (!name.empty() && std::isspace(static_cast<unsigned char>(name.back()))) name.pop_back();
      size_t v0 = s.find_first_of("\"'", q);
      if (v0 == std::string::npos) break;
      const size_t v1 = s.find(s[v0], v0 + 1);
      if (v1 == std::string::npos) break;
      el.attr[name] = s.substr(v0 + 1, v1 - v0 - 1);
      e = v1 + 1;
    }
    stack.back()->kids.push_back(std::move(el));
    if (!selfClosing) stack.push_back(&stack.back()->kids.back());
    i = e;
  }
  if (root.kids.empty()) throw std::invalid_argument("[b200sqp::host] no XML element in " + path);
  return root.kids.front();
}

// ---- small fixed-size algebra (row-major 3 x 3) ------------------------------------------------------------------------------------------------
struct M3 {
  double m[9];
};
struct V3 {
  double x, y, z;
};
inline M3 eye() { return M3{{1, 0, 0, 0, 1, 0, 0, 0, 1}}; }
inline M3 mul(const M3& a, const M3& b) {
  M3 c{};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c.m[3 * i + j] = a.m[3 * i] * b.m[j] + a.m[3 * i + 1] * b.m[3 + j] + a.m[3 * i + 2] * b.m[6 + j];
  return c;
}
inline M3 tr(const M3& a) { return M3{{a.m[0], a.m[3], a.m[6], a.m[1], a.m[4], a.m[7], a.m[2], a.m[5], a.m[8]}}; }
inline V3 mul(const M3& a, V3 v) { return V3{a.m[0] * v.x + a.m[1] * v.y + a.m[2] * v.z, a.m[3] * v.x + a.m[4] * v.y + a.m[5] * v.z, a.m[6] * v.x + a.m[7] * v.y + a.m[8] * v.z}; }
inline V3 add(V3 a, V3 b) { return V3{a.x + b.x, a.y + b.y, a.z + b.z}; }
inline V3 sub(V3 a, V3 b) { return V3{a.x - b.x, a.y - b.y, a.z - b.z}; }
inline V3 vec3(const std::string& s) {
  std::istringstream ss(s);
  V3 v{};
  if (!(ss >> v.x >> v.y >> v.z)) throw std::invalid_argument("[b200sqp::host] URDF: expected three numbers in '" + s + "'");
  return v;
}
inline M3 rpyToR(V3 rpy) {   // urdfdom / Pinocchio: R = Rz(yaw) Ry(pitch) Rx(roll)
  const double cr = std::cos(rpy.x), sr = std::sin(rpy.x), cp = std::cos(rpy.y), sp = std::sin(rpy.y), cy = std::cos(rpy.z), sy = std::sin(rpy.z);
  const M3 Rx{{1, 0, 0, 0, cr, -sr, 0, sr, cr}}, Ry{{cp, 0, sp, 0, 1, 0, -sp, 0, cp}}, Rz{{cy, -sy, 0, sy, cy, 0, 0, 0, 1}};
  return mul(mul(Rz, Ry), Rx);
}

struct Inertia {   // mass, com (in the frame it is expressed in), rotational inertia about the com (same axes)
  double m = 0.0;
  V3 c{0, 0, 0};
  M3 I{{0, 0, 0, 0, 0, 0, 0, 0, 0}};
  Inertia transformed(const M3& R, V3 p) const { return Inertia{m, add(mul(R, c), p), mul(mul(R, I), tr(R))}; }   // x_parent = R x + p
  static M3 shift(const M3& I, double mm, V3 d) {   // parallel axis: about the point c, com at c + d
    const double dd = d.x * d.x + d.y * d.y + d.z * d.z;
    const double o[9] = {d.x * d.x, d.x * d.y, d.x * d.z, d.y * d.x, d.y * d.y, d.y * d.z, d.z * d.x, d.z * d.y, d.z * d.z};
    M3 r = I;
    for (int k = 0; k < 9; ++k) r.m[k] += mm * ((k % 4 == 0 ? dd : 0.0) - o[k]);
    return r;
  }
  Inertia operator+(const Inertia& o) const {
    const double mt = m + o.m;
    if (mt == 0.0) return Inertia{};
    const V3 cc{(m * c.x + o.m * o.c.x) / mt, (m * c.y + o.m * o.c.y) / mt, (m * c.z + o.m * o.c.z) / mt};
    const M3 a = shift(I, m, sub(c, cc)), b = shift(o.I, o.m, sub(o.c, cc));
    Inertia r{mt, cc, a};
    for (int k = 0; k < 9; ++k) r.I.m[k] += b.m[k];
    return r;
  }
};

struct UrdfJoint {
  std::string type, parent, child;
  M3 R;
  V3 p, axis;
  double lower, upper;
};
struct Body {
  std::string joint;
  int parent;
  M3 R;
  V3 p, axis;
  Inertia inertia;
  double lower, upper;
};

}  // namespace cfg

// the MPC of WBMpcInterface (or, centroidal = true, of CentroidalMpcInterface) from its own files; gaitFile may be empty (no gait table)
// WBMpcInterface::getJointTorqueCost: loadEigenMatrix(taskFile, "joint_torque_weights") into nj entries (MPC joint order); empty when the key is
// absent.  Reading the key does not switch the term on (SqpSolver::setJointTorqueCost does), as the key alone does nothing in the reference.
inline std::vector<double> loadJointTorqueWeights(const std::string& taskFile, int nj = 23) {
  const cfg::Info task = cfg::parseInfo(taskFile);
  if (!task.find("joint_torque_weights")) return {};
  return task.column("joint_torque_weights", nj);
}

inline HostModel loadModelFromConfig(const std::string& urdfFile, const std::string& taskFile, const std::string& referenceFile,
                                     const std::string& gaitFile, bool centroidal = false) {
  using namespace cfg;
  const Info task = parseInfo(taskFile);
  // ---- URDF -> links, joints -----------------------------------------------------------------------------------------------------------------
  const Xml robot = parseXml(urdfFile);
  std::map<std::string, Inertia> links;
  std::map<std::string, UrdfJoint> joints;   // std::map: alphabetical, as urdfdom keeps them
  for (const Xml& el : robot.kids) {
    if (el.tag == "link") {
      Inertia in;
      if (const Xml* ine = el.child("inertial")) {
        const Xml* org = ine->child("origin");
        const V3 xyz = org ? vec3(org->get("xyz", "0 0 0")) : V3{0, 0, 0}, rpy = org ? vec3(org->get("rpy", "0 0 0")) : V3{0, 0, 0};
        const Xml *ms = ine->child("mass"), *it = ine->child("inertia");
        if (!ms || !it) throw std::invalid_argument("[b200sqp::host] URDF: <inertial> of link '" + el.get("name") + "' lacks mass / inertia");
        auto f = [&](const char* a) { return std::stod(it->get(a, "0")); };
        const M3 I{{f("ixx"), f("ixy"), f("ixz"), f("ixy"), f("iyy"), f("iyz"), f("ixz"), f("iyz"), f("izz")}};
        const M3 R = rpyToR(rpy);
        in = Inertia{std::stod(ms->get("value")), xyz, mul(mul(R, I), tr(R))};
      }
      links[el.get("name")] = in;
    } else if (el.tag == "joint") {
      UrdfJoint j;
      j.type = el.get("type");
      const Xml *org = el.child("origin"), *ax = el.child("axis"), *lim = el.child("limit"), *pa = el.child("parent"), *ch = el.child("child");
      if (!pa || !ch) throw std::invalid_argument("[b200sqp::host] URDF: joint '" + el.get("name") + "' lacks parent / child");
      j.parent = pa->get("link");
      j.child = ch->get("link");
      j.p = org ? vec3(org->get("xyz", "0 0 0")) : V3{0, 0, 0};
      j.R = rpyToR(org ? vec3(org->get("rpy", "0 0 0")) : V3{0, 0, 0});
      j.axis = ax ? vec3(ax->get("xyz")) : V3{1, 0, 0};
      j.lower = (lim && !lim->get("lower").empty()) ? std::stod(lim->get("lower")) : -INFINITY;
      j.upper = (lim && !lim->get("upper").empty()) ? std::stod(lim->get("upper")) : INFINITY;
      joints[el.get("name")] = j;
    }
  }
  // ---- weld the fixed joints, order the bodies as Pinocchio orders its joints ----------------------------------------------------------------
  const std::vector<std::string> fixedList = task.list("model_settings.fixedJointNames");
  const std::set<std::string> fixed(fixedList.begin(), fixedList.end());
  std::set<std::string> childLinks;
  std::map<std::string, std::vector<std::string>> byParent;
  for (const auto& kv : joints) {
    childLinks.insert(kv.second.child);
    byParent[kv.second.parent].push_back(kv.first);
  }
  std::string rootLink;
  for (const auto& kv : links)
    if (!childLinks.count(kv.first)) {
      if (!rootLink.empty()) throw std::invalid_argument("[b200sqp::host] URDF: more than one root link");
      rootLink = kv.first;
    }
  std::vector<Body> bodies{Body{"", -1, eye(), V3{0, 0, 0}, V3{0, 0, 0}, Inertia{}, 0.0, 0.0}};
  struct LinkPlacement {
    int body;
    M3 R;
    V3 p;
  };
  std::map<std::string, LinkPlacement> linkBody;   // link frame in the joint frame of the body it is welded to
  std::function<void(const std::string&, int, const M3&, V3)> visit = [&](const std::string& link, int bi, const M3& R, V3 p) {
    linkBody[link] = LinkPlacement{bi, R, p};
    bodies[bi].inertia = bodies[bi].inertia + links.at(link).transformed(R, p);
    auto it = byParent.find(link);
    if (it == byParent.end()) return;
    for (const std::string& jn : it->second) {
      const UrdfJoint& j = joints.at(jn);
      const M3 Rj = mul(R, j.R);
      const V3 pj = add(mul(R, j.p), p);
      const bool isFixed = fixed.count(jn) != 0;
      if (!isFixed && (j.type == "floating" || j.type == "prismatic" || j.type == "planar"))
        throw std::invalid_argument("[b200sqp::host] unsupported joint type " + j.type + " for " + jn);
      if (!isFixed && (j.type == "revolute" || j.type == "continuous")) {
        const double nrm = std::sqrt(j.axis.x * j.axis.x + j.axis.y * j.axis.y + j.axis.z * j.axis.z);
        bodies.push_back(Body{jn, bi, Rj, pj, V3{j.axis.x / nrm, j.axis.y / nrm, j.axis.z / nrm}, Inertia{}, j.lower, j.upper});
        visit(j.child, static_cast<int>(bodies.size()) - 1, eye(), V3{0, 0, 0});
      } else {
        visit(j.child, bi, Rj, pj);
      }
    }
  };
  visit(rootLink, 0, eye(), V3{0, 0, 0});

  HostModel m;
  m.name = centroidal ? "g1_centroidal" : "g1_wb";
  m.centroidal = centroidal;
  m.nj = static_cast<int>(bodies.size()) - 1;
  m.nx = centroidal ? 12 + m.nj : 2 * (6 + m.nj);   // CentroidalMpcRobotModel.h:52-160 / WBAccelMpcRobotModel.h:76-241
  m.nu = 12 + m.nj;
  if (m.nj + 1 > 32 || m.nx > 64 || m.nu > 40) throw std::invalid_argument("[b200sqp::host] model exceeds the sizes of b200sqp_model_desc");
  std::map<std::string, int> jidx;
  for (int i = 1; i <= m.nj; ++i) jidx[bodies[i].joint] = i - 1;
  auto jointIndex = [&](const std::string& n) {
    auto it = jidx.find(n);
    if (it == jidx.end()) throw std::invalid_argument("[b200sqp::host] '" + n + "' is not an MPC joint");
    return it->second;
  };
  b200sqp_model_desc& d = m.desc;
  std::memset(&d, 0, sizeof(d));
  d.nj = m.nj;
  for (int i = 0; i <= m.nj; ++i) {
    const Body& b = bodies[i];
    d.parent[i] = b.parent;
    for (int k = 0; k < 9; ++k) {
      d.joint_R[i][k] = b.R.m[k];
      d.inertia[i][k] = b.inertia.I.m[k];
    }
    const double jp[3] = {b.p.x, b.p.y, b.p.z}, ax[3] = {b.axis.x, b.axis.y, b.axis.z}, cm[3] = {b.inertia.c.x, b.inertia.c.y, b.inertia.c.z};
    for (int k = 0; k < 3; ++k) {
      d.joint_p[i][k] = jp[k];
      d.joint_axis[i][k] = i ? ax[k] : 0.0;
      d.com[i][k] = cm[k];
    }
    d.mass[i] = b.inertia.m;
    m.totalMass += b.inertia.m;
    if (i) {
      d.q_lower[i - 1] = b.lower;
      d.q_upper[i - 1] = b.upper;
    }
  }
  // ---- frames: contact points, collision points, ankle / knee collision frames (createPinocchioModel.cpp:76-131) --------------------------------
  const auto contactNames = task.list("model_settings.contactNames6DoF"), contactParents = task.list("model_settings.contactParentJointNames");
  const V3 ct{task.num("contacts.contact_frame_translation.x"), task.num("contacts.contact_frame_translation.y"), task.num("contacts.contact_frame_translation.z")};
  const double xmax = task.num("contacts.contact_rectangle.x_max"), xmin = task.num("contacts.contact_rectangle.x_min"),
               ymax = task.num("contacts.contact_rectangle.y_max"), ymin = task.num("contacts.contact_rectangle.y_min");
  std::vector<std::pair<int, V3>> frames;
  for (size_t c = 0; c < contactNames.size() && c < contactParents.size(); ++c) {
    const int b = jointIndex(contactParents[c]) + 1;
    frames.emplace_back(b, ct);
    frames.emplace_back(b, add(ct, V3{xmax * 0.6, 0, 0}));
    frames.emplace_back(b, add(ct, V3{xmin * 0.6, 0, 0}));
  }
  for (const char* key : {"foot.leftAnkleFrame", "foot.rightAnkleFrame", "knee.leftKneeFrame", "knee.rightKneeFrame"})
    frames.emplace_back(jointIndex(task.at(std::string("collision_constraint.") + key).value) + 1, V3{0, 0, 0});
  if (frames.size() > 16) throw std::invalid_argument("[b200sqp::host] too many frames");
  d.n_frames = static_cast<int32_t>(frames.size());
  for (size_t f = 0; f < frames.size(); ++f) {
    d.frame_body[f] = frames[f].first;
    d.frame_p[f][0] = frames[f].second.x;
    d.frame_p[f][1] = frames[f].second.y;
    d.frame_p[f][2] = frames[f].second.z;
  }
  d.gravity = 9.81;
  d.contact_rect[0] = xmin;
  d.contact_rect[1] = xmax;
  d.contact_rect[2] = ymin;
  d.contact_rect[3] = ymax;
  // ---- weights, gains, penalties -----------------------------------------------------------------------------------------------------------------
  const std::vector<double> Q = task.diagonal("Q", m.nx), R = task.diagonal("R", m.nu), Qf = task.diagonal("Q_final", m.nx);
  const double termScale = task.num("terminalCostScaling");
  for (int i = 0; i < m.nx; ++i) {
    d.Q_diag[i] = Q[i];
    d.Qf_diag[i] = Qf[i] * termScale;
  }
  for (int i = 0; i < m.nu; ++i) d.R_diag[i] = R[i];
  const std::string fc = "model_settings.foot_constraint.";
  d.foot_gain_pos_z = task.num(fc + "positionErrorGain_z");
  d.foot_gain_ori = task.num(fc + "orientationErrorGain");
  d.foot_gain_linvel_z = task.num(fc + "linearVelocityErrorGain_z");
  d.foot_gain_linvel_xy = task.num(fc + "linearVelocityErrorGain_xy");
  d.foot_gain_angvel = task.num(fc + "angularVelocityErrorGain");
  d.foot_gain_linacc_z = task.num(fc + "linearAccelerationErrorGain_z");
  d.foot_gain_linacc_xy = task.num(fc + "linearAccelerationErrorGain_xy");
  d.foot_gain_angacc = task.num(fc + "angularAccelerationErrorGain");
  // EndEffectorDynamicsWeights::getWeights (humanoid_wb_mpc/src/cost/EndEffectorDynamicsCostHelpers.cpp:97-110) overwrites the velocity weights with
  // the acceleration entries and leaves the acceleration weights at their defaults 0.01 (EndEffectorDynamicsCostHelpers.h:45-50): reproduced.
  const std::string w = "task_space_foot_cost_weights.";
  const char* axes[3] = {"x", "y", "z"};
  // EndEffectorKinematicsWeights::toVector (centroidal): position, orientation, linear velocity, angular velocity
  auto kinematicsWeights = [&](const std::string& prefix, double* out) {
    const char* kinds[4] = {"pos_", "orientation_", "lin_velocity_", "ang_velocity_"};
    for (int k = 0; k < 4; ++k)
      for (int a = 0; a < 3; ++a) out[3 * k + a] = task.num(prefix + kinds[k] + axes[a]);
  };
  if (centroidal) {
    kinematicsWeights(w, d.foot_cost_w);   // entries 12..17 stay zero
  } else {
    for (int a = 0; a < 3; ++a) {
      d.foot_cost_w[a] = task.num(w + "pos_" + axes[a]);
      d.foot_cost_w[3 + a] = task.num(w + "orientation_" + axes[a]);
      d.foot_cost_w[6 + a] = task.num(w + "lin_acceleration_" + axes[a]);
      d.foot_cost_w[9 + a] = task.num(w + "ang_acceleration_" + axes[a]);
      d.foot_cost_w[12 + a] = 0.01;
      d.foot_cost_w[15 + a] = 0.01;
    }
  }
  d.fric_coeff = task.num("contacts.frictionForceConeSoftConstraint.frictionCoefficient");
  d.fric_mu = task.num("contacts.frictionForceConeSoftConstraint.mu");
  d.fric_delta = task.num("contacts.frictionForceConeSoftConstraint.delta");
  d.fric_reg = 25.0;          // FrictionForceConeConstraint.h:66-69 defaults
  d.fric_hess_shift = 1e-6;
  d.momxy_mu = task.num("contacts.contactMomentXYSoftConstraint.mu");
  d.momxy_delta = task.num("contacts.contactMomentXYSoftConstraint.delta");
  d.jlim_mu = task.num("jointLimits.mu");
  d.jlim_delta = task.num("jointLimits.delta");
  d.coll_mu = task.num("collision_constraint.mu");
  d.coll_delta = task.num("collision_constraint.delta");
  d.coll_r_foot = task.num("collision_constraint.foot.footCollisionSphereRadius");
  d.coll_r_knee = task.num("collision_constraint.knee.kneeCollisionSphereRadius");
  const char* arms[4] = {"left_shoulder_y", "right_shoulder_y", "left_elbow_y", "right_elbow_y"};
  for (int i = 0; i < 4; ++i) d.arm_swing_joint[i] = jointIndex(task.at(std::string("model_settings.armJointNames.") + arms[i]).value);
  // ---- reference-manager parameters -----------------------------------------------------------------------------------------------------------
  m.initialState = task.column("initialState", m.nx);
  const std::string sw = "swing_trajectory_config.";
  m.swing = SwingTrajectoryConfig{task.num(sw + "liftOffVelocity"),
                                  task.num(sw + "touchDownVelocity"),
                                  task.num(sw + "swingHeight"),
                                  task.num(sw + "touchDownHeightOffset"),
                                  task.num(sw + "swingTimeScale"),
                                  task.num(sw + "impactProximityFactorLiftOffVelocity"),
                                  task.num(sw + "impactProximityFactorTouchDownVelocity"),
                                  task.num(sw + "impactProximityFactorMidPointValue")};
  m.dt = task.num("multiple_shooting.dt");
  m.timeHorizon = task.num("mpc.timeHorizon");
  b200sqp_default_settings(&m.sqpSettings);   // sqp::Settings defaults, then task.info:77-94
  m.sqpSettings.sqp_iteration = static_cast<int32_t>(task.num("multiple_shooting.sqpIteration"));
  m.sqpSettings.delta_tol = task.num("multiple_shooting.deltaTol");
  m.sqpSettings.g_max = task.num("multiple_shooting.g_max");
  m.sqpSettings.g_min = task.num("multiple_shooting.g_min");
  const Info ref = parseInfo(referenceFile);
  m.defaultBaseHeight = ref.num("defaultBaseHeight");
  m.maxDisplacementVelocityX = ref.num("maxDisplacementVelocityX");   // ProceduralMpcMotionManager.cpp:54-57
  m.maxDisplacementVelocityY = ref.num("maxDisplacementVelocityY");
  m.maxRotationVelocity = ref.num("maxRotationVelocity");
  m.targetDisplacementVelocity = ref.num("targetDisplacementVelocity");   // TargetTrajectoriesCalculatorBase's pose-command constants
  m.targetRotationVelocity = ref.num("targetRotationVelocity");
  m.maxDeltaPelvisHeight = ref.num("maxDeltaPelvisHeight");
  m.defaultJointState = ref.column("defaultJointState", m.nj);
  if (centroidal) {
    b200sqp_cen_desc& c = m.cen;
    std::memset(&c, 0, sizeof(c));
    // task_space_costs: one EndEffectorKinematicsQuadraticCost per listed link (CentroidalMpcInterface.cpp:331-362); the device path carries one
    const Info& costs = task.at("task_space_costs");
    if (costs.kids.size() != 1) throw std::invalid_argument("[b200sqp::host] exactly one task-space link cost is supported (G1: the torso)");
    const std::string cname = costs.kids.front().first;
    const auto lb = linkBody.find(costs.kids.front().second.at("link_name").value);
    if (lb == linkBody.end()) throw std::invalid_argument("[b200sqp::host] task-space cost link not in the URDF");
    if (d.n_frames >= 16) throw std::invalid_argument("[b200sqp::host] too many frames");
    c.torso_frame = d.n_frames;   // the task-space link rides as the last frame of the table
    d.frame_body[d.n_frames] = lb->second.body;
    d.frame_p[d.n_frames][0] = lb->second.p.x;
    d.frame_p[d.n_frames][1] = lb->second.p.y;
    d.frame_p[d.n_frames][2] = lb->second.p.z;
    d.n_frames += 1;
    for (int k = 0; k < 9; ++k) c.torso_R[k] = lb->second.R.m[k];
    kinematicsWeights("task_space_costs." + cname + ".weights.", c.torso_w);
    c.icp_weight = task.num("icp_cost_weights.icpErrorWeight");
    const char* sides[2] = {"left_leg_torque_cost", "right_leg_torque_cost"};   // ExternalTorqueQuadraticCostAD (HumanoidCostConstraintFactory.cpp:234-245)
    for (int sd = 0; sd < 2; ++sd) {
      const auto names = task.list(std::string(sides[sd]) + ".activeJointNames");
      if (names.size() != 6) throw std::invalid_argument("[b200sqp::host] leg torque cost: six active joints expected");
      const std::vector<double> wts = task.at(sides[sd]).column("weights", 6);
      for (int k = 0; k < 6; ++k) {
        c.torque_joint[sd][k] = jointIndex(names[k]);
        c.torque_w[sd][k] = wts[k];
      }
    }
    c.model_type = static_cast<int32_t>(task.num("centroidalModelType"));
    // createCentroidalModelInfo, SingleRigidBodyDynamics (ocs2_centroidal_model/src/FactoryFunctions.cpp:113-121): pinocchio::ccrba at
    // q = (0_6, nominal joint angles) -> rotational inertia about the centre of mass (base axes) and base - com
    std::vector<M3> Rw{eye()};
    std::vector<V3> pw{V3{0, 0, 0}};
    for (int i = 1; i <= m.nj; ++i) {
      const Body& b = bodies[i];
      const double th = m.defaultJointState[i - 1], sn = std::sin(th), cs = 1.0 - std::cos(th);
      const M3 K{{0, -b.axis.z, b.axis.y, b.axis.z, 0, -b.axis.x, -b.axis.y, b.axis.x, 0}};
      const M3 KK = mul(K, K);
      M3 Rq = eye();
      for (int k = 0; k < 9; ++k) Rq.m[k] += sn * K.m[k] + cs * KK.m[k];
      Rw.push_back(mul(mul(Rw[b.parent], b.R), Rq));
      pw.push_back(add(pw[b.parent], mul(Rw[b.parent], b.p)));
    }
    std::vector<V3> cw;
    V3 G{0, 0, 0};
    for (int i = 0; i <= m.nj; ++i) {
      cw.push_back(add(pw[i], mul(Rw[i], bodies[i].inertia.c)));
      G = add(G, V3{bodies[i].inertia.m * cw[i].x, bodies[i].inertia.m * cw[i].y, bodies[i].inertia.m * cw[i].z});
    }
    G = V3{G.x / m.totalMass, G.y / m.totalMass, G.z / m.totalMass};
    M3 Ig{{0, 0, 0, 0, 0, 0, 0, 0, 0}};
    for (int i = 0; i <= m.nj; ++i) {
      const M3 Iw = Inertia::shift(mul(mul(Rw[i], bodies[i].inertia.I), tr(Rw[i])), bodies[i].inertia.m, sub(cw[i], G));
      for (int k = 0; k < 9; ++k) Ig.m[k] += Iw.m[k];
    }
    for (int k = 0; k < 9; ++k) c.inertia_nominal[k] = Ig.m[k];
    c.com_to_base_nominal[0] = -G.x;
    c.com_to_base_nominal[1] = -G.y;
    c.com_to_base_nominal[2] = -G.z;
  }
  if (!gaitFile.empty()) {
    const Info g = parseInfo(gaitFile);
    for (const std::string& name : g.list("list")) {
      if (!g.find(name)) continue;
      GaitTemplate t;
      for (const std::string& mode : g.list(name + ".modeSequence")) t.modeSequence.push_back(modeFromString(mode));
      for (const std::string& v : g.list(name + ".switchingTimes")) t.switchingTimes.push_back(std::stod(v));
      m.gaits[name] = t;
    }
  }
  return m;
}

}  // namespace b200sqp::host
