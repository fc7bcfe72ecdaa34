// Scene-file front end: the subset of Mitsuba 0.6's SceneHandler (src/librender/scenehandler.cpp:70-106,
// 300-700) that describes the `path` hot path, parsed with expat and lowered onto the C-ABI (b2mts.h).
//
// Supported elements: scene, integrator(path, volpath, direct), sensor(perspective) with transform/sampler/film/rfilter,
// bsdf(diffuse | roughconductor | roughdielectric | coating) incl. id/ref, shape(obj | rectangle | cube) with
// toWorld transform, bsdf child / ref and emitter(area) child; property tags integer, float, boolean, string,
// rgb, srgb, spectrum (1 or 3 values), point, vector, transform{translate, rotate, scale, lookat, matrix},
// default, and $name substitution from `defines` (src/mitsuba/mitsuba.cpp:154 -D).
// Anything else is rejected with an error naming the element -- nothing is silently ignored.
#include "../../include/b2mts.h"
#include <expat.h>
#include <zlib.h>
#include "spectrum.h"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <sstream>
extern "C" const char *b2_data_dir_(void); // b2_host.cpp: <dir of libb2mts.so>/data or $B2MTS_DATA
#include <stdexcept>
#include <string>
#include <vector>

namespace {

struct M4 {
    double m[16];
    M4() { for (int i = 0; i < 16; ++i) m[i] = (i % 5 == 0) ? 1.0 : 0.0; }
    M4 operator*(const M4 &o) const {
        M4 r;
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) {
                double s = 0;
                for (int k = 0; k < 4; ++k) s += m[i * 4 + k] * o.m[k * 4 + j];
                r.m[i * 4 + j] = s;
            }
        return r;
    }
    void point(const double *p, double *o) const {
        for (int i = 0; i < 3; ++i) o[i] = m[i * 4] * p[0] + m[i * 4 + 1] * p[1] + m[i * 4 + 2] * p[2] + m[i * 4 + 3];
    }
    bool inverse(M4 &out) const {
        double a[4][8];
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) { a[i][j] = m[i * 4 + j]; a[i][4 + j] = i == j; }
        for (int c = 0; c < 4; ++c) {
            int piv = c;
            for (int r = c + 1; r < 4; ++r) if (std::fabs(a[r][c]) > std::fabs(a[piv][c])) piv = r;
            if (std::fabs(a[piv][c]) < 1e-300) return false;
            for (int j = 0; j < 8; ++j) std::swap(a[piv][j], a[c][j]);
            double d = a[c][c];
            for (int j = 0; j < 8; ++j) a[c][j] /= d;
            for (int r = 0; r < 4; ++r) if (r != c) { double f = a[r][c]; for (int j = 0; j < 8; ++j) a[r][j] -= f * a[c][j]; }
        }
        for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) out.m[i * 4 + j] = a[i][4 + j];
        return true;
    }
    // normals: inverse transpose (transform.h operator()(Normal))
    void normal(const M4 &inv, const double *n, double *o) const {
        for (int i = 0; i < 3; ++i) o[i] = inv.m[0 * 4 + i] * n[0] + inv.m[1 * 4 + i] * n[1] + inv.m[2 * 4 + i] * n[2];
    }
};

struct Value {
    enum Kind { Int, Float, Bool, String, Spectrum, Vec, Transform } kind = Float;
    double f = 0; long long i = 0; bool b = false; std::string s; double v[3] = {0, 0, 0}; M4 t;
};

struct Node {
    std::string tag, type, id, name;
    std::map<std::string, Value> props;
    std::vector<std::unique_ptr<Node>> children;
    Node *parent = nullptr;
    M4 xform;          // while parsing a <transform>
    bool queried(const std::string &) { return true; }
};

struct Err : std::runtime_error { using std::runtime_error::runtime_error; };

struct Parser {
    std::map<std::string, std::string> defines;
    std::unique_ptr<Node> root;
    Node *cur = nullptr;
    std::string baseDir;
    XML_Parser xp = nullptr;

    std::string subst(const std::string &s) { // scenehandler.cpp:214-236: $key replacement
        if (s.find('$') == std::string::npos) return s;
        std::string out = s;
        // longest keys first
        std::vector<std::pair<std::string, std::string>> kv(defines.begin(), defines.end());
        std::sort(kv.begin(), kv.end(), [](auto &a, auto &b) { return a.first.size() > b.first.size(); });
        for (auto &p : kv) {
            std::string key = "$" + p.first;
            size_t pos;
            while ((pos = out.find(key)) != std::string::npos) out.replace(pos, key.size(), p.second);
        }
        if (out.find('$') != std::string::npos) throw Err("The scene referenced an undefined parameter: \"" + out + "\"");
        return out;
    }
    static double toF(const std::string &s, const char *what) {
        char *end = nullptr;
        double v = strtod(s.c_str(), &end);
        if (end == s.c_str() || *end != '\0') throw Err(std::string("Could not parse floating point value \"") + s + "\" (" + what + ")");
        return v;
    }
    static std::vector<std::string> tokenize(const std::string &s, const char *delim = ", ") {
        std::vector<std::string> out;
        size_t i = 0;
        while (i < s.size()) {
            size_t j = s.find_first_of(delim, i);
            if (j == std::string::npos) j = s.size();
            if (j > i) out.push_back(s.substr(i, j - i));
            i = j + 1;
        }
        return out;
    }
    static void srgbToLinear(double *v) { // Spectrum::fromSRGB
        for (int i = 0; i < 3; ++i) v[i] = v[i] <= 0.04045 ? v[i] / 12.92 : std::pow((v[i] + 0.055) / 1.055, 2.4);
    }

    void start(const char *tagC, const char **atts) {
        std::string tag = tagC;
        std::map<std::string, std::string> a;
        for (int i = 0; atts[i]; i += 2) a[atts[i]] = subst(atts[i + 1]);
        auto need = [&](const char *k) -> const std::string & {
            auto it = a.find(k);
            if (it == a.end()) throw Err("<" + tag + ">: missing attribute '" + k + "'");
            return it->second;
        };
        auto opt = [&](const char *k, double dflt) { auto it = a.find(k); return it == a.end() || it->second.empty() ? dflt : toF(it->second, k); };
        if (tag == "default") { // scenehandler.cpp:646-652
            if (!defines.count(need("name"))) defines[need("name")] = need("value");
            return;
        }
        static const char *objects[] = {"scene", "integrator", "sensor", "sampler", "film", "rfilter", "bsdf", "shape", "emitter", "ref", "transform",
                                        "medium", "volume", "phase", "texture"};
        bool isObject = std::find_if(std::begin(objects), std::end(objects), [&](const char *o) { return tag == o; }) != std::end(objects);
        if (isObject) {
            auto n = std::make_unique<Node>();
            n->tag = tag; n->type = a.count("type") ? a["type"] : ""; n->id = a.count("id") ? a["id"] : ""; n->name = a.count("name") ? a["name"] : "";
            n->parent = cur;
            Node *raw = n.get();
            if (!cur) { if (tag != "scene") throw Err("root element must be <scene>"); root = std::move(n); }
            else cur->children.push_back(std::move(n));
            cur = raw;
            return;
        }
        if (!cur) throw Err("unexpected <" + tag + "> outside <scene>");
        // transform operations (scenehandler.cpp:348-441): each one is applied on the left
        if (cur->tag == "transform") {
            M4 op;
            if (tag == "translate") { op.m[3] = opt("x", 0); op.m[7] = opt("y", 0); op.m[11] = opt("z", 0); }
            else if (tag == "scale") {
                bool hasV = a.count("value") && !a["value"].empty();
                double x = hasV ? toF(a["value"], "scale") : opt("x", 1), y = hasV ? x : opt("y", 1), z = hasV ? x : opt("z", 1);
                op.m[0] = x; op.m[5] = y; op.m[10] = z;
            } else if (tag == "rotate") { // transform.cpp:65-98
                double ax[3] = {opt("x", 0), opt("y", 0), opt("z", 0)}, ang = toF(need("angle"), "angle") * M_PI / 180.0;
                double l = std::sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]);
                if (l == 0) throw Err("<rotate>: zero axis");
                for (double &c : ax) c /= l;
                double s = std::sin(ang), c = std::cos(ang);
                op.m[0] = ax[0] * ax[0] + (1 - ax[0] * ax[0]) * c; op.m[1] = ax[0] * ax[1] * (1 - c) - ax[2] * s; op.m[2] = ax[0] * ax[2] * (1 - c) + ax[1] * s;
                op.m[4] = ax[0] * ax[1] * (1 - c) + ax[2] * s; op.m[5] = ax[1] * ax[1] + (1 - ax[1] * ax[1]) * c; op.m[6] = ax[1] * ax[2] * (1 - c) - ax[0] * s;
                op.m[8] = ax[0] * ax[2] * (1 - c) - ax[1] * s; op.m[9] = ax[1] * ax[2] * (1 - c) + ax[0] * s; op.m[10] = ax[2] * ax[2] + (1 - ax[2] * ax[2]) * c;
            } else if (tag == "lookat") { // transform.cpp:191-214
                auto v3 = [&](const char *k, double *o, bool required) {
                    auto it = a.find(k);
                    if (it == a.end() || it->second.empty()) { if (required) throw Err(std::string("<lookat>: invalid '") + k + "' argument"); return false; }
                    auto t = tokenize(it->second);
                    if (t.size() != 3) throw Err(std::string("<lookat>: invalid '") + k + "' argument");
                    for (int i = 0; i < 3; ++i) o[i] = toF(t[i], k);
                    return true;
                };
                double o[3], t[3], u[3] = {0, 0, 0};
                v3("origin", o, true); v3("target", t, true); v3("up", u, false);
                double d[3] = {t[0] - o[0], t[1] - o[1], t[2] - o[2]};
                double l = std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
                if (l == 0) throw Err("lookAt(): 'origin' and 'target' coincide!");
                for (double &c : d) c /= l;
                if (u[0] == 0 && u[1] == 0 && u[2] == 0) { // arbitrary axis (scenehandler.cpp:392-396)
                    double c3[3];
                    if (std::fabs(d[0]) > std::fabs(d[1])) { double il = 1 / std::sqrt(d[0] * d[0] + d[2] * d[2]); c3[0] = d[2] * il; c3[1] = 0; c3[2] = -d[0] * il; }
                    else { double il = 1 / std::sqrt(d[1] * d[1] + d[2] * d[2]); c3[0] = 0; c3[1] = d[2] * il; c3[2] = -d[1] * il; }
                    u[0] = c3[1] * d[2] - c3[2] * d[1]; u[1] = c3[2] * d[0] - c3[0] * d[2]; u[2] = c3[0] * d[1] - c3[1] * d[0];
                }
                double left[3] = {u[1] * d[2] - u[2] * d[1], u[2] * d[0] - u[0] * d[2], u[0] * d[1] - u[1] * d[0]};
                l = std::sqrt(left[0] * left[0] + left[1] * left[1] + left[2] * left[2]);
                if (l == 0) throw Err("lookAt(): the forward and upward direction must be linearly independent!");
                for (double &c : left) c /= l;
                double nu[3] = {d[1] * left[2] - d[2] * left[1], d[2] * left[0] - d[0] * left[2], d[0] * left[1] - d[1] * left[0]};
                for (int i = 0; i < 3; ++i) { op.m[i * 4] = left[i]; op.m[i * 4 + 1] = nu[i]; op.m[i * 4 + 2] = d[i]; op.m[i * 4 + 3] = o[i]; }
            } else if (tag == "matrix") {
                auto t = tokenize(need("value"));
                if (t.size() != 16) throw Err("Invalid matrix specified");
                for (int i = 0; i < 16; ++i) op.m[i] = toF(t[i], "matrix");
            } else throw Err("unsupported transform operation <" + tag + ">");
            cur->xform = op * cur->xform;
            return;
        }
        // plain properties
        Value v;
        const std::string &pname = need("name");
        if (tag == "integer") { v.kind = Value::Int; v.i = (long long) toF(need("value"), "integer"); v.f = (double) v.i; }
        else if (tag == "float") { v.kind = Value::Float; v.f = toF(need("value"), "float"); }
        else if (tag == "boolean") {
            std::string b = need("value");
            std::transform(b.begin(), b.end(), b.begin(), ::tolower);
            if (b != "true" && b != "false") throw Err("Could not parse boolean value \"" + b + "\"");
            v.kind = Value::Bool; v.b = b == "true";
        } else if (tag == "string") { v.kind = Value::String; v.s = need("value"); }
        else if (tag == "rgb" || tag == "srgb" || tag == "spectrum") {
            v.kind = Value::Spectrum;
            if (tag == "spectrum" && a.count("filename")) { // scenehandler.cpp:557-568: InterpolatedSpectrum(path), zeroExtend, fromContinuousSpectrum, clampNegative
                if (a.count("value")) throw Err("<spectrum>: please provide one of 'value' or 'filename'");
                if (a.count("intent")) throw Err("<spectrum>: 'intent' and 'filename' cannot be specified at the same time!");
                std::string fn = a.at("filename");
                if (!fn.empty() && fn[0] != '/') fn = baseDir + "/" + fn;
                std::vector<double> wl, val;
                std::string err;
                float rgb[3];
                if (!b2host::readSpd(fn, wl, val, err) || !b2host::spectrumToRGB(wl, val, true, rgb, err)) throw Err(err);
                for (int i = 0; i < 3; ++i) v.v[i] = rgb[i];
                cur->props[pname] = v;
                return;
            }
            auto t = tokenize(need("value"));
            if (tag == "spectrum" && !t.empty() && t[0].find(':') != std::string::npos) { // wavelength:value pairs, scenehandler.cpp:594-611
                if (a.count("intent")) throw Err("<spectrum>: 'intent' can only be specified when given a single-valued argument.");
                std::vector<double> wl, val;
                for (const std::string &tok : t) {
                    auto pr = tokenize(tok, ":");
                    if (pr.size() != 2) throw Err("Invalid spectrum->value mapping specified");
                    wl.push_back(toF(pr[0], "spectrum")); val.push_back(toF(pr[1], "spectrum"));
                }
                std::string err;
                float rgb[3];
                if (!b2host::spectrumToRGB(wl, val, true, rgb, err)) throw Err(err);
                for (int i = 0; i < 3; ++i) v.v[i] = rgb[i];
                cur->props[pname] = v;
                return;
            }
            if (t.size() == 1 && t[0].size() == 7 && t[0][0] == '#' && tag != "spectrum") {
                long enc = strtol(t[0].c_str() + 1, nullptr, 16);
                v.v[0] = ((enc >> 16) & 0xFF) / 255.0; v.v[1] = ((enc >> 8) & 0xFF) / 255.0; v.v[2] = (enc & 0xFF) / 255.0;
            } else if (t.size() == 1) {
                v.v[0] = v.v[1] = v.v[2] = toF(t[0], "spectrum"); // reflectance: flat; illuminant: D65 == white in the RGB build
            } else if (t.size() == 3) { for (int i = 0; i < 3; ++i) v.v[i] = toF(t[i], "spectrum"); }
            else throw Err("Invalid spectrum value specified (length does not match the current spectral discretization!)");
            if (tag == "srgb") srgbToLinear(v.v);
        } else if (tag == "point" || tag == "vector") {
            v.kind = Value::Vec; v.v[0] = opt("x", 0); v.v[1] = opt("y", 0); v.v[2] = opt("z", 0);
        } else throw Err("unsupported element <" + tag + ">");
        cur->props[pname] = v;
    }
    void end(const char *tagC) {
        std::string tag = tagC;
        if (!cur || cur->tag != tag) return; // property / transform-op tags
        Node *n = cur;
        cur = n->parent;
        if (tag == "transform" && cur) {
            Value v; v.kind = Value::Transform; v.t = n->xform;
            cur->props[n->name.empty() ? "toWorld" : n->name] = v;
        }
    }
};

// exceptions must not unwind through expat's C frames: record the first error and stop the parser
std::string g_parseError;
void XMLCALL onStart(void *u, const char *t, const char **a) {
    Parser *P = (Parser *) u;
    try { P->start(t, a); } catch (const std::exception &e) { if (g_parseError.empty()) g_parseError = e.what(); XML_StopParser(P->xp, XML_FALSE); }
}
void XMLCALL onEnd(void *u, const char *t) {
    Parser *P = (Parser *) u;
    try { P->end(t); } catch (const std::exception &e) { if (g_parseError.empty()) g_parseError = e.what(); XML_StopParser(P->xp, XML_FALSE); }
}

// ---- property access with the reference's defaults and "unqueried property" discipline ----
struct Props {
    Node *n;
    std::map<std::string, bool> used;
    explicit Props(Node *n_) : n(n_) {}
    bool has(const std::string &k) const { return n->props.count(k) != 0; }
    double f(const std::string &k, double d) { used[k] = true; auto it = n->props.find(k); if (it == n->props.end()) return d; if (it->second.kind != Value::Float && it->second.kind != Value::Int) throw Err("property '" + k + "' has the wrong type"); return it->second.f; }
    long long i(const std::string &k, long long d) { used[k] = true; auto it = n->props.find(k); if (it == n->props.end()) return d; if (it->second.kind != Value::Int) throw Err("property '" + k + "' must be an integer"); return it->second.i; }
    bool b(const std::string &k, bool d) { used[k] = true; auto it = n->props.find(k); if (it == n->props.end()) return d; if (it->second.kind != Value::Bool) throw Err("property '" + k + "' must be a boolean"); return it->second.b; }
    std::string s(const std::string &k, const std::string &d) { used[k] = true; auto it = n->props.find(k); if (it == n->props.end()) return d; if (it->second.kind != Value::String) throw Err("property '" + k + "' must be a string"); return it->second.s; }
    void spec(const std::string &k, const double *d, float *out) { used[k] = true; auto it = n->props.find(k); const double *v = d; if (it != n->props.end()) { if (it->second.kind != Value::Spectrum) throw Err("property '" + k + "' must be a spectrum"); v = it->second.v; } for (int c = 0; c < 3; ++c) out[c] = (float) v[c]; }
    bool vec(const std::string &k, double *out) { used[k] = true; auto it = n->props.find(k); if (it == n->props.end()) return false; if (it->second.kind != Value::Vec) throw Err("property '" + k + "' must be a point"); for (int c = 0; c < 3; ++c) out[c] = it->second.v[c]; return true; }
    M4 xf(const std::string &k) { used[k] = true; auto it = n->props.find(k); return it == n->props.end() ? M4() : it->second.t; }
    void checkAllUsed() { // Properties "unqueried" check (src/libcore/plugin.cpp:185-196)
        for (auto &p : n->props) if (!used.count(p.first)) throw Err("<" + n->tag + " type=\"" + n->type + "\">: unreferenced property \"" + p.first + "\"");
    }
};

static double namedIOR(Props &p, const std::string &key, const char *dflt) { // src/bsdfs/ior.h:39-100
    static const std::map<std::string, double> table = {
        {"vacuum", 1.0}, {"helium", 1.000036}, {"hydrogen", 1.000132}, {"air", 1.000277}, {"carbon dioxide", 1.00045}, {"water", 1.3330},
        {"acetone", 1.36}, {"ethanol", 1.361}, {"carbon tetrachloride", 1.461}, {"glycerol", 1.4729}, {"benzene", 1.501}, {"silicone oil", 1.52045},
        {"bromine", 1.661}, {"water ice", 1.31}, {"fused quartz", 1.458}, {"pyrex", 1.470}, {"acrylic glass", 1.49}, {"polypropylene", 1.49},
        {"bk7", 1.5046}, {"sodium chloride", 1.544}, {"amber", 1.55}, {"pet", 1.5750}, {"diamond", 2.419}};
    p.used[key] = true;
    auto it = p.n->props.find(key);
    std::string name = dflt;
    if (it != p.n->props.end()) {
        if (it->second.kind == Value::Float || it->second.kind == Value::Int) return it->second.f;
        if (it->second.kind != Value::String) throw Err("property '" + key + "' must be a float or a material name");
        name = it->second.s;
    }
    std::transform(name.begin(), name.end(), name.begin(), ::tolower);
    auto t = table.find(name);
    if (t == table.end()) throw Err("Unable to find an IOR value for \"" + name + "\"");
    return t->second;
}

// util.cpp:807-859 fresnelDiffuseReflectance(eta, fast = false): integral over xi in [0,1] of F(sqrt(xi), eta), composite Simpson
static double fresnelDiffuseReflectance(double eta) {
    auto F = [eta](double cosI) { // util.cpp:651-681 for cosI >= 0
        if (eta == 1) return 0.0;
        const double scale = 1 / eta, ct2 = 1 - (1 - cosI * cosI) * scale * scale;
        if (ct2 <= 0) return 1.0;
        const double ct = std::sqrt(ct2), rs = (cosI - eta * ct) / (cosI + eta * ct), rp = (eta * cosI - ct) / (eta * cosI + ct);
        return 0.5 * (rs * rs + rp * rp);
    };
    const int n = 1 << 14;
    double acc = F(0.0) + F(1.0);
    for (int i = 1; i < n; ++i) acc += ((i & 1) ? 4.0 : 2.0) * F(std::sqrt((double) i / n));
    return acc / (3.0 * n);
}

struct Loader {
    b2_scene *scene = nullptr;
    std::map<std::string, int> bsdfIds; // id -> material id
    std::string baseDir;

    // material="<name>" of the conductor plugins (roughconductor.cpp:174-190): the RGB (eta, k) the reference derives from
    // data/ior/<name>.{eta,k}.spd, read from the table mitsuba_b200/data/conductor_presets.txt (generated with the reference's own
    // spectrum code by tools/extract_conductor_presets.py; hex floats)
    static bool conductorPreset(const std::string &material, double eta[3], double k[3]) {
        const char *dir = b2_data_dir_();
        std::ifstream f(std::string(dir ? dir : "data") + "/conductor_presets.txt");
        std::string line;
        while (std::getline(f, line)) {
            if (line.empty() || line[0] == '#') continue;
            std::istringstream is(line);
            std::string name, tok[6];
            is >> name >> tok[0] >> tok[1] >> tok[2] >> tok[3] >> tok[4] >> tok[5];
            if (name != material || !is) continue;
            for (int i = 0; i < 3; ++i) { eta[i] = strtod(tok[i].c_str(), nullptr); k[i] = strtod(tok[3 + i].c_str(), nullptr); }
            return true;
        }
        return false;
    }
    static void microfacet(Props &p, b2_material_desc &m) { // microfacet.h:95-148
        m.distr = B2_DISTR_BECKMANN; m.alpha_u = m.alpha_v = 0.1f;
        if (p.has("distribution")) {
            std::string d = p.s("distribution", "beckmann");
            std::transform(d.begin(), d.end(), d.begin(), ::tolower);
            if (d == "beckmann") m.distr = B2_DISTR_BECKMANN; else if (d == "ggx") m.distr = B2_DISTR_GGX; else if (d == "phong" || d == "as") m.distr = B2_DISTR_PHONG;
            else throw Err("Specified an invalid distribution \"" + d + "\", must be \"beckmann\", \"ggx\", or \"phong\"/\"as\"!");
        }
        if (p.has("alpha")) {
            if (p.has("alphaU") || p.has("alphaV")) throw Err("Microfacet model: please specify either 'alpha' or 'alphaU'/'alphaV'.");
            m.alpha_u = m.alpha_v = (float) p.f("alpha", 0.1);
        } else if (p.has("alphaU") || p.has("alphaV")) {
            if (!p.has("alphaU") || !p.has("alphaV")) throw Err("Microfacet model: both 'alphaU' and 'alphaV' must be specified.");
            m.alpha_u = (float) p.f("alphaU", 0.1); m.alpha_v = (float) p.f("alphaV", 0.1);
        }
        m.sample_visible = p.b("sampleVisible", true) ? 1 : 0;
        if (m.distr == B2_DISTR_PHONG) m.sample_visible = 0;
        // the plugins read the roughness as `m_alphaU->eval(its).average()` of a constant texture (roughconductor.cpp:273-274):
        // TSpectrum::average() = (a + a + a) * (1.0f / 3) in float (spectrum.h:481-486), which is not always a itself
        auto avg3 = [](float a) { volatile float r = 0.0f; r = r + a; r = r + a; r = r + a; return (float) (r * (1.0f / 3)); };
        m.alpha_u = avg3(m.alpha_u); m.alpha_v = avg3(m.alpha_v);
    }

    int addBsdf(Node *n) {
        Props p(n);
        b2_material_desc m;
        memset(&m, 0, sizeof(m));
        m.nested = -1; m.nested2 = -1; m.eta = 1.0f; m.thickness = 1.0f; m.sample_visible = 1; m.alpha_u = m.alpha_v = 0.1f;
        const double one[3] = {1, 1, 1}, zero[3] = {0, 0, 0}, half[3] = {0.5, 0.5, 0.5};
        for (int c = 0; c < 3; ++c) { m.transmittance[c] = 1; m.k_c[c] = 1; }
        if (n->type == "diffuse") {
            m.type = B2_BSDF_DIFFUSE;
            p.spec(p.has("reflectance") ? "reflectance" : "diffuseReflectance", half, m.reflectance); // diffuse.cpp:75-77
            for (auto &c : n->children) { // diffuse.cpp:191-200 addChild: a Texture named reflectance / diffuseReflectance
                const bool isTex = c->tag == "texture" || (c->tag == "ref" && textureIds.count(c->id));
                if (!isTex) continue;
                if (c->name != "reflectance" && c->name != "diffuseReflectance") throw Err("diffuse: texture child must be named 'reflectance' or 'diffuseReflectance'");
                m.reflectance_texture = 1 + (c->tag == "texture" ? addTexture(c.get()) : textureIds[c->id]);
            }
        } else if (n->type == "roughconductor") {
            m.type = B2_BSDF_ROUGHCONDUCTOR;
            p.spec("specularReflectance", one, m.reflectance);
            m.reflectance_texture = textureChild(n, "specularReflectance", "roughconductor");
            std::string material = p.s("material", "Cu");
            std::string lower = material;
            std::transform(lower.begin(), lower.end(), lower.begin(), ::tolower);
            double eta[3] = {0, 0, 0}, k[3] = {1, 1, 1};
            if (lower != "none" && !conductorPreset(material, eta, k) && !(p.has("eta") && p.has("k")))
                throw Err("roughconductor: unknown material preset \"" + material + "\" (data/ior/" + material + ".eta.spd); pass RGB 'eta' and 'k'");
            float fe[3], fk[3];
            p.spec("eta", eta, fe); p.spec("k", k, fk);
            float ext = (float) namedIOR(p, "extEta", "air");
            const float recip = 1.0f / ext; // Spectrum / Float multiplies by the reciprocal (spectrum.h:415-425)
            for (int c = 0; c < 3; ++c) { m.eta_c[c] = fe[c] * recip; m.k_c[c] = fk[c] * recip; } // roughconductor.cpp:189-190
            microfacet(p, m);
        } else if (n->type == "roughdielectric") {
            m.type = B2_BSDF_ROUGHDIELECTRIC;
            p.spec("specularReflectance", one, m.reflectance); p.spec("specularTransmittance", one, m.transmittance);
            float intI = (float) namedIOR(p, "intIOR", "bk7"), extI = (float) namedIOR(p, "extIOR", "air");
            if (intI < 0 || extI < 0 || intI == extI) throw Err("The interior and exterior indices of refraction must be positive and differ!");
            m.eta = intI / extI;
            microfacet(p, m);
        } else if (n->type == "coating") {
            m.type = B2_BSDF_COATING;
            float intI = (float) namedIOR(p, "intIOR", "bk7"), extI = (float) namedIOR(p, "extIOR", "air");
            if (intI < 0 || extI < 0 || intI == extI) throw Err("The interior and exterior indices of refraction must be positive and differ!");
            m.eta = intI / extI;
            m.thickness = (float) p.f("thickness", 1);
            p.spec("sigmaA", zero, m.sigma_a); p.spec("specularReflectance", one, m.reflectance);
            int nested = -1;
            for (auto &c : n->children) {
                if (c->tag == "bsdf") { if (nested >= 0) throw Err("Only a single nested BRDF can be added!"); nested = addBsdf(c.get()); }
                else if (c->tag == "ref") { if (nested >= 0) throw Err("Only a single nested BRDF can be added!"); nested = resolveRef(c.get()); }
            }
            if (nested < 0) throw Err("coating: A child BSDF instance is required");
            m.nested = nested;
        } else if (n->type == "twosided") { // twosided.cpp:186-197
            m.type = B2_BSDF_TWOSIDED;
            int kids[2] = {-1, -1}, nk = 0;
            for (auto &c : n->children) {
                if (c->tag != "bsdf" && c->tag != "ref") continue;
                if (nk == 2) throw Err("No more than two nested BRDFs can be added!");
                kids[nk++] = c->tag == "bsdf" ? addBsdf(c.get()) : resolveRef(c.get());
            }
            if (nk == 0) throw Err("A nested one-sided material is required!");
            m.nested = kids[0]; m.nested2 = nk == 2 ? kids[1] : kids[0];
        } else if (n->type == "dielectric") { // dielectric.cpp:145-162
            m.type = B2_BSDF_DIELECTRIC;
            p.spec("specularReflectance", one, m.reflectance); p.spec("specularTransmittance", one, m.transmittance);
            float intI = (float) namedIOR(p, "intIOR", "bk7"), extI = (float) namedIOR(p, "extIOR", "air");
            if (intI < 0 || extI < 0) throw Err("The interior and exterior indices of refraction must be positive!");
            m.eta = intI / extI;
        } else if (n->type == "conductor") { // conductor.cpp:153-176
            m.type = B2_BSDF_CONDUCTOR;
            p.spec("specularReflectance", one, m.reflectance);
            m.reflectance_texture = textureChild(n, "specularReflectance", "conductor");
            std::string material = p.s("material", "Cu");
            std::string lower = material;
            std::transform(lower.begin(), lower.end(), lower.begin(), ::tolower);
            double eta[3] = {0, 0, 0}, k[3] = {1, 1, 1};
            if (lower != "none" && !conductorPreset(material, eta, k) && !(p.has("eta") && p.has("k")))
                throw Err("conductor: unknown material preset \"" + material + "\" (data/ior/" + material + ".eta.spd); pass RGB 'eta' and 'k'");
            float fe[3], fk[3];
            p.spec("eta", eta, fe); p.spec("k", k, fk);
            float ext = (float) namedIOR(p, "extEta", "air");
            const float recip = 1.0f / ext; // Spectrum / Float multiplies by the reciprocal (spectrum.h:415-425)
            for (int c = 0; c < 3; ++c) { m.eta_c[c] = fe[c] * recip; m.k_c[c] = fk[c] * recip; }
        } else if (n->type == "plastic") { // plastic.cpp:145-204
            m.type = B2_BSDF_PLASTIC;
            float intI = (float) namedIOR(p, "intIOR", "polypropylene"), extI = (float) namedIOR(p, "extIOR", "air");
            if (intI < 0 || extI < 0) throw Err("The interior and exterior indices of refraction must be positive!");
            m.eta = intI / extI;
            p.spec("specularReflectance", one, m.reflectance); p.spec("diffuseReflectance", half, m.diffuse_reflectance);
            m.nonlinear = p.b("nonlinear", false) ? 1 : 0;
            m.fdr_int = (float) fresnelDiffuseReflectance(1.0 / m.eta); m.fdr_ext = (float) fresnelDiffuseReflectance(m.eta);
            auto lum = [](const float *c) { return c[0] * 0.212671f + c[1] * 0.715160f + c[2] * 0.072169f; }; // spectrum.h:725-727
            float dAvg = lum(m.diffuse_reflectance);
            for (auto &c : n->children) { // plastic.cpp:217-230 addChild: a Texture named diffuseReflectance
                const bool isTex = c->tag == "texture" || (c->tag == "ref" && textureIds.count(c->id));
                if (!isTex) continue;
                if (c->name != "diffuseReflectance") throw Err("plastic: bitmap textures are supported on 'diffuseReflectance' only");
                const int tid = c->tag == "texture" ? addTexture(c.get()) : textureIds[c->id];
                m.reflectance_texture = 1 + tid;
                dAvg = textureAvgLum[tid]; // m_diffuseReflectance->getAverage().getLuminance(), plastic.cpp:199
            }
            const float sAvg = lum(m.reflectance);
            m.spec_sampling_weight = sAvg / (dAvg + sAvg);
        } else throw Err("unsupported BSDF plugin \"" + n->type + "\" (supported: diffuse, roughconductor, roughdielectric, coating, twosided, dielectric, conductor, plastic)");
        p.checkAllUsed();
        int id = b2_scene_add_material(scene, &m);
        if (id < 0) throw Err(b2_last_error(nullptr));
        if (!n->id.empty()) bsdfIds[n->id] = id;
        return id;
    }
    // ---- bitmap textures (SURVEY.md 8f-4) ----
    std::map<std::string, int> textureIds;
    std::vector<float> textureAvgLum; // per texture id: luminance of its average (what plastic's specular sampling weight reads)
    // Bitmap::readPFM (bitmap.cpp:3764-3814) and Bitmap::readPPM (:3857-3895, 8-bit P6), then Bitmap::convert(.., EFloat32, gamma 1)
    // as TMIPMap's constructor applies it (mipmap.h:225-226; fmtconv.cpp:1092-1101,1136-1147): linear float, top row first
    // OpenEXR scan-line images (Bitmap::readOpenEXR, bitmap.cpp, goes through the OpenEXR library; this is a reader of the published file
    // layout): single-part, flat, not tiled; channels R, G, B (others ignored) or a lone Y / single channel; HALF, FLOAT or UINT samples;
    // compression NONE, RLE, ZIPS or ZIP (what Mitsuba's own hdrfilm writes).  PIZ / PXR24 / B44 / DWA files are refused by name.
    static float halfBitsToFloat(uint16_t hb) {
        const uint32_t sign = (uint32_t) (hb & 0x8000u) << 16, exp = (hb >> 10) & 0x1Fu, man = hb & 0x3FFu;
        uint32_t bits;
        if (exp == 0) {
            if (man == 0) bits = sign;
            else { // denormal: normalise
                int e = -1; uint32_t m = man;
                do { ++e; m <<= 1; } while (!(m & 0x400u));
                bits = sign | ((uint32_t) (127 - 15 - e) << 23) | ((m & 0x3FFu) << 13);
            }
        } else if (exp == 31) bits = sign | 0x7F800000u | (man << 13);
        else bits = sign | ((exp + 112u) << 23) | (man << 13);
        float r; memcpy(&r, &bits, 4);
        return r;
    }
    static void loadOpenEXR(const std::string &path, int &w, int &h, int &ch, std::vector<float> &px) {
        std::ifstream f(path, std::ios::binary);
        std::vector<unsigned char> d((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        size_t pos = 8;
        auto need = [&](size_t n) { if (pos + n > d.size()) throw Err("readOpenEXR(): \"" + path + "\" is truncated"); };
        auto i32 = [&](size_t at) { int32_t v; memcpy(&v, &d[at], 4); return v; };
        if (d.size() < 8) throw Err("readOpenEXR(): \"" + path + "\" is truncated");
        const uint32_t version = (uint32_t) i32(4);
        if ((version & 0xFFu) != 2) throw Err("readOpenEXR(): unsupported file version");
        if (version & 0x200u) throw Err("readOpenEXR(): tiled images are not supported (\"" + path + "\")");
        if (version & 0x1800u) throw Err("readOpenEXR(): deep / multi-part images are not supported (\"" + path + "\")");
        struct Chan { std::string name; int type; size_t offset; }; // offset of the channel's samples inside one scan line
        std::vector<Chan> chans;
        int compression = -1, xMin = 0, yMin = 0, xMax = -1, yMax = -1;
        auto cstr = [&]() { std::string t; while (true) { need(1); const char c = (char) d[pos++]; if (!c) break; t += c; } return t; };
        while (true) { // attributes: name\0 type\0 size value
            const std::string name = cstr();
            if (name.empty()) break;
            const std::string type = cstr();
            need(4);
            const int32_t size = i32(pos); pos += 4;
            if (size < 0) throw Err("readOpenEXR(): corrupt header");
            need((size_t) size);
            const size_t end = pos + (size_t) size;
            if (name == "channels") {
                while (pos < end && d[pos]) {
                    Chan c; c.name = cstr();
                    need(16);
                    c.type = i32(pos);
                    if (i32(pos + 8) != 1 || i32(pos + 12) != 1) throw Err("readOpenEXR(): sub-sampled channels are not supported");
                    if (c.type < 0 || c.type > 2) throw Err("readOpenEXR(): unknown pixel type");
                    pos += 16;
                    c.offset = 0;
                    chans.push_back(c);
                }
            } else if (name == "compression" && size >= 1) compression = d[pos];
            else if (name == "dataWindow" && size >= 16) { xMin = i32(pos); yMin = i32(pos + 4); xMax = i32(pos + 8); yMax = i32(pos + 12); }
            pos = end;
        }
        w = xMax - xMin + 1; h = yMax - yMin + 1;
        if (w <= 0 || h <= 0 || chans.empty() || compression < 0) throw Err("readOpenEXR(): incomplete header in \"" + path + "\"");
        static const char *cname[] = {"NONE", "RLE", "ZIPS", "ZIP", "PIZ", "PXR24", "B44", "B44A", "DWAA", "DWAB"};
        if (compression > 3) throw Err(std::string("readOpenEXR(): ") + (compression < 10 ? cname[compression] : "this") + " compression is not supported (supported: NONE, RLE, ZIPS, ZIP); re-save \"" + path + "\" with ZIP compression");
        const int linesPerBlock = compression == 3 ? 16 : 1;
        size_t lineBytes = 0;
        for (Chan &c : chans) { c.offset = lineBytes; lineBytes += (size_t) w * (c.type == 1 ? 2 : 4); } // the list is stored in alphabetical order = file order
        int src[3] = {-1, -1, -1};
        for (size_t k = 0; k < chans.size(); ++k) {
            if (chans[k].name == "R") src[0] = (int) k; else if (chans[k].name == "G") src[1] = (int) k; else if (chans[k].name == "B") src[2] = (int) k;
        }
        if (src[0] >= 0 && src[1] >= 0 && src[2] >= 0) ch = 3;
        else {
            ch = 1; src[0] = -1;
            for (size_t k = 0; k < chans.size(); ++k) if (chans[k].name == "Y") src[0] = (int) k;
            if (src[0] < 0 && chans.size() == 1) src[0] = 0;
            if (src[0] < 0) throw Err("readOpenEXR(): \"" + path + "\" has neither R, G, B nor a luminance channel");
        }
        px.assign((size_t) w * h * ch, 0.0f);
        const int nBlocks = (h + linesPerBlock - 1) / linesPerBlock;
        need((size_t) nBlocks * 8);
        const size_t table = pos;
        std::vector<unsigned char> raw, tmp;
        for (int b = 0; b < nBlocks; ++b) {
            uint64_t off; memcpy(&off, &d[table + (size_t) b * 8], 8);
            if (off + 8 > d.size()) throw Err("readOpenEXR(): \"" + path + "\" is truncated");
            const int y0 = i32((size_t) off) - yMin, dataSize = i32((size_t) off + 4);
            if (y0 < 0 || y0 >= h || dataSize < 0 || off + 8 + (uint64_t) dataSize > d.size()) throw Err("readOpenEXR(): corrupt chunk in \"" + path + "\"");
            const int lines = std::min(linesPerBlock, h - y0);
            const size_t expect = lineBytes * (size_t) lines;
            const unsigned char *in = &d[(size_t) off + 8];
            raw.resize(expect);
            if ((size_t) dataSize == expect || compression == 0) { // stored as is (also what the compressors fall back to when they do not shrink the block)
                if ((size_t) dataSize != expect) throw Err("readOpenEXR(): chunk size mismatch");
                memcpy(raw.data(), in, expect);
            } else {
                tmp.resize(expect);
                if (compression == 1) { // run-length: n >= 0: the next byte n + 1 times; n < 0: -n literal bytes
                    size_t o = 0, i = 0;
                    while (i < (size_t) dataSize) {
                        const int n = (signed char) in[i++];
                        if (n < 0) { const size_t c = (size_t) -n; if (i + c > (size_t) dataSize || o + c > expect) throw Err("readOpenEXR(): corrupt RLE data"); memcpy(&tmp[o], in + i, c); i += c; o += c; }
                        else { const size_t c = (size_t) n + 1; if (i >= (size_t) dataSize || o + c > expect) throw Err("readOpenEXR(): corrupt RLE data"); memset(&tmp[o], in[i++], c); o += c; }
                    }
                    if (o != expect) throw Err("readOpenEXR(): corrupt RLE data");
                } else {
                    uLongf got = (uLongf) expect;
                    if (uncompress(tmp.data(), &got, in, (uLong) dataSize) != Z_OK || got != expect) throw Err("readOpenEXR(): corrupt zlib data in \"" + path + "\"");
                }
                for (size_t i = 1; i < expect; ++i) tmp[i] = (unsigned char) (tmp[i - 1] + tmp[i] - 128); // byte-delta predictor
                const size_t half = (expect + 1) / 2;                                                     // then the two interleaved halves
                for (size_t i = 0; i < half; ++i) { raw[2 * i] = tmp[i]; if (2 * i + 1 < expect) raw[2 * i + 1] = tmp[half + i]; }
            }
            for (int l = 0; l < lines; ++l)
                for (int c = 0; c < ch; ++c) {
                    const Chan &cn = chans[src[c]];
                    const unsigned char *row = raw.data() + (size_t) l * lineBytes + cn.offset;
                    float *out = &px[((size_t) (y0 + l) * w) * ch + c];
                    for (int x = 0; x < w; ++x) {
                        float v;
                        if (cn.type == 1) { uint16_t hb; memcpy(&hb, row + 2 * (size_t) x, 2); v = halfBitsToFloat(hb); }
                        else if (cn.type == 2) memcpy(&v, row + 4 * (size_t) x, 4);
                        else { uint32_t u; memcpy(&u, row + 4 * (size_t) x, 4); v = (float) u; }
                        out[(size_t) x * ch] = v;
                    }
                }
        }
    }
    // PNG (Bitmap::readPNG, bitmap.cpp:2465-2555, goes through libpng; this is a reader of the published format on top of zlib): non-interlaced,
    // 8- or 16-bit grey / grey+alpha / RGB / RGBA, 2-, 4- and 8-bit palettes and 2- / 4-bit grey expanded to 8 bits; alpha is dropped (bitmap.cpp:
    // 270-275); the file's gamma is the sRGB curve unless a gAMA chunk (without an sRGB chunk) says otherwise (:2534-2541).  Returns that gamma.
    static double loadPNG(const std::string &path, int &w, int &h, int &ch, std::vector<float> &px) {
        std::ifstream f(path, std::ios::binary);
        std::vector<unsigned char> d((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        auto be32 = [&](size_t at) { return ((uint32_t) d[at] << 24) | ((uint32_t) d[at + 1] << 16) | ((uint32_t) d[at + 2] << 8) | (uint32_t) d[at + 3]; };
        size_t pos = 8;
        int depth = 0, ctype = -1, interlace = 0;
        bool haveSRGB = false, haveGamma = false;
        double fileGamma = 0;
        std::vector<unsigned char> idat, palette;
        w = h = 0;
        while (pos + 12 <= d.size()) {
            const uint32_t len = be32(pos);
            const std::string type((const char *) &d[pos + 4], 4);
            const size_t body = pos + 8;
            if (body + (size_t) len + 4 > d.size()) throw Err("readPNG(): \"" + path + "\" is truncated");
            if (type == "IHDR" && len >= 13) {
                w = (int) be32(body); h = (int) be32(body + 4); depth = d[body + 8]; ctype = d[body + 9]; interlace = d[body + 12];
                if (d[body + 10] != 0 || d[body + 11] != 0) throw Err("readPNG(): unknown compression / filter method");
            } else if (type == "PLTE") palette.assign(d.begin() + (long) body, d.begin() + (long) (body + len));
            else if (type == "IDAT") idat.insert(idat.end(), d.begin() + (long) body, d.begin() + (long) (body + len));
            else if (type == "sRGB") haveSRGB = true;
            else if (type == "gAMA" && len >= 4) { haveGamma = true; fileGamma = be32(body) / 100000.0; }
            else if (type == "IEND") break;
            pos = body + len + 4;
        }
        if (w <= 0 || h <= 0 || idat.empty()) throw Err("readPNG(): \"" + path + "\" holds no image");
        if (interlace != 0) throw Err("readPNG(): interlaced files are not supported (\"" + path + "\")");
        int nch;
        switch (ctype) { case 0: nch = 1; break; case 2: nch = 3; break; case 3: nch = 1; break; case 4: nch = 2; break; case 6: nch = 4; break; default: throw Err("readPNG(): Unknown color type"); }
        const bool okDepth = ctype == 3 ? (depth == 2 || depth == 4 || depth == 8) : ctype == 0 ? (depth == 2 || depth == 4 || depth == 8 || depth == 16) : (depth == 8 || depth == 16);
        if (!okDepth) throw Err("readPNG(): Unsupported bit depth: " + std::to_string(depth));
        if (ctype == 3 && palette.size() < 3) throw Err("readPNG(): palette image without a palette");
        const size_t rowBytes = ((size_t) w * nch * depth + 7) / 8, bpp = std::max<size_t>(1, (size_t) nch * depth / 8);
        std::vector<unsigned char> raw((rowBytes + 1) * (size_t) h);
        uLongf got = (uLongf) raw.size();
        if (uncompress(raw.data(), &got, idat.data(), (uLong) idat.size()) != Z_OK || got != raw.size()) throw Err("readPNG(): corrupt image data in \"" + path + "\"");
        std::vector<unsigned char> prev(rowBytes, 0), cur(rowBytes);
        ch = (ctype == 0 || ctype == 4) ? 1 : 3;
        px.assign((size_t) w * h * ch, 0.0f);
        const float s8 = 1.0f / 255.0f, s16 = 1.0f / 65535.0f; // fmtconv: unsigned integer samples -> [0, 1]
        for (int y = 0; y < h; ++y) {
            const unsigned char *in = &raw[(size_t) y * (rowBytes + 1)];
            const int filter = in[0];
            for (size_t i = 0; i < rowBytes; ++i) {
                const int a = i >= bpp ? cur[i - bpp] : 0, b = prev[i], c = i >= bpp ? prev[i - bpp] : 0;
                int pred = 0;
                switch (filter) {
                    case 0: pred = 0; break;
                    case 1: pred = a; break;
                    case 2: pred = b; break;
                    case 3: pred = (a + b) >> 1; break;
                    case 4: { const int p = a + b - c, pa = std::abs(p - a), pb = std::abs(p - b), pc = std::abs(p - c); pred = (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c); break; }
                    default: throw Err("readPNG(): corrupt image data in \"" + path + "\"");
                }
                cur[i] = (unsigned char) (in[1 + i] + pred);
            }
            float *out = &px[(size_t) y * w * ch];
            for (int x = 0; x < w; ++x) {
                if (ctype == 3 || (ctype == 0 && depth < 8)) { // packed indices / packed grey
                    const int perByte = 8 / depth, shift = (perByte - 1 - x % perByte) * depth, v = depth == 8 ? cur[x] : (cur[x / perByte] >> shift) & ((1 << depth) - 1);
                    if (ctype == 3) {
                        if ((size_t) v * 3 + 2 >= palette.size()) throw Err("readPNG(): palette index out of range");
                        for (int c = 0; c < 3; ++c) out[3 * x + c] = (float) palette[(size_t) v * 3 + c] * s8;
                    } else out[x] = (float) (v * (255 / ((1 << depth) - 1))) * s8; // png_set_expand_gray_1_2_4_to_8
                } else if (depth == 8) {
                    for (int c = 0; c < ch; ++c) out[(size_t) x * ch + c] = (float) cur[(size_t) x * nch + c] * s8;
                } else {
                    for (int c = 0; c < ch; ++c) { const size_t at = ((size_t) x * nch + c) * 2; out[(size_t) x * ch + c] = (float) (((unsigned) cur[at] << 8) | cur[at + 1]) * s16; }
                }
            }
            prev.swap(cur);
        }
        if (haveSRGB || !haveGamma) return -1.0;
        return (double) (1.0f / (float) fileGamma);
    }
    static void loadImage(const std::string &path, double gammaOverride, int &w, int &h, int &ch, std::vector<float> &px) {
        std::ifstream f(path, std::ios::binary);
        if (!f) throw Err("bitmap: cannot open \"" + path + "\"");
        {
            unsigned char m4[4] = {0, 0, 0, 0};
            f.read((char *) m4, 4);
            if (f.gcount() == 4 && m4[0] == 0x76 && m4[1] == 0x2f && m4[2] == 0x31 && m4[3] == 0x01) { // OpenEXR magic 20000630
                f.close();
                loadOpenEXR(path, w, h, ch, px);
                const double g = gammaOverride != 0 ? gammaOverride : 1.0; // the file is linear; a `gamma` property overrides that (bitmap.cpp:251-252)
                if (g == -1.0) { for (float &v : px) v = v <= 0.04045f ? v * (float) (1.0 / 12.92) : std::pow((float) ((v + 0.055f) * (float) (1.0 / 1.055)), 2.4f); }
                else if (g != 1.0) for (float &v : px) v = std::pow(v, (float) g);
                return;
            }
            unsigned char m8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            f.clear(); f.seekg(0);
            f.read((char *) m8, 8);
            static const unsigned char pngMagic[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
            if (f.gcount() == 8 && memcmp(m8, pngMagic, 8) == 0) {
                f.close();
                double g = loadPNG(path, w, h, ch, px);
                if (gammaOverride != 0) g = gammaOverride; // bitmap.cpp:251-252
                if (g == -1.0) { for (float &v : px) v = v <= 0.04045f ? v * (float) (1.0 / 12.92) : std::pow((float) ((v + 0.055f) * (float) (1.0 / 1.055)), 2.4f); }
                else if (g != 1.0) for (float &v : px) v = std::pow(v, (float) g);
                return;
            }
            f.clear(); f.seekg(0);
        }
        auto token = [&]() { std::string t; char c; while (f.get(c)) { if (c == ' ' || c == '\t' || c == '\n' || c == '\r') { if (!t.empty()) break; } else t += c; } return t; };
        const std::string magic = token();
        double gamma; // bitmap gamma: -1 = sRGB curve
        if (magic == "PF" || magic == "Pf") {
            ch = magic == "PF" ? 3 : 1;
            w = atoi(token().c_str()); h = atoi(token().c_str());
            const double scaleAndOrder = strtod(token().c_str(), nullptr);
            if (w <= 0 || h <= 0 || scaleAndOrder == 0) throw Err("readPFM(): Invalid header!");
            px.resize((size_t) w * h * ch);
            f.read((char *) px.data(), (std::streamsize) (px.size() * 4));
            if (!f) throw Err("readPFM(): file is truncated");
            if (scaleAndOrder > 0) // big endian
                for (float &v : px) { unsigned char *b = (unsigned char *) &v; std::swap(b[0], b[3]); std::swap(b[1], b[2]); }
            const float scale = (float) std::fabs(scaleAndOrder);
            if (scale != 1) for (float &v : px) v *= scale;
            for (int y = 0; y < h / 2; ++y) // flipVertically: PFM stores the bottom row first
                std::swap_ranges(px.begin() + (size_t) y * w * ch, px.begin() + (size_t) (y + 1) * w * ch, px.begin() + (size_t) (h - 1 - y) * w * ch);
            gamma = 1.0;
        } else if (magic == "P6") {
            ch = 3;
            w = atoi(token().c_str()); h = atoi(token().c_str());
            const int maxVal = atoi(token().c_str());
            if (w <= 0 || h <= 0 || maxVal <= 0) throw Err("readPPM(): unable to parse the file header!");
            if (maxVal > 0xFF) throw Err("readPPM(): 16-bit PPM files are not supported");
            std::vector<unsigned char> raw((size_t) w * h * 3);
            f.read((char *) raw.data(), (std::streamsize) raw.size());
            if (!f) throw Err("readPPM(): file is truncated");
            px.resize(raw.size());
            for (size_t i = 0; i < raw.size(); ++i) px[i] = (float) raw[i] * (1.0f / 255.0f);
            gamma = -1.0;
        } else if (magic.size() >= 2 && magic[0] == '#' && magic[1] == '?') {
            // Radiance RGBE (.hdr / .pic), Bitmap::readRGBE (bitmap.cpp:3590-3689): text header up to the "-Y h +X w" line, then either flat
            // 4-byte pixels or per-scanline run-length coding of the four byte planes; value = mantissa * 2^(e - 136) (:3522-3530)
            f.seekg(0);
            std::vector<unsigned char> file((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
            size_t pos = 0;
            auto line = [&]() { std::string t; while (pos < file.size() && file[pos] != '\n') t += (char) file[pos++]; ++pos; return t; };
            line();
            bool knownFormat = false;
            w = h = 0;
            while (pos < file.size()) {
                const std::string l = line();
                if (l.compare(0, 22, "FORMAT=32-bit_rle_rgbe") == 0) knownFormat = true;
                if (l.compare(0, 3, "-Y ") == 0) {
                    if (sscanf(l.c_str(), "-Y %i +X %i", &h, &w) < 2) throw Err("readRGBE(): parser error!");
                    break;
                }
            }
            if (!knownFormat) throw Err("readRGBE(): invalid format!");
            if (w <= 0 || h <= 0) throw Err("readRGBE(): parser error!");
            ch = 3;
            px.assign((size_t) w * h * 3, 0.0f);
            auto need = [&](size_t n) { if (pos + n > file.size()) throw Err("readRGBE(): file is truncated"); };
            auto decode = [](const unsigned char *q, float *o) {
                if (q[3]) { const float m = std::ldexp(1.0f, (int) q[3] - 136); o[0] = q[0] * m; o[1] = q[1] * m; o[2] = q[2] * m; }
                else o[0] = o[1] = o[2] = 0.0f;
            };
            auto flat = [&](size_t firstPixel) { // the rest of the file is uncompressed
                const size_t n = (size_t) w * h - firstPixel;
                need(4 * n);
                for (size_t k = 0; k < n; ++k, pos += 4) decode(&file[pos], &px[3 * (firstPixel + k)]);
            };
            if (w < 8 || w > 0x7fff) flat(0);
            else {
                std::vector<unsigned char> planes((size_t) 4 * w);
                for (int y = 0; y < h; ++y) {
                    need(4);
                    const unsigned char *hd = &file[pos];
                    if (hd[0] != 2 || hd[1] != 2 || (hd[2] & 0x80)) { // no scanline marker: the file is flat from here on (only legal in row 0)
                        flat((size_t) y * w);
                        break;
                    }
                    if ((((int) hd[2]) << 8 | hd[3]) != w) throw Err("readRGBE(): wrong scanline width!");
                    pos += 4;
                    for (int c = 0; c < 4; ++c) {
                        unsigned char *out = &planes[(size_t) c * w], *end = out + w;
                        while (out < end) {
                            need(2);
                            int count = file[pos];
                            if (count > 128) { // run
                                count -= 128;
                                if (count > end - out) throw Err("readRGBE(): bad scanline data!");
                                std::fill(out, out + count, file[pos + 1]);
                                pos += 2;
                            } else { // literal bytes
                                if (count == 0 || count > end - out) throw Err("readRGBE(): bad scanline data!");
                                need(1 + (size_t) count);
                                std::copy(&file[pos + 1], &file[pos + 1] + count, out);
                                pos += 1 + (size_t) count;
                            }
                            out += count;
                        }
                    }
                    for (int x = 0; x < w; ++x) {
                        const unsigned char q[4] = {planes[x], planes[(size_t) w + x], planes[(size_t) 2 * w + x], planes[(size_t) 3 * w + x]};
                        decode(q, &px[3 * ((size_t) y * w + x)]);
                    }
                }
            }
            gamma = 1.0;
        } else throw Err("bitmap: unsupported image format in \"" + path + "\" (supported: OpenEXR scan-line NONE / RLE / ZIP, PNG, PFM, Radiance RGBE, 8-bit binary PPM)");
        if (gammaOverride != 0) gamma = gammaOverride; // bitmap.cpp:251-252
        if (gamma == -1.0) {
            for (float &v : px) v = v <= 0.04045f ? v * (float) (1.0 / 12.92) : std::pow((float) ((v + 0.055f) * (float) (1.0 / 1.055)), 2.4f);
        } else if (gamma != 1.0) {
            for (float &v : px) v = std::pow(v, (float) gamma);
        }
    }
    // <emitter type="envmap"> (src/emitters/envmap.cpp:106-181): filename, scale, toWorld, gamma, samplingWeight; `cache` is accepted and
    // ignored (MIP map cache files are neither read nor written: the pyramid is rebuilt at commit)
    void addEnvMap(Node *n) {
        Props p(n);
        std::string fn = p.s("filename", "");
        if (fn.empty()) throw Err("envmap: 'filename' is required");
        if (fn[0] != '/') fn = baseDir + "/" + fn;
        if (p.has("intensityScale")) throw Err("The 'intensityScale' parameter has been deprecated and is now called scale."); // envmap.cpp:177-178
        const double gamma = p.f("gamma", 0);
        const float scale = (float) p.f("scale", 1.0);
        const float weight = (float) p.f("samplingWeight", 1.0);
        p.b("cache", false);
        M4 tw = p.xf("toWorld"), inv;
        if (!tw.inverse(inv)) throw Err("envmap: singular toWorld transform");
        p.checkAllUsed();
        int w, h, ch;
        std::vector<float> px;
        loadImage(fn, gamma, w, h, ch, px);
        if (ch == 1) { // luminance image -> RGB (Bitmap::convert to ERGB)
            std::vector<float> rgb((size_t) w * h * 3);
            for (size_t k = 0; k < (size_t) w * h; ++k) rgb[3 * k] = rgb[3 * k + 1] = rgb[3 * k + 2] = px[k];
            px.swap(rgb);
        }
        float a[16], b[16];
        for (int i = 0; i < 16; ++i) { a[i] = (float) tw.m[i]; b[i] = (float) inv.m[i]; }
        if (b2_scene_add_envmap_emitter(scene, w, h, px.data(), scale, a, b, weight) < 0) throw Err(b2_last_error(nullptr));
    }
    // a Texture child (or reference) named `name` of BSDF node n -> reflectance_texture binding (0 = none)
    int textureChild(Node *n, const char *name, const char *plugin) {
        int bound = 0;
        for (auto &c : n->children) {
            const bool isTex = c->tag == "texture" || (c->tag == "ref" && textureIds.count(c->id));
            if (!isTex) continue;
            if (c->name != name) throw Err(std::string(plugin) + ": bitmap textures are supported on '" + name + "' only");
            bound = 1 + (c->tag == "texture" ? addTexture(c.get()) : textureIds[c->id]);
        }
        return bound;
    }
    int addTexture(Node *n) {
        if (n->type != "bitmap") throw Err("unsupported texture plugin \"" + n->type + "\" (supported: bitmap)");
        Props p(n);
        std::string fn = p.s("filename", "");
        if (fn.empty()) throw Err("bitmap: 'filename' is required");
        if (fn[0] != '/') fn = baseDir + "/" + fn;
        if (!p.s("channel", "").empty()) throw Err("bitmap: the 'channel' parameter is not supported");
        b2_texture_desc t;
        memset(&t, 0, sizeof(t));
        auto lowerOf = [](std::string v) { std::transform(v.begin(), v.end(), v.begin(), ::tolower); return v; };
        const std::string ft = lowerOf(p.s("filterType", "ewa")); // bitmap.cpp:213-230
        if (ft == "ewa") t.filter_type = B2_TEX_EWA; else if (ft == "bilinear") t.filter_type = B2_TEX_BILINEAR;
        else if (ft == "trilinear") t.filter_type = B2_TEX_TRILINEAR; else if (ft == "nearest") t.filter_type = B2_TEX_NEAREST;
        else throw Err("Invalid filter type '" + ft + "', must be 'ewa', 'trilinear', or 'nearest'!");
        auto wrapOf = [](const std::string &m) { // bitmap.cpp:324-338
            if (m == "repeat") return (int) B2_WRAP_REPEAT; if (m == "clamp") return (int) B2_WRAP_CLAMP; if (m == "mirror") return (int) B2_WRAP_MIRROR;
            if (m == "zero" || m == "black") return (int) B2_WRAP_ZERO; if (m == "one" || m == "white") return (int) B2_WRAP_ONE;
            throw Err("Invalid wrap mode '" + m + "', must be 'repeat', 'clamp', 'black', or 'white'!");
        };
        const std::string wm = p.s("wrapMode", "repeat");
        t.wrap_u = wrapOf(p.s("wrapModeU", wm)); t.wrap_v = wrapOf(p.s("wrapModeV", wm));
        t.max_anisotropy = (float) p.f("maxAnisotropy", 20);
        const double gamma = p.f("gamma", 0);
        p.b("cache", false); // MIP map cache files are not written
        if (p.s("coordinates", "uv") != "uv") throw Err("Only UV coordinates are supported at the moment!"); // texture.cpp:81,95
        t.uoffset = (float) p.f("uoffset", 0); t.voffset = (float) p.f("voffset", 0);
        const double uvscale = p.f("uvscale", 1);
        t.uscale = (float) p.f("uscale", uvscale); t.vscale = (float) p.f("vscale", uvscale);
        p.checkAllUsed();
        std::vector<float> px;
        loadImage(fn, gamma, t.width, t.height, t.channels, px);
        t.pixels = px.data();
        const int id = b2_scene_add_texture(scene, &t);
        if (id < 0) throw Err(b2_last_error(nullptr));
        { // Texture::getAverage().getLuminance() as the BSDF constructors read it: float running sums of level 0 (after clampNegative) in
          // raster order over the texel count (barray.h:102-124), times the energy-conservation scale for images that exceed 1 (bsdf.cpp:88-111)
            const size_t nTexel = (size_t) t.width * t.height;
            float sum[3] = {0, 0, 0}, mx = 0;
            for (size_t k = 0; k < nTexel; ++k)
                for (int c = 0; c < t.channels; ++c) { const float v = std::max(px[k * t.channels + c], 0.0f); sum[c] += v; mx = std::max(mx, v); }
            const float scale = mx > 1.0f ? 0.99f * (1.0f / mx) : 1.0f;
            float avg[3];
            for (int c = 0; c < 3; ++c) avg[c] = sum[t.channels == 3 ? c : 0] / (float) nTexel * scale;
            if ((int) textureAvgLum.size() <= id) textureAvgLum.resize((size_t) id + 1, 0.0f);
            textureAvgLum[id] = avg[0] * 0.212671f + avg[1] * 0.715160f + avg[2] * 0.072169f;
        }
        if (!n->id.empty()) textureIds[n->id] = id;
        return id;
    }

    int resolveRef(Node *r) {
        auto it = bsdfIds.find(r->id);
        if (it == bsdfIds.end()) throw Err("Referenced object \"" + r->id + "\" not found (BSDF and medium references are supported)");
        return it->second;
    }

    // ---- participating media (SURVEY.md 8f-1) ----
    std::map<std::string, int> mediumIds;
    // GridDataSource::loadFromFile, gridvolume.cpp:225-296: "VOL" 3, type (1 = float32), res x/y/z, channels, data box, data
    static void loadVol(const std::string &path, int res[3], double lo[3], double hi[3], std::vector<float> &data) {
        std::ifstream f(path, std::ios::binary);
        if (!f) throw Err("gridvolume: cannot open \"" + path + "\"");
        char hdr[4];
        f.read(hdr, 4);
        if (!f || hdr[0] != 'V' || hdr[1] != 'O' || hdr[2] != 'L') throw Err("Encountered an invalid volume data file (incorrect header identifier)");
        if (hdr[3] != 3) throw Err("Encountered an invalid volume data file (incorrect file version)");
        int32_t h[5];
        f.read((char *) h, 20);
        if (h[0] != 1 || h[4] != 1) throw Err("gridvolume: only single-channel float32 density grids are supported (type " + std::to_string(h[0]) + ", channels " + std::to_string(h[4]) + ")");
        res[0] = h[1]; res[1] = h[2]; res[2] = h[3];
        float bb[6];
        f.read((char *) bb, 24);
        for (int i = 0; i < 3; ++i) { lo[i] = bb[i]; hi[i] = bb[3 + i]; }
        const size_t n = (size_t) res[0] * res[1] * res[2];
        if (!f || res[0] < 2 || res[1] < 2 || res[2] < 2) throw Err("gridvolume: invalid resolution");
        data.resize(n);
        f.read((char *) data.data(), (std::streamsize) (n * 4));
        if (!f) throw Err("gridvolume: file is truncated");
    }
    int addMedium(Node *n) {
        if (!n->id.empty() && mediumIds.count(n->id)) return mediumIds[n->id];
        Props p(n);
        b2_medium_desc m;
        memset(&m, 0, sizeof(m));
        m.scale = 1;
        for (int c = 0; c < 3; ++c) m.albedo[c] = 0;
        std::vector<float> density;
        double g = 0;
        // phase function child (medium.cpp:57-65: isotropic when absent)
        m.phase = B2_PHASE_ISOTROPIC;
        for (auto &c : n->children) {
            if (c->tag == "phase") {
                Props pp(c.get());
                if (c->type == "isotropic") m.phase = B2_PHASE_ISOTROPIC;
                else if (c->type == "hg") {
                    m.phase = B2_PHASE_HG;
                    m.g = (float) pp.f("g", 0.8); // hg.cpp:49
                    if (m.g >= 1 || m.g <= -1) throw Err("The asymmetry parameter must lie in the interval (-1, 1)!"); // hg.cpp:50-51
                } else throw Err("unsupported phase function \"" + c->type + "\" (supported: isotropic, hg)");
                pp.checkAllUsed();
            }
        }
        if (n->type == "homogeneous") { // medium.cpp:27-37 + materials.h:90-190 (no preset table) + homogeneous.cpp:156-222
            m.type = B2_MEDIUM_HOMOGENEOUS;
            // materials.h:90-160 lookupMaterial: the coefficients START from a preset -- "Skin1" unless `material` names another one -- in
            // mm^-1, times 100; whatever the scene gives overrides its half of the pair (a scene that only sets sigmaS keeps Skin1's sigmaA)
            if (p.has("material") && p.s("material", "Skin1") != "Skin1" && p.s("material", "Skin1") != "skin1")
                throw Err("homogeneous: of the measured material presets only the default \"Skin1\" is known here; give sigmaS/sigmaA or sigmaT/albedo");
            const bool hasAS = p.has("sigmaS") || p.has("sigmaA"), hasTA = p.has("sigmaT") || p.has("albedo");
            if (hasAS && hasTA) throw Err("You can either specify sigmaS & sigmaA *or* sigmaT & albedo, but no other combinations!");
            const double skinS[3] = {0.74 * 100, 0.88 * 100, 1.01 * 100}, skinA[3] = {0.032 * 100, 0.17 * 100, 0.48 * 100}; // materials.h:44
            float sS[3], sA[3];
            p.spec("sigmaS", skinS, sS); p.spec("sigmaA", skinA, sA);
            if (!hasAS) for (int c = 0; c < 3; ++c) { sS[c] = (float) skinS[c]; sA[c] = (float) skinA[c]; }
            if (hasTA) { // sigmaT defaults to sigmaA + sigmaS, albedo to sigmaS / (sigmaS + sigmaA) of the preset (materials.h:150-156)
                const double dT[3] = {sA[0] + sS[0], sA[1] + sS[1], sA[2] + sS[2]};
                const double dAl[3] = {sS[0] / dT[0], sS[1] / dT[1], sS[2] / dT[2]};
                float sT[3], al[3];
                p.spec("sigmaT", dT, sT); p.spec("albedo", dAl, al);
                for (int c = 0; c < 3; ++c) { sS[c] = al[c] * sT[c]; sA[c] = sT[c] - sS[c]; }
            }
            if (p.has("g")) g = p.f("g", 0);
            if (g <= -1 || g >= 1) throw Err("The anisotropy parameter 'g' must be in the range (-1, 1)!");
            const float scale = (float) p.f("scale", 1.0);
            for (int c = 0; c < 3; ++c) { m.sigma_s[c] = sS[c] * scale * (1.0f - (float) g); m.sigma_a[c] = sA[c] * scale; }
            float sT[3] = {m.sigma_a[0] + m.sigma_s[0], m.sigma_a[1] + m.sigma_s[1], m.sigma_a[2] + m.sigma_s[2]};
            float w = (float) p.f("mediumSamplingWeight", -1);
            if (w == -1) { // homogeneous.cpp:168-184
                for (int c = 0; c < 3; ++c) { float alb = m.sigma_s[c] / sT[c]; if (alb > w && sT[c] != 0) w = alb; }
                if (w > 0) w = std::max(w, 0.5f);
            }
            m.medium_sampling_weight = w;
            std::string strategy = p.s("strategy", "balance");
            if (strategy == "balance") m.strategy = 0;
            else if (strategy == "single") {
                m.strategy = 1;
                int channel = 0;
                float smallest = INFINITY;
                for (int c = 0; c < 3; ++c) if (sT[c] < smallest) { smallest = sT[c]; channel = c; }
                channel = (int) p.i("channel", channel);
                if (channel < 0 || channel > 2) throw Err("homogeneous: 'channel' out of range");
                m.sampling_density = sT[channel];
                if (p.b("monochromatic", false)) throw Err("homogeneous: 'monochromatic' is not supported");
            } else if (strategy == "manual") { m.strategy = 2; m.sampling_density = (float) p.f("samplingDensity", 0); }
            else throw Err("Specified an unknown sampling strategy"); // `maximum` is not on the path
        } else if (n->type == "heterogeneous") { // heterogeneous.cpp:182-260
            m.type = B2_MEDIUM_HETEROGENEOUS;
            if (p.has("sigmaS") || p.has("sigmaA"))
                throw Err("The 'sigmaS' and 'sigmaA' properties are only supported by homogeneous media. Please use nested volume instances to supply these parameters");
            std::string method = p.s("method", "woodcock");
            std::transform(method.begin(), method.end(), method.begin(), ::tolower);
            if (method != "woodcock") throw Err("Unsupported integration method \"" + method + "\"! (this library implements woodcock)");
            m.scale = (float) p.f("scale", 1.0);
            p.f("stepSize", 0);
            bool haveDensity = false, haveAlbedo = false;
            for (auto &c : n->children) {
                if (c->tag != "volume") continue;
                Props vp(c.get());
                if (c->name == "density") {
                    if (c->type != "gridvolume") throw Err("heterogeneous: the density must be a `gridvolume` (got \"" + c->type + "\")");
                    std::string fn = vp.s("filename", "");
                    if (fn.empty()) throw Err("gridvolume: missing 'filename'");
                    if (fn[0] != '/') fn = baseDir + "/" + fn;
                    double lo[3], hi[3];
                    loadVol(fn, m.res, lo, hi, density);
                    double pmin[3], pmax[3];
                    const bool hasMin = vp.vec("min", pmin), hasMax = vp.vec("max", pmax);
                    if (hasMin && hasMax) for (int i = 0; i < 3; ++i) { lo[i] = pmin[i]; hi[i] = pmax[i]; } // gridvolume.cpp:112-117
                    vp.b("sendData", false);
                    M4 v2w = vp.xf("toWorld"), w2v;
                    if (!v2w.inverse(w2v)) throw Err("gridvolume: singular toWorld transform");
                    // m_worldToGrid = scale((res - 1) / extents) * translate(-min) * worldToVolume (gridvolume.cpp:186-193)
                    M4 S, T;
                    for (int i = 0; i < 3; ++i) { S.m[i * 5] = (m.res[i] - 1) / (hi[i] - lo[i]); T.m[i * 4 + 3] = -lo[i]; }
                    M4 w2g = S * (T * w2v);
                    for (int i = 0; i < 12; ++i) m.world_to_grid[i] = (float) w2g.m[i];
                    for (int i = 0; i < 3; ++i) { m.aabb_min[i] = INFINITY; m.aabb_max[i] = -INFINITY; }
                    for (int k = 0; k < 8; ++k) { // gridvolume.cpp:197-199
                        const double q[3] = {(k & 4) ? hi[0] : lo[0], (k & 2) ? hi[1] : lo[1], (k & 1) ? hi[2] : lo[2]};
                        double o[3];
                        v2w.point(q, o);
                        for (int i = 0; i < 3; ++i) { m.aabb_min[i] = std::min(m.aabb_min[i], (float) o[i]); m.aabb_max[i] = std::max(m.aabb_max[i], (float) o[i]); }
                    }
                    haveDensity = true;
                } else if (c->name == "albedo") {
                    if (c->type != "constvolume") throw Err("heterogeneous: the albedo must be a `constvolume` (got \"" + c->type + "\")");
                    auto it = c->props.find("value");
                    if (it == c->props.end()) throw Err("constvolume: missing 'value'");
                    vp.used["value"] = true;
                    if (it->second.kind == Value::Spectrum) for (int k = 0; k < 3; ++k) m.albedo[k] = (float) it->second.v[k];
                    else if (it->second.kind == Value::Float || it->second.kind == Value::Int) for (int k = 0; k < 3; ++k) m.albedo[k] = (float) it->second.f;
                    else throw Err("constvolume: 'value' must be a spectrum or a float");
                    haveAlbedo = true;
                } else throw Err("heterogeneous: unsupported volume \"" + c->name + "\" (supported: density, albedo)");
                vp.checkAllUsed();
            }
            if (!haveDensity) throw Err("No density specified!");
            if (!haveAlbedo) throw Err("No albedo specified!");
            m.density = density.data();
        } else throw Err("unsupported medium \"" + n->type + "\" (supported: homogeneous, heterogeneous)");
        for (auto &c : n->children)
            if (c->tag != "phase" && c->tag != "volume" && c->tag != "transform") throw Err("unsupported child <" + c->tag + "> of <medium>");
        p.checkAllUsed();
        const int id = b2_scene_add_medium(scene, &m);
        if (id < 0) throw Err(b2_last_error(nullptr));
        if (!n->id.empty()) mediumIds[n->id] = id;
        return id;
    }

    struct MeshData { std::vector<float> P, N, UV; std::vector<uint32_t> idx; };

    void loadObj(const std::string &path, MeshData &md, bool flipTexCoords = true) {
        std::ifstream f(path);
        if (!f) throw Err("OBJ file \"" + path + "\" could not be found!");
        std::vector<double> v, vn, vt;
        std::map<std::tuple<int, int, int>, uint32_t> uniq;
        bool anyN = false, anyT = false, allN = true, allT = true;
        struct Corner { int v, t, n; };
        std::vector<std::vector<Corner>> faces;
        std::string line;
        while (std::getline(f, line)) {
            std::istringstream ss(line);
            std::string k;
            if (!(ss >> k)) continue;
            if (k == "v") { double x, y, z; ss >> x >> y >> z; v.insert(v.end(), {x, y, z}); }
            else if (k == "vn") { double x, y, z; ss >> x >> y >> z; vn.insert(vn.end(), {x, y, z}); }
            else if (k == "vt") { float x = 0, y = 0; ss >> x >> y; if (flipTexCoords) y = 1 - y; vt.insert(vt.end(), {x, y}); } // obj.cpp:305-308
            else if (k == "f") {
                std::vector<Corner> face;
                std::string tok;
                while (ss >> tok) {
                    Corner c{0, 0, 0};
                    int part = 0; size_t i = 0;
                    while (i <= tok.size()) {
                        size_t j = tok.find('/', i);
                        if (j == std::string::npos) j = tok.size();
                        std::string s = tok.substr(i, j - i);
                        int val = s.empty() ? 0 : atoi(s.c_str());
                        if (part == 0) c.v = val; else if (part == 1) c.t = val; else c.n = val;
                        ++part; i = j + 1;
                    }
                    auto fix = [](int idx, size_t count) { return idx < 0 ? (int) count + idx + 1 : idx; };
                    c.v = fix(c.v, v.size() / 3); c.t = fix(c.t, vt.size() / 2); c.n = fix(c.n, vn.size() / 3);
                    if (c.v <= 0 || (size_t) c.v > v.size() / 3) throw Err("OBJ: vertex index out of range in \"" + path + "\"");
                    face.push_back(c);
                }
                if (face.size() < 3) continue;
                faces.push_back(face);
                for (auto &c : face) { anyN |= c.n > 0; anyT |= c.t > 0; allN &= c.n > 0; allT &= c.t > 0; }
            }
        }
        bool useN = anyN && allN, useT = anyT && allT;
        for (auto &face : faces)
            for (size_t k = 1; k + 1 < face.size(); ++k) { // fan triangulation
                const Corner cs[3] = {face[0], face[k], face[k + 1]};
                for (auto &c : cs) {
                    auto key = std::make_tuple(c.v, useT ? c.t : 0, useN ? c.n : 0);
                    auto it = uniq.find(key);
                    uint32_t id;
                    if (it == uniq.end()) {
                        id = (uint32_t) (md.P.size() / 3);
                        uniq[key] = id;
                        for (int d = 0; d < 3; ++d) md.P.push_back((float) v[3 * (c.v - 1) + d]);
                        if (useN) for (int d = 0; d < 3; ++d) md.N.push_back((float) vn[3 * (c.n - 1) + d]);
                        if (useT) for (int d = 0; d < 2; ++d) md.UV.push_back((float) vt[2 * (c.t - 1) + d]);
                    } else id = it->second;
                    md.idx.push_back(id);
                }
            }
        if (md.idx.empty()) throw Err("OBJ file \"" + path + "\" contains no faces");
    }

    // TriMesh::computeNormals (trimesh.cpp:608-681): face-normal mode or angle-weighted smooth normals
    static void computeNormals(MeshData &md, bool faceNormals, bool flipNormals) {
        const size_t nV = md.P.size() / 3, nT = md.idx.size() / 3;
        if (faceNormals) {
            md.N.clear();
            if (flipNormals) for (size_t t = 0; t < nT; ++t) std::swap(md.idx[3 * t], md.idx[3 * t + 1]);
            return;
        }
        if (!md.N.empty()) { if (flipNormals) for (float &x : md.N) x = -x; return; }
        std::vector<double> acc(3 * nV, 0.0);
        auto sub = [&](uint32_t a, uint32_t b, float *o) { for (int d = 0; d < 3; ++d) o[d] = md.P[3 * a + d] - md.P[3 * b + d]; };
        for (size_t t = 0; t < nT; ++t) {
            float n[3] = {0, 0, 0};
            for (int i = 0; i < 3; ++i) {
                uint32_t i0 = md.idx[3 * t + i], i1 = md.idx[3 * t + (i + 1) % 3], i2 = md.idx[3 * t + (i + 2) % 3];
                float sa[3], sb[3];
                sub(i1, i0, sa); sub(i2, i0, sb);
                if (i == 0) {
                    n[0] = sa[1] * sb[2] - sa[2] * sb[1]; n[1] = sa[2] * sb[0] - sa[0] * sb[2]; n[2] = sa[0] * sb[1] - sa[1] * sb[0];
                    float len = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
                    if (len == 0) break;
                    for (float &c : n) c /= len;
                }
                float la = std::sqrt(sa[0] * sa[0] + sa[1] * sa[1] + sa[2] * sa[2]), lb = std::sqrt(sb[0] * sb[0] + sb[1] * sb[1] + sb[2] * sb[2]);
                float ua[3] = {sa[0] / la, sa[1] / la, sa[2] / la}, ub[3] = {sb[0] / lb, sb[1] / lb, sb[2] / lb};
                // unitAngle (vector.h): numerically robust angle between unit vectors
                float dp = ua[0] * ub[0] + ua[1] * ub[1] + ua[2] * ub[2], angle;
                if (dp < 0) { float s[3] = {ub[0] + ua[0], ub[1] + ua[1], ub[2] + ua[2]}; angle = (float) M_PI - 2 * std::asin(0.5f * std::sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2])); }
                else { float s[3] = {ub[0] - ua[0], ub[1] - ua[1], ub[2] - ua[2]}; angle = 2 * std::asin(0.5f * std::sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2])); }
                for (int d = 0; d < 3; ++d) acc[3 * i0 + d] += n[d] * angle;
            }
        }
        md.N.resize(3 * nV);
        for (size_t i = 0; i < nV; ++i) {
            double len = std::sqrt(acc[3 * i] * acc[3 * i] + acc[3 * i + 1] * acc[3 * i + 1] + acc[3 * i + 2] * acc[3 * i + 2]);
            if (flipNormals) len = -len;
            if (len != 0) for (int d = 0; d < 3; ++d) md.N[3 * i + d] = (float) (acc[3 * i + d] / len);
            else { md.N[3 * i] = 1; md.N[3 * i + 1] = 0; md.N[3 * i + 2] = 0; }
        }
    }

    // Stanford PLY (src/shapes/ply.cpp): ascii and binary (either byte order); vertex x y z [nx ny nz] [u|s|texture_u v|t|texture_v],
    // other vertex properties are skipped; faces with 3 or 4 vertices, a quad (f0 f1 f2 f3) becomes (f0 f1 f2)(f3 f0 f2) (ply.cpp:276-287)
    void loadPly(const std::string &path, MeshData &md) {
        std::ifstream f(path, std::ios::binary);
        if (!f) throw Err("PLY file \"" + path + "\" could not be found!");
        std::string line;
        std::getline(f, line);
        if (line.substr(0, 3) != "ply") throw Err("\"" + path + "\" is not a PLY file");
        enum Fmt { Ascii, LE, BE } fmt = Ascii;
        struct Prop { std::string name, type, countType; bool list = false; };
        struct Elem { std::string name; size_t count = 0; std::vector<Prop> props; };
        std::vector<Elem> elems;
        while (std::getline(f, line)) {
            if (!line.empty() && line.back() == '\r') line.pop_back();
            std::istringstream ls(line);
            std::string k;
            ls >> k;
            if (k == "format") { std::string v; ls >> v; fmt = v == "ascii" ? Ascii : (v == "binary_little_endian" ? LE : BE); }
            else if (k == "element") { Elem e; ls >> e.name >> e.count; elems.push_back(e); }
            else if (k == "property") {
                if (elems.empty()) throw Err("PLY: property before element");
                Prop pr; std::string t; ls >> t;
                if (t == "list") { pr.list = true; ls >> pr.countType >> pr.type >> pr.name; } else { pr.type = t; ls >> pr.name; }
                elems.back().props.push_back(pr);
            } else if (k == "end_header") break;
        }
        auto typeSize = [](const std::string &t) -> int {
            if (t == "char" || t == "uchar" || t == "int8" || t == "uint8") return 1;
            if (t == "short" || t == "ushort" || t == "int16" || t == "uint16") return 2;
            if (t == "int" || t == "uint" || t == "float" || t == "int32" || t == "uint32" || t == "float32") return 4;
            if (t == "double" || t == "float64") return 8;
            throw Err("PLY: unknown property type \"" + t + "\"");
        };
        auto readNum = [&](const std::string &t) -> double {
            if (fmt == Ascii) { double v; if (!(f >> v)) throw Err("PLY: unexpected end of file"); return v; }
            unsigned char b[8];
            const int n = typeSize(t);
            f.read((char *) b, n);
            if (!f) throw Err("PLY: unexpected end of file");
            if (fmt == BE) std::reverse(b, b + n);
            if (t == "float" || t == "float32") { float v; memcpy(&v, b, 4); return v; }
            if (t == "double" || t == "float64") { double v; memcpy(&v, b, 8); return v; }
            if (t == "char" || t == "int8") return (double) (int8_t) b[0];
            if (t == "uchar" || t == "uint8") return (double) b[0];
            if (t == "short" || t == "int16") { int16_t v; memcpy(&v, b, 2); return v; }
            if (t == "ushort" || t == "uint16") { uint16_t v; memcpy(&v, b, 2); return v; }
            if (t == "int" || t == "int32") { int32_t v; memcpy(&v, b, 4); return v; }
            uint32_t v; memcpy(&v, b, 4); return v;
        };
        bool hasN = false, hasUV = false;
        for (auto &e : elems) {
            if (e.name == "vertex") {
                for (auto &pr : e.props) { hasN |= pr.name == "nx"; hasUV |= pr.name == "u" || pr.name == "s" || pr.name == "texture_u"; }
                md.P.resize(3 * e.count);
                if (hasN) md.N.resize(3 * e.count);
                if (hasUV) md.UV.resize(2 * e.count);
                for (size_t i = 0; i < e.count; ++i)
                    for (auto &pr : e.props) {
                        if (pr.list) { const int n = (int) readNum(pr.countType); for (int k = 0; k < n; ++k) readNum(pr.type); continue; }
                        const double v = readNum(pr.type);
                        if (pr.name == "x") md.P[3 * i] = (float) v; else if (pr.name == "y") md.P[3 * i + 1] = (float) v; else if (pr.name == "z") md.P[3 * i + 2] = (float) v;
                        else if (pr.name == "nx") md.N[3 * i] = (float) v; else if (pr.name == "ny") md.N[3 * i + 1] = (float) v; else if (pr.name == "nz") md.N[3 * i + 2] = (float) v;
                        else if (pr.name == "u" || pr.name == "s" || pr.name == "texture_u") md.UV[2 * i] = (float) v;
                        else if (pr.name == "v" || pr.name == "t" || pr.name == "texture_v") md.UV[2 * i + 1] = (float) v;
                    }
            } else if (e.name == "face") {
                for (size_t i = 0; i < e.count; ++i)
                    for (auto &pr : e.props) {
                        if (!pr.list) { readNum(pr.type); continue; }
                        const int n = (int) readNum(pr.countType);
                        if (pr.name != "vertex_indices" && pr.name != "vertex_index") { for (int k = 0; k < n; ++k) readNum(pr.type); continue; }
                        if (n != 3 && n != 4) throw Err("Only triangle and quad-based PLY meshes are supported for now."); // ply.cpp:252-254
                        uint32_t face[4];
                        for (int k = 0; k < n; ++k) {
                            const double v = readNum(pr.type);
                            if (v < 0 || (size_t) v >= md.P.size() / 3) throw Err("PLY: vertex index out of range");
                            face[k] = (uint32_t) v;
                        }
                        md.idx.insert(md.idx.end(), {face[0], face[1], face[2]});
                        if (n == 4) md.idx.insert(md.idx.end(), {face[3], face[0], face[2]});
                    }
            } else { // skip unknown elements
                for (size_t i = 0; i < e.count; ++i)
                    for (auto &pr : e.props) {
                        if (pr.list) { const int n = (int) readNum(pr.countType); for (int k = 0; k < n; ++k) readNum(pr.type); } else readNum(pr.type);
                    }
            }
        }
        if (md.idx.empty() || md.P.empty()) throw Err("Unable to load \"" + path + "\" (no triangles or vertices found)!");
    }

    // Mitsuba's compressed triangle-mesh format (src/librender/trimesh.cpp:147-300, src/shapes/serialized.cpp): u16 0x041C, u16 version
    // (3 | 4), zlib stream {u32 flags, [v4: name\0], u64 nV, u64 nT, positions, [normals], [texcoords], [colors], u32 indices}; several
    // shapes per file are addressed through the offset dictionary at the end (u32 offsets in v3, u64 in v4, then u32 count)
    void loadSerialized(const std::string &path, int shapeIndex, MeshData &md, bool &fileFaceNormals) {
        std::ifstream f(path, std::ios::binary);
        if (!f) throw Err("serialized: cannot open \"" + path + "\"");
        std::vector<unsigned char> file((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        auto rd16 = [&](size_t o) { if (o + 2 > file.size()) throw Err("serialized: truncated file"); return (uint16_t) (file[o] | (file[o + 1] << 8)); };
        auto rd32 = [&](size_t o) { if (o + 4 > file.size()) throw Err("serialized: truncated file"); uint32_t v; memcpy(&v, &file[o], 4); return v; };
        auto rd64 = [&](size_t o) { if (o + 8 > file.size()) throw Err("serialized: truncated file"); uint64_t v; memcpy(&v, &file[o], 8); return v; };
        auto header = [&](size_t o) -> int {
            const uint16_t format = rd16(o), version = rd16(o + 2);
            if (format != 0x041C) throw Err("Encountered an invalid file format!");
            if (version != 3 && version != 4) throw Err("Encountered an incompatible file version!");
            return version;
        };
        const int version = header(0);
        size_t offset = 0;
        if (shapeIndex != 0) { // trimesh.cpp:273-292 readOffset
            const uint32_t count = rd32(file.size() - 4);
            if (shapeIndex < 0 || shapeIndex >= (int) count) throw Err("Unable to unserialize mesh, shape index is out of range!");
            offset = version == 4 ? (size_t) rd64(file.size() - 8 * (size_t) (count - shapeIndex) - 4) : (size_t) rd32(file.size() - 4 * (size_t) (count - shapeIndex + 1));
            header(offset);
        }
        // inflate everything from offset + 4 (the stream ends at Z_STREAM_END)
        std::vector<unsigned char> data;
        z_stream zs;
        memset(&zs, 0, sizeof(zs));
        if (inflateInit(&zs) != Z_OK) throw Err("serialized: inflateInit failed");
        zs.next_in = file.data() + offset + 4;
        zs.avail_in = (uInt) std::min<size_t>(file.size() - offset - 4, 0xFFFFFFFFu);
        unsigned char buf[1 << 16];
        int rc;
        do {
            zs.next_out = buf; zs.avail_out = sizeof(buf);
            rc = inflate(&zs, Z_NO_FLUSH);
            if (rc != Z_OK && rc != Z_STREAM_END) { inflateEnd(&zs); throw Err("serialized: corrupt zlib stream"); }
            data.insert(data.end(), buf, buf + (sizeof(buf) - zs.avail_out));
        } while (rc != Z_STREAM_END);
        inflateEnd(&zs);
        size_t pos = 0;
        auto need = [&](size_t n) { if (pos + n > data.size()) throw Err("serialized: truncated mesh record"); };
        need(4);
        uint32_t flags; memcpy(&flags, &data[pos], 4); pos += 4;
        if (version == 4) { while (true) { need(1); if (data[pos++] == 0) break; } }
        need(16);
        uint64_t nV, nT; memcpy(&nV, &data[pos], 8); memcpy(&nT, &data[pos + 8], 8); pos += 16;
        const bool dbl = (flags & 0x2000) != 0;
        fileFaceNormals = (flags & 0x0010) != 0;
        auto readFloats = [&](std::vector<float> &out, size_t n) {
            out.resize(n);
            if (dbl) { need(8 * n); for (size_t i = 0; i < n; ++i) { double v; memcpy(&v, &data[pos + 8 * i], 8); out[i] = (float) v; } pos += 8 * n; }
            else { need(4 * n); memcpy(out.data(), &data[pos], 4 * n); pos += 4 * n; }
        };
        readFloats(md.P, 3 * (size_t) nV);
        if (flags & 0x0001) readFloats(md.N, 3 * (size_t) nV);
        if (flags & 0x0002) readFloats(md.UV, 2 * (size_t) nV);
        if (flags & 0x0008) { std::vector<float> colors; readFloats(colors, 3 * (size_t) nV); }
        need(12 * (size_t) nT);
        md.idx.resize(3 * (size_t) nT);
        memcpy(md.idx.data(), &data[pos], 12 * (size_t) nT);
        for (uint32_t i : md.idx) if (i >= nV) throw Err("serialized: vertex index out of range");
        if (nT == 0 || nV == 0) throw Err("Encountered an empty triangle mesh!");
    }

    std::map<std::string, int> groupIds;
    void addShape(Node *n, int group = -1) {
        if (n->type == "shapegroup") { // shapegroup.cpp:107-135: children live in the group's object space
            if (group >= 0) throw Err("Nested instancing is not permitted");
            const int gid = b2_scene_add_shapegroup(scene);
            for (auto &c : n->children) {
                if (c->tag != "shape") throw Err("unsupported child <" + c->tag + "> of <shape type=\"shapegroup\">");
                if (c->type == "shapegroup" || c->type == "instance") throw Err("Nested instancing is not permitted");
                addShape(c.get(), gid);
            }
            if (!n->id.empty()) groupIds[n->id] = gid;
            return;
        }
        if (n->type == "instance") { // instance.cpp:49-78
            if (group >= 0) throw Err("Nested instancing is not permitted");
            Props ip(n);
            int gid = -1;
            for (auto &c : n->children) {
                if (c->tag == "ref") { auto it = groupIds.find(c->id); if (it == groupIds.end()) throw Err("Referenced object \"" + c->id + "\" not found"); gid = it->second; }
                else if (c->tag != "transform") throw Err("unsupported child <" + c->tag + "> of <shape type=\"instance\">");
            }
            if (gid < 0) throw Err("A reference to a 'shapegroup' must be specified!");
            M4 tw = ip.xf("toWorld"), inv;
            if (!tw.inverse(inv)) throw Err("instance: singular toWorld transform");
            ip.checkAllUsed();
            float a[16], b[16];
            for (int i = 0; i < 16; ++i) { a[i] = (float) tw.m[i]; b[i] = (float) inv.m[i]; }
            if (b2_scene_add_instance(scene, gid, a, b) < 0) throw Err(b2_last_error(nullptr));
            return;
        }
        Props p(n);
        MeshData md;
        M4 toWorld = p.xf("toWorld"), inv;
        if (!toWorld.inverse(inv)) throw Err("shape: singular toWorld transform");
        bool flip = p.b("flipNormals", false);
        if (n->type == "obj" || n->type == "ply" || n->type == "serialized") {
            std::string fn = p.s("filename", "");
            if (fn.empty()) throw Err(n->type + ": missing 'filename'");
            if (fn[0] != '/') fn = baseDir + "/" + fn;
            bool fileFaceNormals = false;
            if (n->type == "obj") { loadObj(fn, md, p.b("flipTexCoords", true)); p.b("collapse", false); }
            else if (n->type == "ply") { loadPly(fn, md); p.b("srgb", true); }
            else loadSerialized(fn, (int) p.i("shapeIndex", 0), md, fileFaceNormals);
            bool faceN = p.b("faceNormals", false) || fileFaceNormals;
            p.f("maxSmoothAngle", 0.0);
            // object -> world
            for (size_t i = 0; i < md.P.size() / 3; ++i) {
                double q[3] = {md.P[3 * i], md.P[3 * i + 1], md.P[3 * i + 2]}, o[3];
                toWorld.point(q, o);
                for (int d = 0; d < 3; ++d) md.P[3 * i + d] = (float) o[d];
                if (!md.N.empty()) {
                    double nn[3] = {md.N[3 * i], md.N[3 * i + 1], md.N[3 * i + 2]}, on[3];
                    toWorld.normal(inv, nn, on);
                    double l = std::sqrt(on[0] * on[0] + on[1] * on[1] + on[2] * on[2]);
                    for (int d = 0; d < 3; ++d) md.N[3 * i + d] = (float) (l > 0 ? on[d] / l : on[d]);
                }
            }
            computeNormals(md, faceN, flip);
        } else if (n->type == "rectangle") { // rectangle.cpp:170-205 createTriMesh
            const double v[4][3] = {{-1, -1, 0}, {1, -1, 0}, {1, 1, 0}, {-1, 1, 0}}, uv[4][2] = {{0, 0}, {1, 0}, {1, 1}, {0, 1}};
            double nz[3] = {0, 0, flip ? -1.0 : 1.0}, nw[3];
            toWorld.normal(inv, nz, nw);
            double l = std::sqrt(nw[0] * nw[0] + nw[1] * nw[1] + nw[2] * nw[2]);
            for (int i = 0; i < 4; ++i) {
                double o[3];
                toWorld.point(v[i], o);
                for (int d = 0; d < 3; ++d) { md.P.push_back((float) o[d]); md.N.push_back((float) (nw[d] / l)); }
                md.UV.push_back((float) uv[i][0]); md.UV.push_back((float) uv[i][1]);
            }
            md.idx = {0, 1, 2, 2, 3, 0};
        } else if (n->type == "cube") { // cube.cpp:73-106: 24 unshared vertices, per-face normals and UVs
            const double fn[6][3] = {{0, 0, -1}, {0, 0, 1}, {0, -1, 0}, {0, 1, 0}, {-1, 0, 0}, {1, 0, 0}};
            for (int f = 0; f < 6; ++f) {
                const double *nn = fn[f];
                double a[3], b[3];
                int ax = nn[0] != 0 ? 0 : (nn[1] != 0 ? 1 : 2);
                double s = nn[ax];
                for (int d = 0; d < 3; ++d) { a[d] = 0; b[d] = 0; }
                a[(ax + 1) % 3] = 1; b[(ax + 2) % 3] = s; // right-handed: a x b = n
                const double c[4][2] = {{-1, -1}, {1, -1}, {1, 1}, {-1, 1}};
                double nw[3];
                double nflip[3] = {flip ? -nn[0] : nn[0], flip ? -nn[1] : nn[1], flip ? -nn[2] : nn[2]};
                toWorld.normal(inv, nflip, nw);
                double l = std::sqrt(nw[0] * nw[0] + nw[1] * nw[1] + nw[2] * nw[2]);
                uint32_t base = (uint32_t) (md.P.size() / 3);
                for (int i = 0; i < 4; ++i) {
                    double q[3], o[3];
                    for (int d = 0; d < 3; ++d) q[d] = nn[d] + c[i][0] * a[d] + c[i][1] * b[d];
                    toWorld.point(q, o);
                    for (int d = 0; d < 3; ++d) { md.P.push_back((float) o[d]); md.N.push_back((float) (nw[d] / l)); }
                    md.UV.push_back((float) (0.5 * (c[i][0] + 1))); md.UV.push_back((float) (0.5 * (c[i][1] + 1)));
                }
                md.idx.insert(md.idx.end(), {base, base + 1, base + 2, base + 3, base, base + 2});
            }
        } else throw Err("unsupported shape plugin \"" + n->type + "\" (supported: obj, ply, serialized, rectangle, cube, shapegroup, instance)");
        // children: bsdf / ref / emitter
        int mat = -1, em = -1, interior = -1, exterior = -1;
        bool isEmitter = false;
        for (auto &c : n->children) {
            if (c->tag == "bsdf") mat = addBsdf(c.get());
            else if (c->tag == "medium" || (c->tag == "ref" && (c->name == "interior" || c->name == "exterior"))) { // shape.cpp:160-176
                int mid;
                if (c->tag == "medium") mid = addMedium(c.get());
                else {
                    auto it = mediumIds.find(c->id);
                    if (it == mediumIds.end()) throw Err("Referenced object \"" + c->id + "\" not found");
                    mid = it->second;
                }
                if (c->name == "interior") interior = mid;
                else if (c->name == "exterior") exterior = mid;
                else throw Err("Shape: Invalid medium child (must be named 'interior' or 'exterior')!");
            }
            else if (c->tag == "ref") mat = resolveRef(c.get());
            else if (c->tag == "emitter") {
                if (c->type != "area") throw Err("unsupported emitter plugin \"" + c->type + "\" (hot path: area)");
                Props ep(c.get());
                const double one[3] = {1, 1, 1};
                float rad[3];
                ep.spec("radiance", one, rad);
                float w = (float) ep.f("samplingWeight", 1.0);
                ep.checkAllUsed();
                em = b2_scene_add_area_emitter(scene, rad, w);
                if (em < 0) throw Err(b2_last_error(nullptr));
                isEmitter = true;
            } else if (c->tag != "transform") throw Err("unsupported child <" + c->tag + "> of <shape>");
        }
        if (mat < 0) { // shape.cpp:48-72: emitter -> black diffuse; medium transition -> null; else 0.5 diffuse
            b2_material_desc m;
            memset(&m, 0, sizeof(m));
            const bool transition = interior >= 0 || exterior >= 0;
            m.type = (!isEmitter && transition) ? B2_BSDF_NULL : B2_BSDF_DIFFUSE;
            m.nested = -1; m.eta = 1; m.thickness = 1; m.sample_visible = 1; m.alpha_u = m.alpha_v = 0.1f;
            for (int c = 0; c < 3; ++c) { m.reflectance[c] = isEmitter ? 0.0f : 0.5f; m.transmittance[c] = 1; m.k_c[c] = 1; }
            mat = b2_scene_add_material(scene, &m);
        }
        p.checkAllUsed();
        int id = b2_scene_add_mesh(scene, md.P.data(), md.N.empty() ? nullptr : md.N.data(), md.UV.empty() ? nullptr : md.UV.data(),
                                   (uint32_t) (md.P.size() / 3), md.idx.data(), (uint32_t) (md.idx.size() / 3), mat, em);
        if (id < 0) throw Err(b2_last_error(nullptr));
        if ((interior >= 0 || exterior >= 0) && b2_scene_set_mesh_media(scene, id, interior, exterior)) throw Err(b2_last_error(nullptr));
        if (group >= 0 && b2_scene_set_mesh_group(scene, id, group)) throw Err(b2_last_error(nullptr));
    }

    void run(Node *root, b2_render_params *rp) {
        memset(rp, 0, sizeof(*rp));
        rp->spp = 4; rp->sampler = B2_SAMPLER_INDEPENDENT; rp->max_depth = -1; rp->rr_depth = 5; // independent is Mitsuba's default sampler
        rp->rfilter = B2_RFILTER_GAUSSIAN; rp->rfilter_param = 0.5f;
        bool haveSensor = false;
        for (auto &c : root->children) if (c->tag == "texture") addTexture(c.get());
        for (auto &c : root->children) if (c->tag == "bsdf") addBsdf(c.get());
        for (auto &c : root->children) if (c->tag == "medium") addMedium(c.get());
        bool haveIntegrator = false;
        for (auto &cu : root->children) {
            Node *c = cu.get();
            if (c->tag == "bsdf" || c->tag == "medium" || c->tag == "texture") continue;
            if (c->tag == "integrator") {
                haveIntegrator = true;
                if (c->type == "volpath") rp->integrator = B2_INTEGRATOR_VOLPATH;
                else if (c->type == "direct") rp->integrator = B2_INTEGRATOR_DIRECT;
                else if (c->type != "path")
                    throw Err("unsupported integrator \"" + c->type + "\": this library implements the `path`, `volpath` and `direct` plugins");
                Props p(c);
                if (rp->integrator == B2_INTEGRATOR_DIRECT) { // direct.cpp:93-108: shadingSamples is the default of both counts
                    const long long shading = p.i("shadingSamples", 1);
                    const long long ne = p.i("emitterSamples", shading), nb = p.i("bsdfSamples", shading);
                    if (ne < 0 || nb < 0 || ne > 32767 || nb > 32767) throw Err("direct: sample counts must lie in [0, 32767]");
                    rp->emitter_samples = (int16_t) ne; rp->bsdf_samples = (int16_t) nb;
                } else {
                    rp->max_depth = (int) p.i("maxDepth", -1); rp->rr_depth = (int) p.i("rrDepth", 5);
                }
                rp->strict_normals = p.b("strictNormals", false); rp->hide_emitters = p.b("hideEmitters", false);
                p.checkAllUsed();
            } else if (c->tag == "sensor") {
                if (c->type != "perspective" && c->type != "thinlens") throw Err("unsupported sensor \"" + c->type + "\" (supported: perspective, thinlens)");
                Props p(c);
                int W = 768, H = 576; // film.cpp:30-33
                int cropX = 0, cropY = 0, cropW = -1, cropH = -1; // film.cpp:36-43
                for (auto &ch : c->children) {
                    if (ch->tag == "film") {
                        Props fp(ch.get());
                        W = (int) fp.i("width", 768); H = (int) fp.i("height", 576);
                        cropX = (int) fp.i("cropOffsetX", 0); cropY = (int) fp.i("cropOffsetY", 0);
                        cropW = (int) fp.i("cropWidth", W); cropH = (int) fp.i("cropHeight", H);
                        fp.s("pixelFormat", "rgb"); fp.s("fileFormat", "openexr"); fp.s("componentFormat", "float16"); fp.b("banner", true);
                        fp.b("attachLog", true); fp.b("highQualityEdges", false);
                        fp.checkAllUsed();
                        for (auto &rf : ch->children) {
                            if (rf->tag != "rfilter") throw Err("unsupported child <" + rf->tag + "> of <film>");
                            Props rfp(rf.get());
                            if (rf->type == "box") { rp->rfilter = B2_RFILTER_BOX; rp->rfilter_param = (float) rfp.f("radius", 0.5); }
                            else if (rf->type == "gaussian") { rp->rfilter = B2_RFILTER_GAUSSIAN; rp->rfilter_param = (float) rfp.f("stddev", 0.5); }
                            else throw Err("unsupported reconstruction filter \"" + rf->type + "\" (supported: box, gaussian)");
                            rfp.checkAllUsed();
                        }
                    } else if (ch->tag == "sampler") {
                        Props sp(ch.get());
                        rp->spp = (int) sp.i("sampleCount", 4);
                        if (ch->type == "sobol") { rp->sampler = B2_SAMPLER_SOBOL; rp->seed = (uint64_t) sp.i("scramble", 0); }
                        else if (ch->type == "independent") { rp->sampler = B2_SAMPLER_INDEPENDENT; rp->seed = (uint64_t) sp.i("seed", 0); }
                        else throw Err("unsupported sampler \"" + ch->type + "\" (hot path: sobol, independent)");
                        sp.checkAllUsed();
                    } else if (ch->tag != "transform") throw Err("unsupported child <" + ch->tag + "> of <sensor>");
                }
                // fov handling: sensor.cpp:221-275,293-316
                double aspect = (double) W / H, fov = p.f("fov", 0);
                if (!p.has("fov")) {
                    std::string fl = p.s("focalLength", "50mm");
                    if (fl.size() > 2 && fl.substr(fl.size() - 2) == "mm") fl = fl.substr(0, fl.size() - 2);
                    double value = Parser::toF(fl, "focalLength");
                    double diag = 2 * 180 / M_PI * std::atan(std::sqrt(36.0 * 36 + 24 * 24) / (2 * value));
                    double dl = 2 * std::tan(0.5 * diag * M_PI / 180), width = dl / std::sqrt(1.0 + 1.0 / (aspect * aspect));
                    fov = 2 * std::atan(width * 0.5) * 180 / M_PI;
                    p.s("fovAxis", "x");
                } else {
                    std::string ax = p.s("fovAxis", "x");
                    std::transform(ax.begin(), ax.end(), ax.begin(), ::tolower);
                    if (ax == "smaller") ax = aspect > 1 ? "y" : "x"; else if (ax == "larger") ax = aspect > 1 ? "x" : "y";
                    if (ax == "y") fov = 2 * std::atan(std::tan(0.5 * fov * M_PI / 180) * aspect) * 180 / M_PI;
                    else if (ax == "diagonal") { double dl = 2 * std::tan(0.5 * fov * M_PI / 180), width = dl / std::sqrt(1.0 + 1.0 / (aspect * aspect)); fov = 2 * std::atan(width * 0.5) * 180 / M_PI; }
                    else if (ax != "x") throw Err("The 'fovAxis' parameter must be set to one of 'smaller', 'larger', 'diagonal', 'x', or 'y'!");
                }
                M4 tw = p.xf("toWorld");
                float twf[16];
                for (int i = 0; i < 16; ++i) twf[i] = (float) tw.m[i];
                float nearC = (float) p.f("nearClip", 1e-2), farC = (float) p.f("farClip", 1e4);
                const float focusD = (float) p.f("focusDistance", farC); // sensor.cpp:162
                p.f("shutterOpen", 0); p.f("shutterClose", 0);
                float aperture = 0;
                if (c->type == "thinlens") {
                    if (!p.has("apertureRadius")) throw Err("thinlens: missing required property 'apertureRadius'"); // thinlens.cpp:133
                    aperture = (float) p.f("apertureRadius", 0);
                    if (aperture == 0) aperture = 1e-4f; // thinlens.cpp:134-138: a zero radius becomes Epsilon
                }
                p.checkAllUsed();
                if (b2_scene_set_camera(scene, twf, (float) fov, nearC, farC, W, H)) throw Err(b2_last_error(nullptr));
                if (cropW < 0) { cropW = W; cropH = H; }
                if ((cropX != 0 || cropY != 0 || cropW != W || cropH != H) && b2_scene_set_crop(scene, cropX, cropY, cropW, cropH)) throw Err(b2_last_error(nullptr));
                if (aperture > 0 && b2_scene_set_thinlens(scene, aperture, focusD)) throw Err(b2_last_error(nullptr));
                haveSensor = true;
            } else if (c->tag == "shape") addShape(c);
            else if (c->tag == "emitter") {
                if (c->type == "envmap") { addEnvMap(c); continue; }
                if (c->type != "constant") throw Err("unsupported top-level emitter \"" + c->type + "\" (supported: constant, envmap; area emitters are attached to shapes)");
                Props ep(c);
                const double one[3] = {1, 1, 1};
                float rad[3];
                ep.spec("radiance", one, rad); // constant.cpp:47-50
                const float w = (float) ep.f("samplingWeight", 1.0);
                ep.checkAllUsed();
                // position in Scene::m_emitters (= in the emitter-selection CDF): b2_scene_commit puts scene-level emitters ahead of
                // the shapes' area emitters whatever the document order, as Scene::addChild / Scene::initialize do (scene.cpp:510-516, :322-335)
                if (b2_scene_add_constant_emitter(scene, rad, w) < 0) throw Err(b2_last_error(nullptr));
            }
            else throw Err("unsupported top-level element <" + c->tag + ">");
        }
        if (!haveSensor) throw Err("scene has no <sensor>");
        // the reference gives a scene without an <integrator> the `direct` plugin (scene.cpp:274-276); this library asks for it by name
        if (!haveIntegrator) throw Err("scene has no <integrator>: Mitsuba would render it with `direct`; name the integrator (`path`, `volpath` or `direct`)");
    }
};

} // namespace

extern "C" int b2_set_error_(b2_ctx *, int, const char *);

// Host-only: decode an image file the way the scene-file front end does for `bitmap` textures and `envmap` emitters (linear float, top row
// first).  out may be NULL to query the size; returns 0, or -1 with the message in err.
extern "C" int b2_load_image(const char *path, float gamma, int *width, int *height, int *channels, float *out, char *err, int errLen) {
    try {
        int w, h, ch;
        std::vector<float> px;
        Loader::loadImage(path ? path : "", gamma, w, h, ch, px);
        if (width) *width = w;
        if (height) *height = h;
        if (channels) *channels = ch;
        if (out) memcpy(out, px.data(), px.size() * sizeof(float));
        return 0;
    } catch (const std::exception &e) {
        if (err && errLen > 0) { strncpy(err, e.what(), (size_t) errLen - 1); err[errLen - 1] = 0; }
        return -1;
    }
}
extern "C" int b2_load_xml(b2_ctx *ctx, const char *path, const char *const *defines, int n_defines, b2_scene **out, b2_render_params *params) {
    if (!ctx || !path || !out || !params) return b2_set_error_(ctx, B2_ERR_INVALID, "b2_load_xml: null argument");
    *out = nullptr;
    Parser P;
    for (int i = 0; i < n_defines; ++i) {
        std::string d = defines[i];
        size_t eq = d.find('=');
        if (eq == std::string::npos) return b2_set_error_(ctx, B2_ERR_INVALID, "b2_load_xml: defines must look like key=value");
        P.defines[d.substr(0, eq)] = d.substr(eq + 1);
    }
    std::string p = path;
    size_t slash = p.find_last_of('/');
    std::string baseDir = slash == std::string::npos ? "." : p.substr(0, slash);
    P.baseDir = baseDir; // <spectrum filename="..."> is resolved while parsing
    std::ifstream f(path, std::ios::binary);
    if (!f) return b2_set_error_(ctx, B2_ERR_IO, (std::string("cannot open scene file ") + path).c_str());
    std::string text((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    b2_scene *scene = nullptr;
    XML_Parser xp = XML_ParserCreate(nullptr);
    try {
        XML_SetUserData(xp, &P);
        XML_SetElementHandler(xp, onStart, onEnd);
        P.xp = xp;
        g_parseError.clear();
        if (XML_Parse(xp, text.data(), (int) text.size(), 1) == XML_STATUS_ERROR) {
            std::ostringstream oss;
            oss << path << ":" << XML_GetCurrentLineNumber(xp) << ": " << (g_parseError.empty() ? XML_ErrorString(XML_GetErrorCode(xp)) : g_parseError.c_str());
            throw Err(oss.str());
        }
        if (!P.root) throw Err("empty scene file");
        if (b2_scene_create(ctx, &scene)) throw Err(b2_last_error(ctx));
        Loader L;
        L.scene = scene;
        L.baseDir = baseDir;
        L.run(P.root.get(), params);
        if (b2_scene_commit(scene)) throw Err(b2_last_error(ctx));
    } catch (const std::exception &e) {
        XML_ParserFree(xp);
        if (scene) b2_scene_destroy(scene);
        return b2_set_error_(ctx, B2_ERR_INVALID, e.what());
    }
    XML_ParserFree(xp);
    *out = scene;
    return B2_OK;
}
