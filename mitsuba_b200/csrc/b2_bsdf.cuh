// BSDF::sample / eval / pdf on the device for the four plugins the hot path names, plus the
// microfacet distribution.  Must agree with: src/bsdfs/diffuse.cpp:110-150, roughconductor.cpp:257-420,
// roughdielectric.cpp:270-614, coating.cpp:208-376, microfacet.h:45-721.  The record is the slice
// of BSDFSamplingRecord (bsdf.h:123-192) that MIPathTracer::Li sets: typeMask = EAll,
// component = -1, mode = ERadiance.  Coating nests one level (a non-coating BSDF underneath), which is
// what the reference's own fixtures use (data/tests/test_bsdf.xml).
#pragma once
#include "b2_math.cuh"
#include "b2_types.h"
#include "b2_sampler.cuh"

namespace b2 {

// include/mitsuba/render/bsdf.h:224-285
enum : uint32_t {
    ENull = 0x00001, EDiffuseReflection = 0x00002, EDiffuseTransmission = 0x00004, EGlossyReflection = 0x00008,
    EGlossyTransmission = 0x00010, EDeltaReflection = 0x00020, EDeltaTransmission = 0x00040, EDelta1DReflection = 0x00080,
    EDelta1DTransmission = 0x00100, EAnisotropic = 0x01000, ENonSymmetric = 0x04000, EFrontSide = 0x08000, EBackSide = 0x10000,
    EUsesSampler = 0x20000,
    ETransmission = EDiffuseTransmission | EDeltaTransmission | EDelta1DTransmission | EGlossyTransmission | ENull,
    EDiffuse = EDiffuseReflection | EDiffuseTransmission, EGlossy = EGlossyReflection | EGlossyTransmission,
    ESmooth = EDiffuse | EGlossy, EDelta = ENull | EDeltaReflection | EDeltaTransmission,
    EDelta1D = EDelta1DReflection | EDelta1DTransmission, EAll = EDiffuse | EGlossy | EDelta | EDelta1D
};

struct Microfacet {
    int type;
    float alphaU, alphaV;
    bool visible;
    float exponentU, exponentV;

    B2_DEV void init(int t, float aU, float aV, bool sv) {
        type = t; visible = sv;
        alphaU = fmaxf(aU, 1e-4f); alphaV = fmaxf(aV, 1e-4f); // microfacet.h:70-71
        exponentU = exponentV = 0.0f;
        if (type == 2) computePhongExponent();
    }
    B2_DEV void computePhongExponent() { // :693-696
        exponentU = fmaxf(2.0f / (alphaU * alphaU) - 2.0f, 0.0f);
        exponentV = fmaxf(2.0f / (alphaV * alphaV) - 2.0f, 0.0f);
    }
    B2_DEV bool isIsotropic() const { return alphaU == alphaV; }
    B2_DEV void scaleAlpha(float v) { alphaU *= v; alphaV *= v; if (type == 2) computePhongExponent(); }
    B2_DEV float interpolatePhongExponent(const V3 &v) const { // :554-565
        const float st2 = sinTheta2(v);
        if (isIsotropic() || st2 <= B2_RCPOVERFLOW) return exponentU;
        float invSinTheta2 = 1 / st2;
        float cosPhi2 = v.x * v.x * invSinTheta2, sinPhi2 = v.y * v.y * invSinTheta2;
        return exponentU * cosPhi2 + exponentV * sinPhi2;
    }
    B2_DEV float eval(const V3 &m) const { // :191-234
        if (cosTheta(m) <= 0) return 0.0f;
        float ct2 = cosTheta2(m);
        float beckmannExponent = ((m.x * m.x) / (alphaU * alphaU) + (m.y * m.y) / (alphaV * alphaV)) / ct2;
        float result;
        if (type == 0) {
            result = fastexp(-beckmannExponent) / (B2_PI * alphaU * alphaV * ct2 * ct2);
        } else if (type == 1) {
            float root = (1.0f + beckmannExponent) * ct2;
            result = 1.0f / (B2_PI * alphaU * alphaV * root * root);
        } else {
            float exponent = interpolatePhongExponent(m);
            result = sqrtf((exponentU + 2) * (exponentV + 2)) * B2_INV_TWOPI * powf(cosTheta(m), exponent);
        }
        if (result * cosTheta(m) < 1e-20f) result = 0;
        return result;
    }
    B2_DEV float projectRoughness(const V3 &v) const { // :541-551
        float invSinTheta2 = 1 / sinTheta2(v);
        if (isIsotropic() || invSinTheta2 <= 0) return alphaU;
        float cosPhi2 = v.x * v.x * invSinTheta2, sinPhi2 = v.y * v.y * invSinTheta2;
        return sqrtf(cosPhi2 * alphaU * alphaU + sinPhi2 * alphaV * alphaV);
    }
    B2_DEV float smithG1(const V3 &v, const V3 &m) const { // :477-514
        if (dot(v, m) * cosTheta(v) <= 0) return 0.0f;
        float tt = fabsf(tanTheta(v));
        if (tt == 0.0f) return 1.0f;
        float alpha = projectRoughness(v);
        if (type == 1) {
            float root = alpha * tt;
            return 2.0f / (1.0f + hypot2(1.0f, root));
        }
        float a = 1.0f / (alpha * tt);
        if (a >= 1.6f) return 1.0f;
        float aSqr = a * a;
        return (3.535f * a + 2.181f * aSqr) / (1.0f + 2.276f * a + 2.577f * aSqr);
    }
    B2_DEV float G(const V3 &wi, const V3 &wo, const V3 &m) const { return smithG1(wi, m) * smithG1(wo, m); }
    B2_DEV void sampleFirstQuadrant(float u1, float &phi, float &exponent) const { // :699-708
        float cosPhi, sinPhi;
        phi = atanf(sqrtf((exponentU + 2.0f) / (exponentV + 2.0f)) * tanf(B2_PI * u1 * 0.5f));
        sincosf(phi, &sinPhi, &cosPhi);
        exponent = exponentU * cosPhi * cosPhi + exponentV * sinPhi * sinPhi;
    }
    B2_DEV V3 sampleAll(float sx, float sy, float &pdf) const { // :287-395
        float cosThetaM = 0.0f, sinPhiM, cosPhiM, alphaSqr;
        if (type == 0 || type == 1) {
            if (isIsotropic()) {
                sincosf((2.0f * B2_PI) * sy, &sinPhiM, &cosPhiM);
                alphaSqr = alphaU * alphaU;
            } else {
                float phiM = atanf(alphaV / alphaU * tanf(B2_PI + 2 * B2_PI * sy)) + B2_PI * floorf(2 * sy + 0.5f);
                sincosf(phiM, &sinPhiM, &cosPhiM);
                float cosSc = cosPhiM / alphaU, sinSc = sinPhiM / alphaV;
                alphaSqr = 1.0f / (cosSc * cosSc + sinSc * sinSc);
            }
            if (type == 0) {
                float tanThetaMSqr = alphaSqr * -fastlog(1.0f - sx);
                cosThetaM = 1.0f / sqrtf(1.0f + tanThetaMSqr);
                pdf = (1.0f - sx) / (B2_PI * alphaU * alphaV * cosThetaM * cosThetaM * cosThetaM);
            } else {
                float tanThetaMSqr = alphaSqr * sx / (1.0f - sx);
                cosThetaM = 1.0f / sqrtf(1.0f + tanThetaMSqr);
                float temp = 1 + tanThetaMSqr / alphaSqr;
                pdf = B2_INV_PI / (alphaU * alphaV * cosThetaM * cosThetaM * cosThetaM * temp * temp);
            }
        } else {
            float phiM, exponent;
            if (isIsotropic()) {
                phiM = (2.0f * B2_PI) * sy;
                exponent = exponentU;
            } else {
                if (sy < 0.25f) { sampleFirstQuadrant(4 * sy, phiM, exponent); }
                else if (sy < 0.5f) { sampleFirstQuadrant(4 * (0.5f - sy), phiM, exponent); phiM = B2_PI - phiM; }
                else if (sy < 0.75f) { sampleFirstQuadrant(4 * (sy - 0.5f), phiM, exponent); phiM += B2_PI; }
                else { sampleFirstQuadrant(4 * (1 - sy), phiM, exponent); phiM = 2 * B2_PI - phiM; }
            }
            sincosf(phiM, &sinPhiM, &cosPhiM);
            cosThetaM = powf(sx, 1.0f / (exponent + 2.0f));
            pdf = sqrtf((exponentU + 2.0f) * (exponentV + 2.0f)) * B2_INV_TWOPI * powf(cosThetaM, exponent + 1.0f);
        }
        if (pdf < 1e-20f) pdf = 0;
        float sinThetaM = sqrtf(fmaxf(0.0f, 1 - cosThetaM * cosThetaM));
        return V3(sinThetaM * cosPhiM, sinThetaM * sinPhiM, cosThetaM);
    }
    B2_DEV float pdfAll(const V3 &m) const { return eval(m) * cosTheta(m); }
    B2_DEV void sampleVisible11(float thetaI, float sx, float sy, float &slopeX, float &slopeY) const { // :573-690
        const float SQRT_PI_INV = 1 / sqrtf(B2_PI);
        if (type == 0) {
            if (thetaI < 1e-4f) {
                float sinPhi, cosPhi;
                float r = sqrtf(-fastlog(1.0f - sx));
                sincosf(2 * B2_PI * sy, &sinPhi, &cosPhi);
                slopeX = r * cosPhi; slopeY = r * sinPhi;
                return;
            }
            float tanThetaI = tanf(thetaI);
            float cotThetaI = 1 / tanThetaI;
            float a = -1, c = erf_as(cotThetaI);
            float sample_x = fmaxf(sx, 1e-6f);
            float fit = 1 + thetaI * (-0.876f + thetaI * (0.4265f - 0.0594f * thetaI));
            float b = c - (1 + c) * powf(1 - sample_x, fit);
            float normalization = 1 / (1 + c + SQRT_PI_INV * tanThetaI * expf(-cotThetaI * cotThetaI));
            int it = 0;
            while (++it < 10) {
                if (!(b >= a && b <= c)) b = 0.5f * (a + c);
                float invErf = erfinv_giles(b);
                float value = normalization * (1 + b + SQRT_PI_INV * tanThetaI * expf(-invErf * invErf)) - sample_x;
                float derivative = normalization * (1 - invErf * tanThetaI);
                if (fabsf(value) < 1e-5f) break;
                if (value > 0) c = b; else a = b;
                b -= value / derivative;
            }
            slopeX = erfinv_giles(b);
            slopeY = erfinv_giles(2.0f * fmaxf(sy, 1e-6f) - 1.0f);
        } else {
            if (thetaI < 1e-4f) {
                float sinPhi, cosPhi;
                float r = safe_sqrt(sx / (1 - sx));
                sincosf(2 * B2_PI * sy, &sinPhi, &cosPhi);
                slopeX = r * cosPhi; slopeY = r * sinPhi;
                return;
            }
            float tanThetaI = tanf(thetaI);
            float a = 1 / tanThetaI;
            float G1 = 2.0f / (1.0f + safe_sqrt(1.0f + 1.0f / (a * a)));
            float A = 2.0f * sx / G1 - 1.0f;
            if (fabsf(A) == 1) A -= signum(A) * B2_EPSILON;
            float tmp = 1.0f / (A * A - 1.0f);
            float B = tanThetaI;
            float D = safe_sqrt(B * B * tmp * tmp - (A * A - B * B) * tmp);
            float slope_x_1 = B * tmp - D;
            float slope_x_2 = B * tmp + D;
            slopeX = (A < 0.0f || slope_x_2 > 1.0f / tanThetaI) ? slope_x_1 : slope_x_2;
            float S;
            if (sy > 0.5f) { S = 1.0f; sy = 2.0f * (sy - 0.5f); }
            else { S = -1.0f; sy = 2.0f * (0.5f - sy); }
            float z = (sy * (sy * (sy * (-0.365728915865723f) + 0.790235037209296f) - 0.424965825137544f) + 0.000152998850436920f) /
                      (sy * (sy * (sy * (sy * 0.169507819808272f - 0.397203533833404f) - 0.232500544458471f) + 1.0f) - 0.539825872510702f);
            slopeY = S * z * sqrtf(1.0f + slopeX * slopeX);
        }
    }
    B2_DEV V3 sampleVisible(const V3 &_wi, float sx, float sy) const { // :421-459
        V3 wi = normalize(V3(alphaU * _wi.x, alphaV * _wi.y, _wi.z));
        float theta = 0, phi = 0;
        if (wi.z < 0.99999f) { theta = acosf(wi.z); phi = atan2f(wi.y, wi.x); }
        float sinPhi, cosPhi;
        sincosf(phi, &sinPhi, &cosPhi);
        float slx, sly;
        sampleVisible11(theta, sx, sy, slx, sly);
        float rx = cosPhi * slx - sinPhi * sly, ry = sinPhi * slx + cosPhi * sly;
        rx *= alphaU; ry *= alphaV;
        float normalization = 1.0f / sqrtf(rx * rx + ry * ry + 1.0f);
        return V3(-rx * normalization, -ry * normalization, normalization);
    }
    B2_DEV float pdfVisible(const V3 &wi, const V3 &m) const { // :462-466
        if (cosTheta(wi) == 0) return 0.0f;
        return smithG1(wi, m) * absDot(wi, m) * eval(m) / fabsf(cosTheta(wi));
    }
    B2_DEV V3 sample(const V3 &wi, float sx, float sy, float &pdf) const { // :236-246
        V3 m;
        if (visible) { m = sampleVisible(wi, sx, sy); pdf = pdfVisible(wi, m); }
        else m = sampleAll(sx, sy, pdf);
        return m;
    }
    B2_DEV float pdf(const V3 &wi, const V3 &m) const { return visible ? pdfVisible(wi, m) : pdfAll(m); }
};

struct BRec {
    V3 wi, wo;
    float eta;
    uint32_t sampledType;
    // value of the bitmap texture bound to the diffuse reflectance of the leaf BSDF this record will reach (`m_reflectance->eval(bRec.its)`,
    // diffuse.cpp:115,148), looked up once per intersection by the caller; hasTex is a compile-time false in the kernels for untextured scenes
    bool hasTex = false;
    V3 texR;
};

B2_DEV V3 ld3(const float *p) { return V3(p[0], p[1], p[2]); }

// ---------------------------------------------------------------------------------------------
// leaf BSDFs (types 0..2)
// ---------------------------------------------------------------------------------------------
template <int HINT> B2_DEV Spectrum leafEval(const DMaterial &d, const BRec &r, bool discrete) {
    const V3 R = (r.hasTex && (d.type == 0 || d.type == 1 || d.type == 7)) ? r.texR : ld3(d.reflectance); // diffuse reflectance, (rough)conductor specularReflectance
    const int type = (HINT >= 0 && HINT < 3) ? HINT : d.type;
    if (type == 4) return Spectrum(discrete ? 1.0f : 0.0f); // null.cpp:45-47 (index-matched boundary)
    if (type == 6) { // dielectric.cpp:229-255
        float cosThetaT;
        const float F = fresnelDielectricExt(cosTheta(r.wi), cosThetaT, d.eta);
        const float invEta = 1 / d.eta;
        if (cosTheta(r.wi) * cosTheta(r.wo) >= 0) {
            if (!discrete || fabsf(dot(V3(-r.wi.x, -r.wi.y, r.wi.z), r.wo) - 1) > B2_DELTA_EPSILON) return Spectrum(0.0f);
            return R * F;
        }
        const float scale = -(cosThetaT < 0 ? invEta : d.eta);
        if (!discrete || fabsf(dot(V3(scale * r.wi.x, scale * r.wi.y, cosThetaT), r.wo) - 1) > B2_DELTA_EPSILON) return Spectrum(0.0f);
        const float factor = cosThetaT < 0 ? invEta : d.eta;
        return ld3(d.transmittance) * factor * factor * (1 - F);
    }
    if (type == 7) { // conductor.cpp:221-235
        if (!discrete || cosTheta(r.wi) <= 0 || cosTheta(r.wo) <= 0 || fabsf(dot(V3(-r.wi.x, -r.wi.y, r.wi.z), r.wo) - 1) > B2_DELTA_EPSILON) return Spectrum(0.0f);
        return R * fresnelConductorExact(cosTheta(r.wi), ld3(d.etaC), ld3(d.kC));
    }
    if (type == 8) { // plastic.cpp:243-279
        if (cosTheta(r.wo) <= 0 || cosTheta(r.wi) <= 0) return Spectrum(0.0f);
        const float Fi = fresnelDielectricExt(cosTheta(r.wi), d.eta);
        if (discrete) {
            if (fabsf(dot(V3(-r.wi.x, -r.wi.y, r.wi.z), r.wo) - 1) < B2_DELTA_EPSILON) return R * Fi;
            return Spectrum(0.0f);
        }
        const float Fo = fresnelDielectricExt(cosTheta(r.wo), d.eta);
        Spectrum diff = r.hasTex ? r.texR : ld3(d.diffuseReflectance); // the caller resolves the bitmap texture of plastic's diffuseReflectance
        if (d.nonlinear) diff = diff / (Spectrum(1.0f) - diff * d.fdrInt);
        else diff = diff / (1 - d.fdrInt);
        const float invEta2 = 1 / (d.eta * d.eta);
        return diff * (squareToCosineHemispherePdf(r.wo) * invEta2 * (1 - Fi) * (1 - Fo));
    }
    if (type == 0) { // diffuse.cpp:110-118
        if (discrete || d.flags == 0 || cosTheta(r.wi) <= 0 || cosTheta(r.wo) <= 0) return Spectrum(0.0f);
        return R * (B2_INV_PI * cosTheta(r.wo));
    } else if (type == 1) { // roughconductor.cpp:257-297
        if (discrete || cosTheta(r.wi) <= 0 || cosTheta(r.wo) <= 0) return Spectrum(0.0f);
        V3 H = normalize(r.wo + r.wi);
        Microfacet ds; ds.init(d.distr, d.alphaU, d.alphaV, d.sampleVisible != 0);
        const float D = ds.eval(H);
        if (D == 0) return Spectrum(0.0f);
        const Spectrum F = fresnelConductorExact(dot(r.wi, H), ld3(d.etaC), ld3(d.kC)) * R;
        const float G = ds.G(r.wi, r.wo, H);
        float model = D * G / (4.0f * cosTheta(r.wi));
        return F * model;
    } else { // roughdielectric.cpp:270-349
        if (discrete || cosTheta(r.wi) == 0) return Spectrum(0.0f);
        const float m_eta = d.eta, m_invEta = 1 / d.eta;
        bool reflect = cosTheta(r.wi) * cosTheta(r.wo) > 0;
        V3 H;
        if (reflect) H = normalize(r.wo + r.wi);
        else { float eta = cosTheta(r.wi) > 0 ? m_eta : m_invEta; H = normalize(r.wi + r.wo * eta); }
        H = H * signum(cosTheta(H));
        Microfacet ds; ds.init(d.distr, d.alphaU, d.alphaV, d.sampleVisible != 0);
        const float D = ds.eval(H);
        if (D == 0) return Spectrum(0.0f);
        const float F = fresnelDielectricExt(dot(r.wi, H), m_eta);
        const float G = ds.G(r.wi, r.wo, H);
        if (reflect) {
            float value = F * D * G / (4.0f * fabsf(cosTheta(r.wi)));
            return R * value;
        } else {
            float eta = cosTheta(r.wi) > 0.0f ? m_eta : m_invEta;
            float sqrtDenom = dot(r.wi, H) + eta * dot(r.wo, H);
            float value = ((1 - F) * D * G * eta * eta * dot(r.wi, H) * dot(r.wo, H)) / (cosTheta(r.wi) * sqrtDenom * sqrtDenom);
            float factor = cosTheta(r.wi) > 0 ? m_invEta : m_eta;
            return ld3(d.transmittance) * fabsf(value * factor * factor);
        }
    }
}

template <int HINT> B2_DEV float leafPdf(const DMaterial &d, const BRec &r, bool discrete) {
    const int type = (HINT >= 0 && HINT < 3) ? HINT : d.type;
    if (type == 4) return discrete ? 1.0f : 0.0f; // null.cpp:49-51
    if (type == 6) { // dielectric.cpp:257-279
        float cosThetaT;
        const float F = fresnelDielectricExt(cosTheta(r.wi), cosThetaT, d.eta);
        const float invEta = 1 / d.eta;
        if (cosTheta(r.wi) * cosTheta(r.wo) >= 0) {
            if (!discrete || fabsf(dot(V3(-r.wi.x, -r.wi.y, r.wi.z), r.wo) - 1) > B2_DELTA_EPSILON) return 0.0f;
            return F;
        }
        const float scale = -(cosThetaT < 0 ? invEta : d.eta);
        if (!discrete || fabsf(dot(V3(scale * r.wi.x, scale * r.wi.y, cosThetaT), r.wo) - 1) > B2_DELTA_EPSILON) return 0.0f;
        return 1 - F;
    }
    if (type == 7) { // conductor.cpp:237-250
        if (!discrete || cosTheta(r.wi) <= 0 || cosTheta(r.wo) <= 0 || fabsf(dot(V3(-r.wi.x, -r.wi.y, r.wi.z), r.wo) - 1) > B2_DELTA_EPSILON) return 0.0f;
        return 1.0f;
    }
    if (type == 8) { // plastic.cpp:281-309
        if (cosTheta(r.wo) <= 0 || cosTheta(r.wi) <= 0) return 0.0f;
        const float Fi = fresnelDielectricExt(cosTheta(r.wi), d.eta);
        const float w = d.specSamplingWeight;
        const float probSpecular = (Fi * w) / (Fi * w + (1 - Fi) * (1 - w));
        if (discrete) return fabsf(dot(V3(-r.wi.x, -r.wi.y, r.wi.z), r.wo) - 1) < B2_DELTA_EPSILON ? probSpecular : 0.0f;
        return squareToCosineHemispherePdf(r.wo) * (1 - probSpecular);
    }
    if (type == 0) { // diffuse.cpp:120-128
        if (discrete || d.flags == 0 || cosTheta(r.wi) <= 0 || cosTheta(r.wo) <= 0) return 0.0f;
        return squareToCosineHemispherePdf(r.wo);
    } else if (type == 1) { // roughconductor.cpp:299-326
        if (discrete || cosTheta(r.wi) <= 0 || cosTheta(r.wo) <= 0) return 0.0f;
        V3 H = normalize(r.wo + r.wi);
        Microfacet ds; ds.init(d.distr, d.alphaU, d.alphaV, d.sampleVisible != 0);
        if (ds.visible) return ds.eval(H) * ds.smithG1(r.wi, H) / (4.0f * cosTheta(r.wi));
        else return ds.pdf(r.wi, H) / (4 * absDot(r.wo, H));
    } else { // roughdielectric.cpp:351-417
        if (discrete) return 0.0f;
        const float m_eta = d.eta, m_invEta = 1 / d.eta;
        bool reflect = cosTheta(r.wi) * cosTheta(r.wo) > 0;
        V3 H;
        float dwh_dwo;
        if (reflect) {
            H = normalize(r.wo + r.wi);
            dwh_dwo = 1.0f / (4.0f * dot(r.wo, H));
        } else {
            float eta = cosTheta(r.wi) > 0 ? m_eta : m_invEta;
            H = normalize(r.wi + r.wo * eta);
            float sqrtDenom = dot(r.wi, H) + eta * dot(r.wo, H);
            dwh_dwo = (eta * eta * dot(r.wo, H)) / (sqrtDenom * sqrtDenom);
        }
        H = H * signum(cosTheta(H));
        Microfacet sd; sd.init(d.distr, d.alphaU, d.alphaV, d.sampleVisible != 0);
        if (!sd.visible) sd.scaleAlpha(1.2f - 0.2f * sqrtf(fabsf(cosTheta(r.wi))));
        float prob = sd.pdf(signum(cosTheta(r.wi)) * r.wi, H);
        float F = fresnelDielectricExt(dot(r.wi, H), m_eta);
        prob *= reflect ? F : (1 - F);
        return fabsf(prob * dwh_dwo);
    }
}

template <int HINT, typename Smp = PathSampler> B2_DEV Spectrum leafSample(const DMaterial &d, BRec &r, float &pdfOut, float sx, float sy, Smp &smp) {
    const V3 R = (r.hasTex && (d.type == 0 || d.type == 1 || d.type == 7)) ? r.texR : ld3(d.reflectance); // diffuse reflectance, (rough)conductor specularReflectance
    const int type = (HINT >= 0 && HINT < 3) ? HINT : d.type;
    if (type == 4) { // null.cpp:65-76
        r.wo = -r.wi; r.sampledType = ENull; r.eta = 1.0f; pdfOut = 1.0f;
        return Spectrum(1.0f);
    }
    if (type == 6) { // dielectric.cpp:281-310 (both components enabled)
        float cosThetaT;
        const float F = fresnelDielectricExt(cosTheta(r.wi), cosThetaT, d.eta);
        const float invEta = 1 / d.eta;
        if (sx <= F) {
            r.sampledType = EDeltaReflection;
            r.wo = V3(-r.wi.x, -r.wi.y, r.wi.z);
            r.eta = 1.0f;
            pdfOut = F;
            return R;
        }
        r.sampledType = EDeltaTransmission;
        const float scale = -(cosThetaT < 0 ? invEta : d.eta);
        r.wo = V3(scale * r.wi.x, scale * r.wi.y, cosThetaT);
        r.eta = cosThetaT < 0 ? d.eta : invEta;
        pdfOut = 1 - F;
        const float factor = cosThetaT < 0 ? invEta : d.eta;
        return ld3(d.transmittance) * (factor * factor);
    }
    if (type == 7) { // conductor.cpp:268-283
        if (cosTheta(r.wi) <= 0) return Spectrum(0.0f);
        r.sampledType = EDeltaReflection;
        r.wo = V3(-r.wi.x, -r.wi.y, r.wi.z);
        r.eta = 1.0f;
        pdfOut = 1.0f;
        return R * fresnelConductorExact(cosTheta(r.wi), ld3(d.etaC), ld3(d.kC));
    }
    if (type == 8) { // plastic.cpp:377-424 (both components enabled)
        if (cosTheta(r.wi) <= 0) return Spectrum(0.0f);
        const float Fi = fresnelDielectricExt(cosTheta(r.wi), d.eta);
        r.eta = 1.0f;
        const float w = d.specSamplingWeight;
        const float probSpecular = (Fi * w) / (Fi * w + (1 - Fi) * (1 - w));
        if (sx < probSpecular) {
            r.sampledType = EDeltaReflection;
            r.wo = V3(-r.wi.x, -r.wi.y, r.wi.z);
            pdfOut = probSpecular;
            return R * Fi / probSpecular;
        }
        r.sampledType = EDiffuseReflection;
        r.wo = squareToCosineHemisphere((sx - probSpecular) / (1 - probSpecular), sy);
        const float Fo = fresnelDielectricExt(cosTheta(r.wo), d.eta);
        Spectrum diff = r.hasTex ? r.texR : ld3(d.diffuseReflectance); // the caller resolves the bitmap texture of plastic's diffuseReflectance
        if (d.nonlinear) diff = diff / (Spectrum(1.0f) - diff * d.fdrInt);
        else diff = diff / (1 - d.fdrInt);
        pdfOut = (1 - probSpecular) * squareToCosineHemispherePdf(r.wo);
        const float invEta2 = 1 / (d.eta * d.eta);
        return diff * (invEta2 * (1 - Fi) * (1 - Fo) / (1 - probSpecular));
    }
    if (type == 0) { // diffuse.cpp:141-150
        if (d.flags == 0 || cosTheta(r.wi) <= 0) return Spectrum(0.0f);
        r.wo = squareToCosineHemisphere(sx, sy);
        r.eta = 1.0f; r.sampledType = EDiffuseReflection;
        pdfOut = squareToCosineHemispherePdf(r.wo);
        return R;
    } else if (type == 1) { // roughconductor.cpp:372-420
        if (cosTheta(r.wi) < 0) return Spectrum(0.0f);
        Microfacet ds; ds.init(d.distr, d.alphaU, d.alphaV, d.sampleVisible != 0);
        V3 m = ds.sample(r.wi, sx, sy, pdfOut);
        if (pdfOut == 0) return Spectrum(0.0f);
        r.wo = reflect(r.wi, m);
        r.eta = 1.0f; r.sampledType = EGlossyReflection;
        if (cosTheta(r.wo) <= 0) return Spectrum(0.0f);
        Spectrum F = fresnelConductorExact(dot(r.wi, m), ld3(d.etaC), ld3(d.kC)) * R;
        float weight;
        if (ds.visible) weight = ds.smithG1(r.wo, m);
        else weight = ds.eval(m) * ds.G(r.wi, r.wo, m) * dot(r.wi, m) / (pdfOut * cosTheta(r.wi));
        pdfOut /= 4.0f * dot(r.wo, m);
        return F * weight;
    } else { // roughdielectric.cpp:515-614
        const float m_eta = d.eta, m_invEta = 1 / d.eta;
        bool sampleReflection = true;
        Microfacet ds; ds.init(d.distr, d.alphaU, d.alphaV, d.sampleVisible != 0);
        Microfacet sd = ds;
        if (!ds.visible) sd.scaleAlpha(1.2f - 0.2f * sqrtf(fabsf(cosTheta(r.wi))));
        float microfacetPDF;
        const V3 m = sd.sample(signum(cosTheta(r.wi)) * r.wi, sx, sy, microfacetPDF);
        if (microfacetPDF == 0) return Spectrum(0.0f);
        pdfOut = microfacetPDF;
        float cosThetaT;
        float F = fresnelDielectricExt(dot(r.wi, m), cosThetaT, m_eta);
        Spectrum weight(1.0f);
        if (smp.next1D() > F) { sampleReflection = false; pdfOut *= 1 - F; }
        else pdfOut *= F;
        float dwh_dwo;
        if (sampleReflection) {
            r.wo = reflect(r.wi, m);
            r.eta = 1.0f; r.sampledType = EGlossyReflection;
            if (cosTheta(r.wi) * cosTheta(r.wo) <= 0) return Spectrum(0.0f);
            weight = weight * R;
            dwh_dwo = 1.0f / (4.0f * dot(r.wo, m));
        } else {
            if (cosThetaT == 0) return Spectrum(0.0f);
            r.wo = refract(r.wi, m, m_eta, cosThetaT);
            r.eta = cosThetaT < 0 ? m_eta : m_invEta;
            r.sampledType = EGlossyTransmission;
            if (cosTheta(r.wi) * cosTheta(r.wo) >= 0) return Spectrum(0.0f);
            float factor = cosThetaT < 0 ? m_invEta : m_eta;
            weight = weight * (ld3(d.transmittance) * (factor * factor));
            float sqrtDenom = dot(r.wi, m) + r.eta * dot(r.wo, m);
            dwh_dwo = (r.eta * r.eta * dot(r.wo, m)) / (sqrtDenom * sqrtDenom);
        }
        if (ds.visible) weight = weight * ds.smithG1(r.wo, m);
        else weight = weight * fabsf(ds.eval(m) * ds.G(r.wi, r.wo, m) * dot(r.wi, m) / (microfacetPDF * cosTheta(r.wi)));
        pdfOut *= fabsf(dwh_dwo);
        return weight;
    }
}

// ---------------------------------------------------------------------------------------------
// coating wrapper (coating.cpp)
// ---------------------------------------------------------------------------------------------
B2_DEV V3 coatRefractIn(const DMaterial &d, const V3 &wi, float &R) { // coating.cpp:193-198
    float cosThetaT, invEta = 1 / d.eta;
    R = fresnelDielectricExt(fabsf(cosTheta(wi)), cosThetaT, d.eta);
    return V3(invEta * wi.x, invEta * wi.y, -signum(cosTheta(wi)) * cosThetaT);
}
B2_DEV V3 coatRefractOut(const DMaterial &d, const V3 &wi, float &R) { // coating.cpp:200-205
    float cosThetaT, invEta = 1 / d.eta;
    R = fresnelDielectricExt(fabsf(cosTheta(wi)), cosThetaT, invEta);
    return V3(d.eta * wi.x, d.eta * wi.y, -signum(cosTheta(wi)) * cosThetaT);
}

template <int HINT> B2_DEV Spectrum bsdfEval1(const DMaterial *mats, int id, const BRec &r) {
    const DMaterial &d = mats[id];
    if (HINT >= 0 && HINT < 3) return leafEval<HINT>(d, r, false);
    if (HINT != 3 && d.type != 3) return leafEval<-1>(d, r, false);
    // coating.cpp:208-248 with measure == ESolidAngle (the specular branch needs EDiscrete)
    const DMaterial &nd = mats[d.nested];
    const float m_invEta = 1 / d.eta;
    if ((nd.flags & EAll) == 0) return Spectrum(0.0f);
    float R12, R21;
    BRec ri = r;
    ri.wi = coatRefractIn(d, r.wi, R12);
    ri.wo = coatRefractIn(d, r.wo, R21);
    if (R12 == 1 || R21 == 1) return Spectrum(0.0f);
    Spectrum result = leafEval<-1>(nd, ri, false) * (1 - R12) * (1 - R21);
    Spectrum sigmaA = ld3(d.sigmaA) * d.thickness;
    if (!isZero(sigmaA)) result = result * expSpec(-sigmaA * (1 / fabsf(cosTheta(ri.wi)) + 1 / fabsf(cosTheta(ri.wo))));
    result = result * (m_invEta * m_invEta * cosTheta(r.wo) / cosTheta(ri.wo));
    return result;
}

template <int HINT> B2_DEV float bsdfPdf1(const DMaterial *mats, int id, const BRec &r) {
    const DMaterial &d = mats[id];
    if (HINT >= 0 && HINT < 3) return leafPdf<HINT>(d, r, false);
    if (HINT != 3 && d.type != 3) return leafPdf<-1>(d, r, false);
    // coating.cpp:250-286
    const DMaterial &nd = mats[d.nested];
    const float m_invEta = 1 / d.eta;
    if ((nd.flags & EAll) == 0) return 0.0f;
    float R12;
    V3 wiPrime = coatRefractIn(d, r.wi, R12);
    float w = d.specSamplingWeight;
    float probSpecular = (R12 * w) / (R12 * w + (1 - R12) * (1 - w));
    float R21;
    BRec ri = r;
    ri.wi = wiPrime;
    ri.wo = coatRefractIn(d, r.wo, R21);
    if (R12 == 1 || R21 == 1) return 0.0f;
    float p = leafPdf<-1>(nd, ri, false);
    p *= m_invEta * m_invEta * cosTheta(r.wo) / cosTheta(ri.wo);
    return p * (1 - probSpecular);
}

template <int HINT, typename Smp = PathSampler> B2_DEV Spectrum bsdfSample1(const DMaterial *mats, int id, BRec &r, float &pdfOut, float sx, float sy, Smp &smp) {
    const DMaterial &d = mats[id];
    if (HINT >= 0 && HINT < 3) return leafSample<HINT>(d, r, pdfOut, sx, sy, smp);
    if (HINT != 3 && d.type != 3) return leafSample<-1>(d, r, pdfOut, sx, sy, smp);
    // coating.cpp:288-371
    const DMaterial &nd = mats[d.nested];
    const float m_invEta = 1 / d.eta;
    bool sampleNested = (nd.flags & EAll) != 0;
    float R12;
    V3 wiPrime = coatRefractIn(d, r.wi, R12);
    float w = d.specSamplingWeight;
    float probSpecular = (R12 * w) / (R12 * w + (1 - R12) * (1 - w));
    bool choseSpecular = true;
    if (sampleNested) {
        if (sx < probSpecular) sx /= probSpecular;
        else { sx = (sx - probSpecular) / (1 - probSpecular); choseSpecular = false; }
    }
    if (choseSpecular) {
        r.sampledType = EDeltaReflection;
        r.wo = V3(-r.wi.x, -r.wi.y, r.wi.z);
        r.eta = 1.0f;
        pdfOut = sampleNested ? probSpecular : 1.0f;
        return ld3(d.reflectance) * (R12 / pdfOut);
    }
    if (R12 == 1.0f) return Spectrum(0.0f);
    V3 wiBackup = r.wi;
    r.wi = wiPrime;
    Spectrum result = leafSample<-1>(nd, r, pdfOut, sx, sy, smp);
    r.wi = wiBackup;
    if (isZero(result)) return Spectrum(0.0f);
    V3 woPrime = r.wo;
    Spectrum sigmaA = ld3(d.sigmaA) * d.thickness;
    if (!isZero(sigmaA)) result = result * expSpec(-sigmaA * (1 / fabsf(cosTheta(wiPrime)) + 1 / fabsf(cosTheta(woPrime))));
    float R21;
    r.wo = coatRefractOut(d, woPrime, R21);
    if (R21 == 1.0f) return Spectrum(0.0f);
    pdfOut *= 1.0f - probSpecular;
    result = result / (1.0f - probSpecular);
    result = result * ((1 - R12) * (1 - R21));
    if (!(r.sampledType & EDelta)) pdfOut *= m_invEta * m_invEta * cosTheta(r.wo) / cosTheta(woPrime);
    return result;
}

// ---------------------------------------------------------------------------------------------
// top level: the twosided adapter (twosided.cpp:109-184) around everything else; only the generic instantiation (HINT < 0)
// can meet it -- the class-specialised kernels are launched for scenes whose materials are all of types 0..3
// ---------------------------------------------------------------------------------------------
template <int HINT> B2_DEV Spectrum bsdfEval(const DMaterial *mats, int id, const BRec &r) {
    if (HINT < 0 && mats[id].type == 5) {
        if (cosTheta(r.wi) > 0) return bsdfEval1<-1>(mats, mats[id].nested, r);
        BRec b = r;
        b.wi.z *= -1; b.wo.z *= -1;
        return bsdfEval1<-1>(mats, mats[id].nested2, b);
    }
    return bsdfEval1<HINT>(mats, id, r);
}
template <int HINT> B2_DEV float bsdfPdf(const DMaterial *mats, int id, const BRec &r) {
    if (HINT < 0 && mats[id].type == 5) {
        if (r.wi.z > 0) return bsdfPdf1<-1>(mats, mats[id].nested, r);
        BRec b = r;
        b.wi.z *= -1; b.wo.z *= -1;
        return bsdfPdf1<-1>(mats, mats[id].nested2, b);
    }
    return bsdfPdf1<HINT>(mats, id, r);
}
template <int HINT, typename Smp = PathSampler> B2_DEV Spectrum bsdfSample(const DMaterial *mats, int id, BRec &r, float &pdfOut, float sx, float sy, Smp &smp) {
    if (HINT < 0 && mats[id].type == 5) {
        bool flipped = false;
        if (cosTheta(r.wi) < 0) { r.wi.z *= -1; flipped = true; }
        const Spectrum result = bsdfSample1<-1>(mats, flipped ? mats[id].nested2 : mats[id].nested, r, pdfOut, sx, sy, smp);
        if (flipped) {
            r.wi.z *= -1;
            if (!isZero(result) && pdfOut != 0) r.wo.z *= -1;
        }
        return result;
    }
    return bsdfSample1<HINT>(mats, id, r, pdfOut, sx, sy, smp);
}

} // namespace b2
