// protocol.cpp -- see protocol.hpp.  Citations are reference file:line.
#include "protocol.hpp"

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <set>

#include "../../include/ertgpu_resample.h"
#include "../../include/ertgpu_signal.h"

namespace {

std::string sprintf_str(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
std::string sprintf_str(const char* fmt, ...) {
    char buf[256];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    return buf;
}

uint64_t bits_uint(const std::string& bits, int from, int to) {  // strconv.ParseUint(bits[from:to], 2, ..)
    uint64_t v = 0;
    for (int i = from; i < to; i++) v = (v << 1) | (uint64_t)(bits[(size_t)i] == '1');
    return v;
}
uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
uint16_t be16(const uint8_t* p) { return (uint16_t)(((uint16_t)p[0] << 8) | p[1]); }
std::string hexbytes(const uint8_t* p, size_t n) {  // fmt "%02X" applied to a []byte
    std::string s;
    for (size_t i = 0; i < n; i++) s += sprintf_str("%02X", p[i]);
    return s;
}
std::string u(uint64_t v) { return std::to_string(v); }
std::string hex0x(uint64_t v) { return sprintf_str("0x%llx", (unsigned long long)v); }  // "0x"+FormatUint(v,16)

using protocol::Field;
Field fu(const char* name, uint64_t v, const char* attr = nullptr) { return Field{name, attr, Field::UINT, v, {}, {}}; }
Field fattr(const char* name, uint64_t v) { return fu(name, v, name); }  // `xml:",attr"`
Field fbytes(const char* name, const uint8_t* p, size_t n) { return Field{name, nullptr, Field::BYTES, 0, {p, p + n}, {}}; }
Field fu16s(const char* name, const uint16_t* p, size_t n) { return Field{name, nullptr, Field::UINT16S, 0, {}, {p, p + n}}; }

}  // namespace

// ======================================================================= crc
namespace crc {

Table NewTable(uint16_t poly) {
    Table t{};
    for (int i = 0; i < 256; i++) {
        uint16_t c = (uint16_t)(i << 8);
        for (int b = 0; b < 8; b++) c = (c & 0x8000) ? (uint16_t)((c << 1) ^ poly) : (uint16_t)(c << 1);
        t[(size_t)i] = c;
    }
    return t;
}

uint16_t Checksum(uint16_t init, const uint8_t* data, size_t n, const Table& t) {
    uint16_t c = init;
    for (size_t i = 0; i < n; i++) c = (uint16_t)((c << 8) ^ t[(size_t)((c >> 8) ^ data[i])]);
    return c;
}

CRC NewCRC(const std::string& name, uint16_t init, uint16_t poly, uint16_t residue) {
    CRC c;
    c.Name = name;
    c.Init = init;
    c.Poly = poly;
    c.Residue = residue;
    c.tbl = NewTable(poly);
    return c;
}

std::string CRC::String() const {
    return sprintf_str("{Name:%s Init:0x%04X Poly:0x%04X Residue:0x%04X}", Name.c_str(), Init, Poly, Residue);
}

}  // namespace crc

// ======================================================================= gf
namespace gf {

Field::Field() {
    int x = 1;
    for (int i = 0; i < 31; i++) {
        exp[(size_t)i] = exp[(size_t)i + 31] = (uint8_t)x;
        log[(size_t)x] = (uint8_t)i;
        x <<= 1;  // multiply by the generator 2 modulo the polynomial 37 (gf.go:88-101)
        if (x & 32) x ^= 37;
    }
    log[0] = 31;
}

uint8_t Field::Mul(uint8_t x, uint8_t y) const {
    if (x == 0 || y == 0) return 0;
    return exp[(size_t)log[x] + (size_t)log[y]];
}

std::vector<uint8_t> Field::Syndrome(const uint8_t* message, int n, int parity, int offset) const {
    std::vector<uint8_t> syn((size_t)parity);
    for (int idx = 0; idx < parity; idx++) {
        uint8_t s = message[0];
        const uint8_t root = exp[(size_t)((offset + idx) % 31)];
        for (int j = 1; j < n; j++) s = (uint8_t)(Mul(s, root) ^ message[j]);
        syn[(size_t)idx] = s;
    }
    return syn;
}

}  // namespace gf

// ======================================================================= protocol
namespace protocol {

Data NewData(const uint8_t* data, size_t n) {
    Data d;
    d.Bytes.assign(data, data + n);
    d.Bits.reserve(n * 8);
    for (size_t i = 0; i < n; i++)
        for (int k = 7; k >= 0; k--) d.Bits.push_back(((data[i] >> k) & 1) ? '1' : '0');  // "%08b"
    return d;
}

namespace {
std::mutex parser_mutex;
std::map<std::string, NewParserFunc>& registry() {
    static std::map<std::string, NewParserFunc> r;
    return r;
}
}  // namespace

void RegisterParser(const std::string& name, NewParserFunc fn) {
    std::lock_guard<std::mutex> lock(parser_mutex);
    if (!fn) throw std::logic_error("parser: new parser func is nil");                                  // parse.go:32-34
    if (registry().count(name)) throw std::logic_error("parser: parser already registered (" + name + ")");  // parse.go:35-37
    registry()[name] = std::move(fn);
}

ParserPtr NewParser(const std::string& name, int chipLength) {
    std::lock_guard<std::mutex> lock(parser_mutex);
    auto it = registry().find(name);
    if (it == registry().end()) throw std::invalid_argument("invalid message type: \"" + name + "\"\n");  // parse.go:49
    return it->second(chipLength);
}

// ----------------------------------------------------------------------- messages
namespace {

struct SCM : Message {  // scm/scm.go:94-101
    uint32_t ID = 0;
    uint8_t Type = 0, TamperPhy = 0, TamperEnc = 0;
    uint32_t Consumption = 0;
    uint16_t ChecksumVal = 0;
    std::string MsgType() const override { return "SCM"; }
    uint32_t MeterID() const override { return ID; }
    uint8_t MeterType() const override { return Type; }
    std::vector<uint8_t> Checksum() const override { return {(uint8_t)(ChecksumVal >> 8), (uint8_t)ChecksumVal}; }
    std::string String() const override {  // scm.go:139-143
        return sprintf_str("{ID:%8u Type:%2u Tamper:{Phy:%02X Enc:%02X} Consumption:%8u CRC:0x%04X}", ID, Type, TamperPhy,
                           TamperEnc, Consumption, ChecksumVal);
    }
    std::vector<std::string> Record() const override {  // scm.go:145-154
        return {u(ID), u(Type), hex0x(TamperPhy), hex0x(TamperEnc), u(Consumption), hex0x(ChecksumVal)};
    }
    std::vector<Field> Fields() const override {  // scm.go:94-101
        return {fattr("ID", ID), fattr("Type", Type), fattr("TamperPhy", TamperPhy), fattr("TamperEnc", TamperEnc),
                fattr("Consumption", Consumption), fu("ChecksumVal", ChecksumVal, "Checksum")};
    }
};

struct SCMPlus : Message {  // scmplus/scmplus.go:94-102
    uint16_t FrameSync = 0;
    uint8_t ProtocolID = 0, EndpointType = 0;
    uint32_t EndpointID = 0, Consumption = 0;
    uint16_t Tamper = 0, PacketCRC = 0;
    std::string MsgType() const override { return "SCM+"; }
    uint32_t MeterID() const override { return EndpointID; }
    uint8_t MeterType() const override { return EndpointType; }
    std::vector<uint8_t> Checksum() const override { return {(uint8_t)(PacketCRC >> 8), (uint8_t)PacketCRC}; }
    std::string String() const override {  // scmplus.go:129-138
        return sprintf_str("{ProtocolID:0x%02X EndpointType:0x%02X EndpointID:%10u Consumption:%10u Tamper:0x%04X PacketCRC:0x%04X}",
                           ProtocolID, EndpointType, EndpointID, Consumption, Tamper, PacketCRC);
    }
    std::vector<std::string> Record() const override {  // scmplus.go:141-151
        return {hex0x(FrameSync), hex0x(ProtocolID), hex0x(EndpointType), u(EndpointID), u(Consumption), hex0x(Tamper), hex0x(PacketCRC)};
    }
    // scmplus.go:94-102.  PacketCRC's tag `xml:"Checksum,attr",json:"Checksum"` has a comma where StructTag.Get wants a
    // space: the xml key parses, the json key does not, so JSON keeps the Go name.
    std::vector<Field> Fields() const override {
        return {fattr("FrameSync", FrameSync), fattr("ProtocolID", ProtocolID), fattr("EndpointType", EndpointType),
                fattr("EndpointID", EndpointID), fattr("Consumption", Consumption), fattr("Tamper", Tamper),
                fu("PacketCRC", PacketCRC, "Checksum")};
    }
};

std::string join_u16(const uint16_t* v, size_t n) {  // fmt "%d" of a [N]uint16
    std::string s = "[";
    for (size_t i = 0; i < n; i++) s += (i ? " " : "") + u(v[i]);
    return s + "]";
}

struct IDM : Message {  // idm/idm.go:101-119
    uint32_t Preamble = 0;
    uint8_t PacketTypeID = 0, PacketLength = 0, HammingCode = 0, ApplicationVersion = 0, ERTType = 0;
    uint32_t ERTSerialNumber = 0;
    uint8_t ConsumptionIntervalCount = 0, ModuleProgrammingState = 0;
    std::array<uint8_t, 6> TamperCounters{};
    uint16_t AsynchronousCounters = 0;
    std::array<uint8_t, 6> PowerOutageFlags{};
    uint32_t LastConsumptionCount = 0;
    std::array<uint16_t, 47> DifferentialConsumptionIntervals{};
    uint16_t TransmitTimeOffset = 0, SerialNumberCRC = 0, PacketCRC = 0;
    std::string MsgType() const override { return "IDM"; }
    uint32_t MeterID() const override { return ERTSerialNumber; }
    uint8_t MeterType() const override { return ERTType; }
    std::vector<uint8_t> Checksum() const override { return {(uint8_t)(PacketCRC >> 8), (uint8_t)PacketCRC}; }
    std::string String() const override {  // idm.go:177-199
        std::string s = "{";
        s += sprintf_str("Preamble:0x%08X PacketTypeID:0x%02X PacketLength:0x%02X HammingCode:0x%02X ", Preamble, PacketTypeID, PacketLength, HammingCode);
        s += sprintf_str("ApplicationVersion:0x%02X ERTType:0x%02X ERTSerialNumber:% 10lld ", ApplicationVersion, ERTType, (long long)ERTSerialNumber);
        s += sprintf_str("ConsumptionIntervalCount:%u ModuleProgrammingState:0x%02X ", ConsumptionIntervalCount, ModuleProgrammingState);
        s += "TamperCounters:" + hexbytes(TamperCounters.data(), 6) + sprintf_str(" AsynchronousCounters:0x%02X ", AsynchronousCounters);
        s += "PowerOutageFlags:" + hexbytes(PowerOutageFlags.data(), 6) + sprintf_str(" LastConsumptionCount:%u ", LastConsumptionCount);
        s += "DifferentialConsumptionIntervals:" + join_u16(DifferentialConsumptionIntervals.data(), 47);
        s += sprintf_str(" TransmitTimeOffset:%u SerialNumberCRC:0x%04X PacketCRC:0x%04X}", TransmitTimeOffset, SerialNumberCRC, PacketCRC);
        return s;
    }
    std::vector<std::string> Record() const override {  // idm.go:201-221
        std::vector<std::string> r = {sprintf_str("0x%08X", Preamble), sprintf_str("0x%02X", PacketTypeID), sprintf_str("0x%02X", PacketLength),
                                      sprintf_str("0x%02X", HammingCode), sprintf_str("0x%02X", ApplicationVersion), sprintf_str("0x%02X", ERTType),
                                      u(ERTSerialNumber), u(ConsumptionIntervalCount), sprintf_str("0x%02X", ModuleProgrammingState),
                                      hexbytes(TamperCounters.data(), 6), sprintf_str("0x%02X", AsynchronousCounters),
                                      hexbytes(PowerOutageFlags.data(), 6), u(LastConsumptionCount)};
        for (uint16_t v : DifferentialConsumptionIntervals) r.push_back(u(v));
        r.push_back(u(TransmitTimeOffset));
        r.push_back(sprintf_str("0x%04X", SerialNumberCRC));
        r.push_back(sprintf_str("0x%04X", PacketCRC));
        return r;
    }
    std::vector<Field> Fields() const override {  // idm.go:101-119, no tags
        return {fu("Preamble", Preamble), fu("PacketTypeID", PacketTypeID), fu("PacketLength", PacketLength),
                fu("HammingCode", HammingCode), fu("ApplicationVersion", ApplicationVersion), fu("ERTType", ERTType),
                fu("ERTSerialNumber", ERTSerialNumber), fu("ConsumptionIntervalCount", ConsumptionIntervalCount),
                fu("ModuleProgrammingState", ModuleProgrammingState), fbytes("TamperCounters", TamperCounters.data(), 6),
                fu("AsynchronousCounters", AsynchronousCounters), fbytes("PowerOutageFlags", PowerOutageFlags.data(), 6),
                fu("LastConsumptionCount", LastConsumptionCount),
                fu16s("DifferentialConsumptionIntervals", DifferentialConsumptionIntervals.data(), 47),
                fu("TransmitTimeOffset", TransmitTimeOffset), fu("SerialNumberCRC", SerialNumberCRC), fu("PacketCRC", PacketCRC)};
    }
};

struct NetIDM : Message {  // netidm/netidm.go:112-129
    uint32_t Preamble = 0;
    uint8_t ProtocolID = 0, PacketLength = 0, HammingCode = 0, ApplicationVersion = 0, ERTType = 0;
    uint32_t ERTSerialNumber = 0;
    uint8_t ConsumptionIntervalCount = 0, ProgrammingState = 0;
    uint32_t LastGeneration = 0, LastConsumption = 0, LastConsumptionNet = 0;
    std::array<uint16_t, 27> DifferentialConsumptionIntervals{};
    uint16_t TransmitTimeOffset = 0, SerialNumberCRC = 0, PacketCRC = 0;
    std::string MsgType() const override { return "NetIDM"; }
    uint32_t MeterID() const override { return ERTSerialNumber; }
    uint8_t MeterType() const override { return ERTType; }
    std::vector<uint8_t> Checksum() const override { return {(uint8_t)(PacketCRC >> 8), (uint8_t)PacketCRC}; }
    std::string String() const override {  // netidm.go:188-209
        std::string s = "{";
        s += sprintf_str("Preamble:0x%08X ProtocolID:0x%02X PacketLength:0x%02X HammingCode:0x%02X ", Preamble, ProtocolID, PacketLength, HammingCode);
        s += sprintf_str("ApplicationVersion:0x%02X ERTType:0x%02X ERTSerialNumber:% 10lld ", ApplicationVersion, ERTType, (long long)ERTSerialNumber);
        s += sprintf_str("ConsumptionIntervalCount:%u ProgrammingState:0x%02X ", ConsumptionIntervalCount, ProgrammingState);
        s += sprintf_str("LastGeneration:%u LastConsumption:%u LastConsumptionNet:%u ", LastGeneration, LastConsumption, LastConsumptionNet);
        s += "DifferentialConsumptionIntervals:" + join_u16(DifferentialConsumptionIntervals.data(), 27);
        s += sprintf_str(" TransmitTimeOffset:%u SerialNumberCRC:0x%04X PacketCRC:0x%04X}", TransmitTimeOffset, SerialNumberCRC, PacketCRC);
        return s;
    }
    std::vector<std::string> Record() const override {  // netidm.go:211-232
        std::vector<std::string> r = {sprintf_str("0x%08X", Preamble), sprintf_str("0x%02X", ProtocolID), sprintf_str("0x%02X", PacketLength),
                                      sprintf_str("0x%02X", HammingCode), sprintf_str("0x%02X", ApplicationVersion), sprintf_str("0x%02X", ERTType),
                                      u(ERTSerialNumber), u(ConsumptionIntervalCount), sprintf_str("0x%02X", ProgrammingState),
                                      u(LastGeneration), u(LastConsumption), u(LastConsumptionNet)};
        for (uint16_t v : DifferentialConsumptionIntervals) r.push_back(u(v));
        r.push_back(u(TransmitTimeOffset));
        r.push_back(sprintf_str("0x%04X", SerialNumberCRC));
        r.push_back(sprintf_str("0x%04X", PacketCRC));
        return r;
    }
    std::vector<Field> Fields() const override {  // netidm.go:112-129, no tags
        return {fu("Preamble", Preamble), fu("ProtocolID", ProtocolID), fu("PacketLength", PacketLength),
                fu("HammingCode", HammingCode), fu("ApplicationVersion", ApplicationVersion), fu("ERTType", ERTType),
                fu("ERTSerialNumber", ERTSerialNumber), fu("ConsumptionIntervalCount", ConsumptionIntervalCount),
                fu("ProgrammingState", ProgrammingState), fu("LastGeneration", LastGeneration), fu("LastConsumption", LastConsumption),
                fu("LastConsumptionNet", LastConsumptionNet),
                fu16s("DifferentialConsumptionIntervals", DifferentialConsumptionIntervals.data(), 27),
                fu("TransmitTimeOffset", TransmitTimeOffset), fu("SerialNumberCRC", SerialNumberCRC), fu("PacketCRC", PacketCRC)};
    }
};

struct R900 : Message {  // r900/r900.go:248-258
    uint32_t ID = 0;
    uint8_t Unkn1 = 0, NoUse = 0, BackFlow = 0;
    uint32_t Consumption = 0;
    uint8_t Unkn3 = 0, Leak = 0, LeakNow = 0;
    std::array<uint8_t, 5> checksum{};
    bool bcd = false;
    std::string MsgType() const override { return bcd ? "R900BCD" : "R900"; }  // r900bcd.go:43-45
    uint32_t MeterID() const override { return ID; }
    uint8_t MeterType() const override { return Unkn1; }
    std::vector<uint8_t> Checksum() const override { return std::vector<uint8_t>(checksum.begin(), checksum.end()); }
    std::string String() const override {  // r900.go:278-289
        return sprintf_str("{ID:%10u Unkn1:0x%02X NoUse:%2u BackFlow:%1u Consumption:%8u Unkn3:0x%02X Leak:%2u LeakNow:%1u}", ID, Unkn1,
                           NoUse, BackFlow, Consumption, Unkn3, Leak, LeakNow);
    }
    std::vector<std::string> Record() const override {  // r900.go:291-302
        return {u(ID), u(Unkn1), u(NoUse), u(BackFlow), u(Consumption), u(Unkn3), u(Leak), u(LeakNow)};
    }
    // r900.go:248-258; `checksum` is unexported.  R900BCD embeds r900.R900 (r900bcd.go:39-41), so its fields are these.
    std::vector<Field> Fields() const override {
        return {fattr("ID", ID), fattr("Unkn1", Unkn1), fattr("NoUse", NoUse), fattr("BackFlow", BackFlow),
                fattr("Consumption", Consumption), fattr("Unkn3", Unkn3), fattr("Leak", Leak), fattr("LeakNow", LeakNow)};
    }
};

// ----------------------------------------------------------------------- parsers
PacketConfig base_cfg(const char* name, const char* preamble, int ps, int pk, int chipLength, uint32_t cf = 912600155u) {
    PacketConfig c;
    c.Protocol = name;
    c.CenterFreq = cf;
    c.DataRate = 32768;
    c.ChipLength = chipLength;
    c.PreambleSymbols = ps;
    c.PacketSymbols = pk;
    c.Preamble = preamble;
    return c;
}

void stamp(Message& m, const Data& d) {
    m.Block = d.Block;
    m.Idx = d.Idx;
}

struct ScmParser : Parser {  // scm/scm.go:33-90
    crc::CRC crc_ = crc::NewCRC("BCH", 0, 0x6F63, 0);
    PacketConfig cfg_;
    explicit ScmParser(int cl) : cfg_(base_cfg("scm", "111110010101001100000", 21, 96, cl)) {}
    PacketConfig Cfg() const override { return cfg_; }
    void Screen(ertgpu_protocol& p) const override {
        p.check_kind = ERTGPU_CHECK_CRC16; p.crc_init = crc_.Init; p.crc_poly = crc_.Poly; p.crc_residue = 0; p.crc_from = 2; p.crc_to = 12;
    }
    void Parse(const std::vector<Data>& pkts, std::vector<MessagePtr>& msgCh) override {
        std::set<std::string> seen;
        for (const Data& pkt : pkts) {
            uint8_t b[12] = {0};
            memcpy(b, pkt.Bytes.data(), std::min<size_t>(12, pkt.Bytes.size()));  // scm.go:66-67
            const std::string bits = pkt.Bits.substr(0, 96);
            if (!seen.insert(std::string((const char*)b, 12)).second) continue;    // scm.go:69-73
            if (crc_.Checksum(b + 2, 10) != 0) continue;                           // scm.go:76
            auto m = std::make_unique<SCM>();                                      // scm.go:103-119
            m->ID = (uint32_t)bits_uint(bits, 21, 23) << 24 | (uint32_t)bits_uint(bits, 56, 80);
            m->Type = (uint8_t)bits_uint(bits, 26, 30);
            m->TamperPhy = (uint8_t)bits_uint(bits, 24, 26);
            m->TamperEnc = (uint8_t)bits_uint(bits, 30, 32);
            m->Consumption = (uint32_t)bits_uint(bits, 32, 56);
            m->ChecksumVal = (uint16_t)bits_uint(bits, 80, 96);
            if (m->ID == 0) continue;                                              // scm.go:83-85
            stamp(*m, pkt);
            msgCh.push_back(std::move(m));
        }
    }
};

struct ScmPlusParser : Parser {  // scmplus/scmplus.go:32-90
    crc::CRC crc_ = crc::NewCRC("CCITT", 0xFFFF, 0x1021, 0x1D0F);
    PacketConfig cfg_;
    explicit ScmPlusParser(int cl) : cfg_(base_cfg("scm+", "0001011010100011", 16, 16 * 8, cl)) {}
    PacketConfig Cfg() const override { return cfg_; }
    void Screen(ertgpu_protocol& p) const override {
        p.check_kind = ERTGPU_CHECK_CRC16; p.crc_init = crc_.Init; p.crc_poly = crc_.Poly; p.crc_residue = crc_.Residue; p.crc_from = 2; p.crc_to = 16;
    }
    void Parse(const std::vector<Data>& pkts, std::vector<MessagePtr>& msgCh) override {
        std::set<std::string> seen;
        for (const Data& pkt : pkts) {
            uint8_t b[16] = {0};
            memcpy(b, pkt.Bytes.data(), std::min<size_t>(16, pkt.Bytes.size()));
            if (!seen.insert(std::string((const char*)b, 16)).second) continue;
            if (crc_.Checksum(b + 2, 14) != crc_.Residue) continue;  // scmplus.go:77
            auto m = std::make_unique<SCMPlus>();                     // scmplus.go:105-109 (big-endian struct read)
            m->FrameSync = be16(b);
            m->ProtocolID = b[2];
            m->EndpointType = b[3];
            m->EndpointID = be32(b + 4);
            m->Consumption = be32(b + 8);
            m->Tamper = be16(b + 12);
            m->PacketCRC = be16(b + 14);
            if (m->EndpointID == 0 || m->ProtocolID != 0x1E) continue;  // scmplus.go:84-86
            stamp(*m, pkt);
            msgCh.push_back(std::move(m));
        }
    }
};

template <bool NET>
struct IdmParser : Parser {  // idm/idm.go:30-98, netidm/netidm.go:30-109
    crc::CRC crc_ = crc::NewCRC("CCITT", 0xFFFF, 0x1021, 0x1D0F);
    PacketConfig cfg_;
    explicit IdmParser(int cl) : cfg_(base_cfg(NET ? "netidm" : "idm", "01010101010101010001011010100011", 32, 92 * 8, cl)) {}
    PacketConfig Cfg() const override { return cfg_; }
    void Screen(ertgpu_protocol& p) const override {
        p.check_kind = ERTGPU_CHECK_IDM; p.crc_init = crc_.Init; p.crc_poly = crc_.Poly; p.crc_residue = crc_.Residue; p.crc_from = 4; p.crc_to = 92;
    }
    void Parse(const std::vector<Data>& pkts, std::vector<MessagePtr>& msgCh) override {
        std::set<std::string> seen;
        for (const Data& pkt : pkts) {
            uint8_t b[92] = {0};
            memcpy(b, pkt.Bytes.data(), std::min<size_t>(92, pkt.Bytes.size()));
            if (!seen.insert(std::string((const char*)b, 92)).second) continue;
            if (crc_.Checksum(b + 4, 88) != crc_.Residue) continue;  // idm.go:77
            uint8_t buf[6];
            memcpy(buf, b + 9, 4);                                   // idm.go:82-84
            memcpy(buf + 4, b + 88, 2);
            if (crc_.Checksum(buf, 6) != crc_.Residue) continue;     // idm.go:85
            const std::string& bits = pkt.Bits;
            if constexpr (!NET) {
                auto m = std::make_unique<IDM>();  // idm.go:121-156
                m->Preamble = be32(b);
                m->PacketTypeID = b[4]; m->PacketLength = b[5]; m->HammingCode = b[6]; m->ApplicationVersion = b[7];
                m->ERTType = b[8] & 0x0F;
                m->ERTSerialNumber = be32(b + 9);
                m->ConsumptionIntervalCount = b[13];
                m->ModuleProgrammingState = b[14];
                memcpy(m->TamperCounters.data(), b + 15, 6);
                m->AsynchronousCounters = be16(b + 21);
                memcpy(m->PowerOutageFlags.data(), b + 23, 6);
                m->LastConsumptionCount = be32(b + 29);
                int off = 264;
                for (auto& iv : m->DifferentialConsumptionIntervals) { iv = (uint16_t)bits_uint(bits, off, off + 9); off += 9; }
                m->TransmitTimeOffset = be16(b + 86); m->SerialNumberCRC = be16(b + 88); m->PacketCRC = be16(b + 90);
                if (m->ERTSerialNumber == 0) continue;  // idm.go:90-92
                stamp(*m, pkt);
                msgCh.push_back(std::move(m));
            } else {
                auto m = std::make_unique<NetIDM>();  // netidm.go:131-160
                m->Preamble = be32(b);
                m->ProtocolID = b[4]; m->PacketLength = b[5]; m->HammingCode = b[6]; m->ApplicationVersion = b[7];
                m->ERTType = b[8] & 0x0F;
                m->ERTSerialNumber = be32(b + 9);
                m->ConsumptionIntervalCount = b[13];
                m->ProgrammingState = b[14];
                m->LastConsumption = (uint32_t)b[25] << 16 | (uint32_t)b[26] << 8 | b[27];
                m->LastGeneration = (uint32_t)b[28] << 16 | (uint32_t)b[29] << 8 | b[30];
                m->LastConsumptionNet = be32(b + 34);
                int off = 38 << 3;
                for (auto& iv : m->DifferentialConsumptionIntervals) { iv = (uint16_t)bits_uint(bits, off, off + 14); off += 14; }
                m->TransmitTimeOffset = be16(b + 86); m->SerialNumberCRC = be16(b + 88); m->PacketCRC = be16(b + 90);
                if (m->ERTSerialNumber == 0) continue;  // netidm.go:103-105
                stamp(*m, pkt);
                msgCh.push_back(std::move(m));
            }
        }
    }
};

// r900/r900.go:160-245.  The DSP half of the reference parser (its own signal history, running
// sum and 4-chip correlators, r900.go:82-150,168-172) runs on the GPU; the candidate arrives with
// the 42 payload digits the reference would read from p.quantized (r900.go:187-193).
struct R900Parser : Parser {
    PacketConfig cfg_;
    gf::Field field_;
    std::array<uint8_t, 31> rsBuf_{};
    bool bcd_;
    R900Parser(int cl, bool bcd) : cfg_(base_cfg(bcd ? "r900bcd" : "r900", "00000000000000001110010101100100", 32, 116, cl, 912380000u)), bcd_(bcd) {}
    PacketConfig Cfg() const override { return cfg_; }
    void Screen(ertgpu_protocol& p) const override { p.check_kind = ERTGPU_CHECK_R900; }
    void Parse(const std::vector<Data>& pkts, std::vector<MessagePtr>& msgCh) override {
        std::set<std::string> seen;
        for (const Data& pkt : pkts) {
            if (!pkt.HasR900) throw std::logic_error("r900: candidate without payload digits");
            uint8_t symbols[21];
            std::string bits;
            bool bad = false;
            for (int k = 0; k < 21; k++) {  // r900.go:199-207: two base-6 digits per 5-bit symbol
                const int sym = pkt.R900Digits[(size_t)(2 * k)] * 6 + pkt.R900Digits[(size_t)(2 * k + 1)];
                if (sym > 31) { bad = true; break; }
                symbols[k] = (uint8_t)sym;
                for (int j = 4; j >= 0; j--) bits.push_back(((sym >> j) & 1) ? '1' : '0');
            }
            if (bad || !seen.insert(bits).second) continue;  // r900.go:209-213
            memcpy(rsBuf_.data(), symbols, 16);              // r900.go:215-216
            memcpy(rsBuf_.data() + 26, symbols + 16, 5);
            const auto syn = field_.Syndrome(rsBuf_.data(), 31, 5, 29);
            if (std::any_of(syn.begin(), syn.end(), [](uint8_t v) { return v != 0; })) continue;  // r900.go:219-221
            auto m = std::make_unique<R900>();  // r900.go:223-242
            m->ID = (uint32_t)bits_uint(bits, 0, 32);
            m->Unkn1 = (uint8_t)bits_uint(bits, 32, 40);
            m->NoUse = (uint8_t)bits_uint(bits, 40, 46);
            m->BackFlow = (uint8_t)bits_uint(bits, 46, 48);
            m->Consumption = (uint32_t)bits_uint(bits, 48, 72);
            m->Unkn3 = (uint8_t)bits_uint(bits, 72, 74);
            m->Leak = (uint8_t)bits_uint(bits, 74, 78);
            m->LeakNow = (uint8_t)bits_uint(bits, 78, 80);
            memcpy(m->checksum.data(), symbols + 16, 5);
            if (bcd_) {  // r900bcd.go:63-65: the hex rendering re-read as decimal; a non-decimal digit parses to 0
                m->bcd = true;
                uint32_t v = m->Consumption, out = 0, mul = 1;
                bool ok = true;
                while (v) {
                    const uint32_t d = v & 0xF;
                    if (d > 9) { ok = false; break; }
                    out += d * mul;
                    mul *= 10;
                    v >>= 4;
                }
                m->Consumption = ok ? out : 0;
            }
            stamp(*m, pkt);
            msgCh.push_back(std::move(m));
        }
    }
};

}  // namespace

void RegisterStockParsers() {
    static std::once_flag once;
    std::call_once(once, [] {
        RegisterParser("scm", [](int cl) { return std::make_shared<ScmParser>(cl); });
        RegisterParser("scm+", [](int cl) { return std::make_shared<ScmPlusParser>(cl); });
        RegisterParser("idm", [](int cl) { return std::make_shared<IdmParser<false>>(cl); });
        RegisterParser("netidm", [](int cl) { return std::make_shared<IdmParser<true>>(cl); });
        RegisterParser("r900", [](int cl) { return std::make_shared<R900Parser>(cl, false); });
        RegisterParser("r900bcd", [](int cl) { return std::make_shared<R900Parser>(cl, true); });
    });
}

// ----------------------------------------------------------------------- Decoder
namespace {
[[noreturn]] void raise(ertgpu_handle* h, int rc, const char* what) {
    throw std::runtime_error(std::string(what) + ": libertgpu error " + std::to_string(rc) + ": " + ertgpu_last_error(h));
}
}  // namespace

Decoder::Decoder() {
    int rc = ertgpu_create(&h_);
    if (rc != ERTGPU_OK) throw std::runtime_error("ertgpu_create failed");
}

Decoder::~Decoder() { ertgpu_destroy(h_); }

void Decoder::RegisterProtocol(ParserPtr p) {
    if (!p) throw std::logic_error("RegisterProtocol(nil)");  // the reference dereferences nil here (main.go:77-82)
    p->SetDecoder(this);                                        // decode.go:102
    const PacketConfig pc = p->Cfg();
    ertgpu_protocol ep;
    memset(&ep, 0, sizeof(ep));
    snprintf(ep.name, sizeof(ep.name), "%s", pc.Protocol.c_str());
    snprintf(ep.preamble, sizeof(ep.preamble), "%s", pc.Preamble.c_str());
    ep.data_rate = pc.DataRate;
    ep.chip_length = pc.ChipLength;
    ep.preamble_symbols = pc.PreambleSymbols;
    ep.packet_symbols = pc.PacketSymbols;
    ep.center_freq = pc.CenterFreq;
    p->Screen(ep);
    int rc = ertgpu_register_protocol(h_, &ep);
    if (rc != ERTGPU_OK) raise(h_, rc, "RegisterProtocol");
    // decode.go:105-109
    Cfg.CenterFreq = pc.CenterFreq;
    Cfg.DataRate = std::max(Cfg.DataRate, pc.DataRate);
    Cfg.ChipLength = std::max(Cfg.ChipLength, pc.ChipLength);
    Cfg.PreambleSymbols = std::max(Cfg.PreambleSymbols, pc.PreambleSymbols);
    Cfg.PacketSymbols = std::max(Cfg.PacketSymbols, pc.PacketSymbols);
    size_t pre = 0;
    for (; pre < preambles_.size(); pre++)
        if (preambles_[pre] == pc.Preamble) break;
    if (pre == preambles_.size()) {  // decode.go:121-124
        preambles_.push_back(pc.Preamble);
        by_pre_.emplace_back();
    }
    by_pre_[pre].push_back(parsers_.size());
    parsers_.push_back(std::move(p));
}

void Decoder::Allocate(int device, int64_t maxBlocksPerCall, int64_t maxCandidates) {
    int rc = ertgpu_allocate(h_, device, maxBlocksPerCall, maxCandidates);
    if (rc == ERTGPU_EINVAL && ertgpu_get_tuning(h_, nullptr) == ERTGPU_OK) throw std::invalid_argument(ertgpu_last_error(h_));  // the channel at the native rate
    if (rc != ERTGPU_OK) raise(h_, rc, "Allocate");
    // a tuned handle at the decoder's own rate gets its resampler here
    resampling_ = ertgpu_get_resampler(h_, &rs_, nullptr, 0, nullptr) == ERTGPU_OK;
    ertgpu_decoder_config c;
    ertgpu_get_config(h_, &c);
    Cfg.SymbolLength = c.symbol_length;  // decode.go:132-141
    Cfg.SampleRate = c.sample_rate;
    Cfg.PreambleLength = c.preamble_length;
    Cfg.PacketLength = c.packet_length;
    Cfg.BlockSize = c.block_size;
    Cfg.BlockSize2 = c.block_size2;
    Cfg.BufferLength = c.buffer_length;
    ertgpu_tuning_info t{};
    SetSignalChannel(ertgpu_get_tuning(h_, &t) == ERTGPU_OK ? t.center_hz : (int64_t)Cfg.CenterFreq, c.sample_rate);
    allocated_ = true;
}

void Decoder::EnableSignal() {
    if (allocated_) throw std::logic_error("EnableSignal after Allocate");
    const int rc = ertgpu_enable_signal(h_);
    if (rc != ERTGPU_OK) raise(h_, rc, "EnableSignal");
    signal_ = true;
}

void Decoder::EnableSpectrum(int32_t log2_n, int64_t frames_per_row) {
    if (allocated_) throw std::logic_error("EnableSpectrum after Allocate");
    const int rc = ertgpu_enable_spectrum(h_, log2_n, frames_per_row);
    if (rc == ERTGPU_EINVAL) throw std::invalid_argument(ertgpu_last_error(h_));
    if (rc != ERTGPU_OK) raise(h_, rc, "EnableSpectrum");
    spectrum_n_ = 1 << log2_n;
}

SpectrumRows Decoder::FetchSpectrum(bool partial) {
    SpectrumRows r;
    r.N = spectrum_n_;
    size_t n = 0;
    int rc = ertgpu_fetch_spectrum(h_, partial, nullptr, nullptr, nullptr, 0, &n);
    if (rc != ERTGPU_OK && rc != ERTGPU_ECAPACITY) raise(h_, rc, "FetchSpectrum");
    if (n == 0) return r;
    r.rows.resize(n);
    r.mean.resize(n * (size_t)r.N);
    r.peak.resize(n * (size_t)r.N);
    rc = ertgpu_fetch_spectrum(h_, partial, r.rows.data(), r.mean.data(), r.peak.data(), n, &n);
    if (rc != ERTGPU_OK) raise(h_, rc, "FetchSpectrum");
    return r;
}

const ertgpu_signal* Decoder::FetchSignal(size_t n) {
    if (!signal_) return nullptr;
    sigs_.resize(std::max<size_t>(n, 1));
    size_t got = 0;
    const int rc = ertgpu_fetch_signal(h_, sigs_.data(), sigs_.size(), &got);
    if (rc != ERTGPU_OK) raise(h_, rc, "FetchSignal");
    if (got != n) throw std::logic_error("FetchSignal: the records do not match the candidates");
    return sigs_.data();
}

void Decoder::Reset() {
    int rc = ertgpu_reset(h_);
    if (rc != ERTGPU_OK) raise(h_, rc, "Reset");
    input_samples_ = 0;
}

void Decoder::SetInput(const Input& in) {
    if (allocated_) throw std::logic_error("SetInput after Allocate");
    const auto check = [this](int rc) {
        if (rc == ERTGPU_EINVAL) throw std::invalid_argument(ertgpu_last_error(h_));
        if (rc != ERTGPU_OK) raise(h_, rc, "SetInput");
    };
    if (in.CaptureFreq > 0 || in.CenterFreq != 0) {
        check(ertgpu_set_input_tuning(h_, in.CaptureFreq, in.CenterFreq));
        check(ertgpu_allow_input_decimation(h_));  // up to 256:1; nothing changes up to 10:1
    }
    if (in.SampleRate > 0) check(ertgpu_set_input_rate(h_, in.SampleRate));
    if (in.AutoScale && in.Format == ERTGPU_FORMAT_CU8) throw std::invalid_argument("automatic gain does not apply to uint8 (cu8) input");
    if (in.Format != ERTGPU_FORMAT_CU8 || in.Scale != 0.0f) {
        check(ertgpu_set_input_format(h_, in.Format, in.Scale));
        sample_bytes_ = FormatBytes(in.Format);
    }
    auto_scale_ = in.AutoScale;
    if (in.ChannelGain >= 0 || in.AutoChannelGain) {
        if (in.CaptureFreq <= 0) throw std::invalid_argument("the channel gain needs a tuned input: a capture frequency");
        check(ertgpu_set_channel_gain(h_, in.AutoChannelGain ? 0 : in.ChannelGain));
    }
    auto_channel_gain_ = in.AutoChannelGain;
    if (in.Signal) EnableSignal();
    if (in.SpectrumLog2) EnableSpectrum(in.SpectrumLog2, in.SpectrumFrames);
}

ertgpu_channel_level Decoder::MeasureChannel(const uint8_t* samples, size_t len) {
    if (!allocated_) throw std::logic_error("MeasureChannel before Allocate");
    ertgpu_channel_level lv{};
    const int rc = ertgpu_measure_channel(h_, samples, len, &lv);
    if (rc != ERTGPU_OK) raise(h_, rc, "MeasureChannel");
    return lv;
}

void Decoder::SetChannelGain(int32_t k) {
    const int rc = ertgpu_set_channel_gain(h_, k);
    if (rc == ERTGPU_EINVAL) throw std::invalid_argument(ertgpu_last_error(h_));
    if (rc != ERTGPU_OK) raise(h_, rc, "SetChannelGain");
}

ertgpu_input_level Decoder::Measure(const uint8_t* samples, size_t len) {
    if (!allocated_) throw std::logic_error("Measure before Allocate");
    ertgpu_input_level lv{};
    const int rc = ertgpu_measure_input(h_, samples, len, &lv);
    if (rc != ERTGPU_OK) raise(h_, rc, "Measure");
    return lv;
}

void Decoder::SetScale(float scale) {
    const int rc = ertgpu_set_input_scale(h_, scale);
    if (rc == ERTGPU_EINVAL) throw std::invalid_argument(ertgpu_last_error(h_));
    if (rc != ERTGPU_OK) raise(h_, rc, "SetScale");
}

int64_t Decoder::BlocksDecoded() const {
    if (!allocated_ || Cfg.BlockSize <= 0) return 0;
    return (resampling_ ? ertrs_out_end(&rs_, input_samples_) : input_samples_) / Cfg.BlockSize;
}

std::vector<std::vector<MessagePtr>> Decoder::DecodeChannels(const std::vector<Decoder*>& ds, const uint8_t* input, size_t len) {
    if (ds.empty()) throw std::invalid_argument("DecodeChannels without a channel");
    for (const Decoder* d : ds)
        if (!d->allocated_) throw std::logic_error("Decode before Allocate");
    Decoder& d0 = *ds[0];
    if (len % d0.InputQuantum()) throw std::length_error("input is not a whole number of IQ samples");
    std::vector<ertgpu_handle*> hs;
    for (const Decoder* d : ds) hs.push_back(d->h_);
    int rc = ertgpu_decode_channels(hs.data(), (int32_t)hs.size(), input, len, ERTGPU_DECODE_ONLY_VALID);
    if (rc == ERTGPU_EINVAL) throw std::invalid_argument(ertgpu_last_error(d0.h_));
    if (rc != ERTGPU_OK) raise(d0.h_, rc, "DecodeChannels");
    std::vector<std::vector<MessagePtr>> out(ds.size());
    for (size_t c = 0; c < ds.size(); c++) {
        Decoder& d = *ds[c];
        size_t n = 0;
        if (d.cands_.size() < 1024) d.cands_.resize(1024);
        rc = ertgpu_fetch(d.h_, d.cands_.data(), d.cands_.size(), &n);
        if (rc == ERTGPU_ECAPACITY && n > d.cands_.size() && std::string(ertgpu_last_error(d.h_)).find("internal") == std::string::npos) {
            d.cands_.resize(n);
            rc = ertgpu_fetch(d.h_, d.cands_.data(), d.cands_.size(), &n);
        }
        if (rc != ERTGPU_OK) raise(d.h_, rc, "DecodeChannels");
        d.input_samples_ += (int64_t)(len / d.sample_bytes_);
        d.Dispatch(d.cands_.data(), n, out[c], d.FetchSignal(n));
    }
    return out;
}

std::vector<MessagePtr> Decoder::Decode(const uint8_t* input, size_t len) {
    if (!allocated_) throw std::logic_error("Decode before Allocate");
    if (len % InputQuantum())
        throw std::length_error(resampling_ ? "input is not a whole number of IQ samples"
                                            : sample_bytes_ == 2 ? "input is not a whole number of BlockSize2-byte blocks"
                                                                 : "input is not a whole number of blocks");
    size_t n = 0;
    if (cands_.size() < 1024) cands_.resize(1024);
    int rc = ertgpu_decode(h_, input, len, ERTGPU_DECODE_ONLY_VALID, cands_.data(), cands_.size(), &n);
    if (rc == ERTGPU_ECAPACITY && n > cands_.size() && std::string(ertgpu_last_error(h_)).find("internal") == std::string::npos) {
        cands_.resize(n);
        rc = ertgpu_fetch(h_, cands_.data(), cands_.size(), &n);
    }
    if (rc != ERTGPU_OK) raise(h_, rc, "Decode");
    input_samples_ += (int64_t)(len / sample_bytes_);

    std::vector<MessagePtr> out;
    Dispatch(cands_.data(), n, out, FetchSignal(n));
    return out;
}

// Rebuild the reference's per-block, per-preamble []Data lists (decode.go:177-187) and hand each to
// the parsers filed under that preamble.  Candidates arrive sorted by (block, preamble, idx).
// Decode only fetches candidates that passed a GPU screen: a parser would reject the others at its own
// checksum test, after the same `seen` bookkeeping, so the emitted messages are identical.
void Decoder::Dispatch(const ertgpu_candidate* cands, size_t n, std::vector<MessagePtr>& out, const ertgpu_signal* sigs) {
    const size_t nbytes = (size_t)((Cfg.PacketSymbols + 7) >> 3);
    size_t i = 0;
    while (i < n) {
        size_t j = i;
        std::vector<Data> pkts;
        if (cands[i].preamble_id < 0 || (size_t)cands[i].preamble_id >= by_pre_.size())
            throw std::out_of_range("candidate with an unregistered preamble");
        while (j < n && cands[j].block == cands[i].block && cands[j].preamble_id == cands[i].preamble_id) {
            const ertgpu_candidate& c = cands[j];
            Data d = NewData(c.bytes, nbytes);
            d.Idx = c.idx;
            d.Block = c.block;
            d.CheckMask = c.check_mask;
            d.HasR900 = (c.flags & ERTGPU_CAND_HAS_R900) != 0;
            memcpy(d.R900Digits.data(), c.r900_digits, ERTGPU_R900_DIGITS);
            pkts.push_back(std::move(d));
            j++;
        }
        const size_t first = out.size();
        for (size_t pi : by_pre_[(size_t)cands[i].preamble_id]) parsers_[pi]->Parse(pkts, out);
        for (size_t k = first; sigs && k < out.size(); k++) {  // this block and preamble: the candidate with the message's Idx
            size_t c = i;
            while (c < j && cands[c].idx != out[k]->Idx) c++;
            if (c == j) throw std::logic_error("a message without its candidate");
            SignalReport r;
            r.Channel = signal_channel_;
            ertsig_summary_t s;
            if ((r.Valid = ertsig_summary(&sigs[c], signal_channel_, signal_rate_, &s) != 0)) {
                r.Freq = s.freq_hz;
                r.Level = s.level_db;
                r.Noise = s.noise_db;
                r.SNR = s.snr_db;
            }
            out[k]->Signal = r;
        }
        i = j;
    }
}

std::string Decoder::Log() const {  // decode.go:73-90
    std::string s;
    ertgpu_tuning_info t;
    if (ertgpu_get_tuning(h_, &t) == ERTGPU_OK) {  // the channel decoded, and the capture's centre
        s += "CenterFreq: " + std::to_string(t.center_hz) + "\nCaptureFreq: " + std::to_string(t.capture_center_hz);
        ertgpu_decimator_info d;
        if (ertgpu_get_decimator(h_, &d, nullptr, 0, nullptr) == ERTGPU_OK && d.D > 1) {  // above 10:1: the first stage
            char mid[64];
            snprintf(mid, sizeof(mid), "%.3f", (double)d.rate_in / d.D);
            s += "\nDecimation: " + std::to_string(d.D) + "\nIntermediateRate: " + mid;
        }
    } else {
        s += "CenterFreq: " + u(Cfg.CenterFreq);
    }
    s += "\nSampleRate: " + u((uint64_t)Cfg.SampleRate) + "\nDataRate: " + u((uint64_t)Cfg.DataRate);
    s += "\nChipLength: " + u((uint64_t)Cfg.ChipLength) + "\nPreambleSymbols: " + u((uint64_t)Cfg.PreambleSymbols);
    s += "\nPreambleLength: " + u((uint64_t)Cfg.PreambleLength) + "\nPacketSymbols: " + u((uint64_t)Cfg.PacketSymbols);
    s += "\nPacketLength: " + u((uint64_t)Cfg.PacketLength) + "\nProtocols: ";
    for (size_t i = 0; i < parsers_.size(); i++) s += (i ? "," : "") + parsers_[i]->Cfg().Protocol;
    s += "\nPreambles: ";
    for (size_t i = 0; i < preambles_.size(); i++) s += (i ? "," : "") + preambles_[i];
    return s + "\n";
}

}  // namespace protocol
