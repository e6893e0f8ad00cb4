// ssq_samhdr.h — SAM header lines as sambamba 0.5.9 writes them into a BAM it makes (sort, merge): host code shared by
// ssq_bam_header_text (ssq_mem.cu) and the merged header of ssq_merge.cuh.
#pragma once
#include <string>
#include <vector>

// The tags of @SQ / @RG / @PG lines in sambamba's fixed field order (v0.5.9: SQ: SN LN AS M5 SP UR; RG: ID CN DS DT FO KS LB PG PI
// PL PU SM; PG: ID PN CL PP VN), tags it does not know after them in input order.  Other lines (@CO) pass through.
static void reorder_tags(const std::string &line, std::string &out)
{
	static const char *SQ[] = {"SN", "LN", "AS", "M5", "SP", "UR", 0}, *RG[] = {"ID", "CN", "DS", "DT", "FO", "KS", "LB", "PG", "PI", "PL", "PU", "SM", 0}, *PG[] = {"ID", "PN", "CL", "PP", "VN", 0};
	const char **ord = !line.compare(0, 3, "@SQ") ? SQ : !line.compare(0, 3, "@RG") ? RG : !line.compare(0, 3, "@PG") ? PG : 0;
	if (!ord) { out += line; out += '\n'; return; }
	std::vector<std::string> f;
	for (size_t p = 0;;) { const size_t e = line.find('\t', p); f.push_back(line.substr(p, e == std::string::npos ? e : e - p)); if (e == std::string::npos) break; p = e + 1; }
	std::vector<char> used(f.size(), 0);
	out += f[0];
	for (int k = 0; ord[k]; ++k)
		for (size_t i = 1; i < f.size(); ++i) if (!used[i] && f[i].size() >= 3 && f[i][2] == ':' && !f[i].compare(0, 2, ord[k])) { out += '\t'; out += f[i]; used[i] = 1; }
	for (size_t i = 1; i < f.size(); ++i) if (!used[i]) { out += '\t'; out += f[i]; }
	out += '\n';
}
